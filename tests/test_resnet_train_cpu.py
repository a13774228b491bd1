"""The training-mode ResNet (slim resnet_v2_50 with is_training=True) without a GPU: the TF stand-in's training batch_norm against the
TF API-doc formulas, the float64 oracle against the reference's own encoder_resnet run over that stand-in (resnet_train_bn_v1.npz),
and the host-side wiring of nets.ResNetTrainPlan on a stubbed device."""
import importlib
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUBS = os.path.join(ROOT, 'oracle', 'ref_exec', 'stubs')
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'resnet_train_bn_v1.npz')


@pytest.fixture(scope='module')
def tf():
    """The stand-in as `tensorflow` with the training batch_norm installed, for this module only."""
    before = set(sys.modules)
    sys.path.insert(0, STUBS)
    try:
        mod = importlib.import_module('tensorflow')
        spec = importlib.util.spec_from_file_location('_train_bn', os.path.join(ROOT, 'oracle', 'ref_exec', 'train_bn.py'))
        train_bn = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(train_bn)
        train_bn.install()
        mod._train_bn = train_bn
        yield mod
    finally:
        sys.path.remove(STUBS)
        for name in set(sys.modules) - before:
            if name == 'tensorflow' or name.startswith('tensorflow.'):
                del sys.modules[name]


def test_standin_training_batch_norm_follows_the_documented_formulas(tf):
    from tensorflow.contrib import layers
    tf.reset_default_graph()
    tf.reset_collections()
    rng = np.random.RandomState(3)
    x = (rng.normal(0, 2, size=(2, 3, 5, 8)) + 40).astype(np.float32)
    with tf.variable_scope('unit'):
        y = layers.batch_norm(tf.constant(x), decay=0.997, epsilon=1e-5, scale=True, center=True, is_training=True,
                              activation_fn=tf.nn.relu, scope='preact')
    names = sorted(v.op_name for v in tf.global_variables())
    assert names == ['unit/preact/beta', 'unit/preact/gamma', 'unit/preact/moving_mean', 'unit/preact/moving_variance']
    assert [v.op_name for v in tf.trainable_variables()] == ['unit/preact/beta', 'unit/preact/gamma']
    vals = {'unit/preact/gamma': rng.uniform(0.5, 1.5, 8), 'unit/preact/beta': rng.normal(0, 0.3, 8),
            'unit/preact/moving_mean': rng.normal(0, 1, 8), 'unit/preact/moving_variance': rng.uniform(0.5, 2, 8)}
    for v in tf.global_variables():
        v.load(vals[v.op_name])
    vals = {k: v.astype(np.float32).astype(np.float64) for k, v in vals.items()}
    xd = x.astype(np.float64)
    mean, var = xd.mean(axis=(0, 1, 2)), xd.var(axis=(0, 1, 2))          # batch moments over N, H, W; biased variance
    want = np.maximum(vals['unit/preact/gamma'] * (xd - mean) / np.sqrt(var + 1e-5) + vals['unit/preact/beta'], 0)
    sess = tf.Session()
    np.testing.assert_allclose(sess.run(y), want, rtol=1e-4, atol=1e-4)
    updates = tf.get_collection(tf.GraphKeys.UPDATE_OPS)
    assert len(updates) == 2
    mm0, mv0 = vals['unit/preact/moving_mean'], vals['unit/preact/moving_variance']
    assert np.array_equal(sess.run(y).shape, x.shape)                         # the forward alone moves nothing
    by = {v.op_name: v for v in tf.global_variables()}
    np.testing.assert_array_equal(by['unit/preact/moving_mean'].value, mm0.astype(np.float32))
    sess.run(tf.group(*updates))
    rows = 2 * 3 * 5
    np.testing.assert_allclose(by['unit/preact/moving_mean'].value, mm0 - (mm0 - mean) * (1 - 0.997), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(by['unit/preact/moving_variance'].value, mv0 - (mv0 - var * rows / (rows - 1)) * (1 - 0.997),
                               rtol=1e-6, atol=1e-6)
    # inference mode is the stand-in's unchanged batch_norm: moving statistics, no update ops
    z = layers.batch_norm(tf.constant(x), epsilon=1e-5, scale=True, is_training=False, reuse=True, scope='unit/preact')
    want_inf = vals['unit/preact/gamma'] * (xd - by['unit/preact/moving_mean'].value) / \
        np.sqrt(by['unit/preact/moving_variance'].value.astype(np.float64) + 1e-5) + vals['unit/preact/beta']
    np.testing.assert_allclose(sess.run(z), want_inf, rtol=1e-4, atol=1e-4)
    assert len(tf.get_collection(tf.GraphKeys.UPDATE_OPS)) == 2


def test_oracle_matches_the_reference_training_trunk():
    """oracle/nets_train_ref (float64) against the reference's encoder_resnet(is_training=True) + UPDATE_OPS over the stand-in (float32):
    phis, the 49 layers' batch moments and the moving statistics after one step, to the float32 rounding of the stand-in (which grows
    to about 3e-5 of a moment by block 4)."""
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.nets import BN_DECAY, resnet_bn_scopes
    from oracle import nets_train_ref
    g = np.load(GOLDEN)
    assert list(g['scopes']) == resnet_bn_scopes()
    w = synthetic.make_synthetic_weights(seed=1)
    img = synthetic.make_images(int(g['frames']), seed=int(g['seed']), size=int(g['size']))
    phi, moments, moving = nets_train_ref.encoder_resnet_train(img, w)
    assert nets_train_ref.BN_DECAY == BN_DECAY
    scale = np.abs(phi).max()
    assert np.abs(phi - g['phi']).max() / scale < 2e-5
    for i, s in enumerate(g['scopes']):
        m, v = moments[s]
        assert np.abs(m - g["mean_%d" % i]).max() <= 1e-4 * (1 + np.abs(m).max()), s
        assert np.abs(v - g["var_%d" % i]).max() <= 1e-4 * np.abs(v).max(), s
        for k in ('moving_mean', 'moving_variance'):
            want = g['%s_%d' % (k, i)]
            assert np.abs(moving[s + '/' + k] - want).max() <= 1e-6 * (1 + np.abs(want).max()), (s, k)
        assert not np.array_equal(g['moving_mean_%d' % i], w[s + '/moving_mean'])


@pytest.fixture
def fake_device(monkeypatch):
    from human_dynamics_b200 import nets

    class FakeLib(object):
        def __getattr__(self, name):
            return lambda *a, **k: 0
    monkeypatch.setattr(nets, 'lib', FakeLib())
    monkeypatch.setattr(nets, '_dev', lambda a, device, dtype=np.float32: torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)))
    monkeypatch.setattr(torch.Tensor, 'to', lambda self, *a, **k: self)
    e, z = torch.empty, torch.zeros
    monkeypatch.setattr(torch, 'empty', lambda *a, **k: e(*a, **{kk: v for kk, v in k.items() if kk != 'device'}))
    monkeypatch.setattr(torch, 'zeros', lambda *a, **k: z(*a, **{kk: v for kk, v in k.items() if kk != 'device'}))
    return nets


def test_train_plan_wiring(fake_device):
    """Every conv's prologue applies the batch statistics of the map it reads (ReLU on); conv1 / conv2 carry no epilogue vectors and
    write raw fp32; conv3 keeps its bias; 49 stats ops, in scope order, each over the map and row count it normalises."""
    nets = fake_device
    from human_dynamics_b200 import synthetic
    w = synthetic.make_resnet_weights(seed=1)
    packed = nets.PackedResNet(w, 'cpu', tc='auto')
    bn = nets.ResNetBatchNorm(w, 'cpu')
    n, size = 3, 64
    plan = nets.ResNetTrainPlan(packed, bn, n, size)
    stats = [o for o in plan.ops if isinstance(o, nets.BatchStatsOp)]
    convs = [o for o in plan.ops if getattr(o, 'd', None) is not None]
    assert len(stats) == 49 == len(bn.scopes) and stats == plan.stats
    assert len(convs) == 52
    assert plan.num_launches == 3 + 2 * 49 + 52 + 1
    by_map = {}
    for i, s in enumerate(stats):
        assert s.C == bn.sizes[i] and s.gamma.data_ptr() == bn.view(bn.gamma, i).data_ptr()
        assert s.scale.data_ptr() == bn.view(plan.scale, i).data_ptr() and s.mean.data_ptr() == bn.view(plan.mean, i).data_ptr()
        by_map.setdefault(s.x.data_ptr(), []).append((plan.ops.index(s), s))
    H = size // 4
    for u, unit in enumerate(packed.units):
        sc = 'shortcut' in unit
        ops = plan.ops[plan.ops.index(stats[3 * u]):]
        seq = ops[:6 + sc]
        kinds = ['S'] + ['C'] * sc + ['C', 'S', 'C', 'S', 'C']
        assert [('S' if isinstance(o, nets.BatchStatsOp) else 'C') for o in seq] == kinds, u
        Ho = (H - 1) // unit['stride'] + 1
        assert stats[3 * u].rows == n * H * H and stats[3 * u + 1].rows == n * H * H and stats[3 * u + 2].rows == n * Ho * Ho
        convs_u = [o for o in seq if not isinstance(o, nets.BatchStatsOp)]
        for c in convs_u:
            d = c.d
            st = [s for i, s in by_map[d.in_] if i < plan.ops.index(c)][-1]        # the latest statistics of the map this conv reads
            assert (d.pre_scale, d.pre_shift, d.pre_relu, d.pre_img_stride) == (st.scale.data_ptr(), st.shift.data_ptr(), 1, 0)
            assert st.rows == d.n_img * d.H * d.W and st.C == d.Cin
        c1, c2, c3 = convs_u[-3:]
        for c in (c1, c2):
            assert not c.d.post_scale and not c.d.post_shift and c.d.post_relu == 0
        assert c2.d.KH == 3 and (c2.d.pad_t, c2.d.stride) == (1, unit['stride'])
        assert c3.d.post_shift == unit['conv3'].post_shift.data_ptr() and not c3.d.post_scale and c3.d.res
        if sc:
            assert convs_u[0].d.post_shift == unit['shortcut'].post_shift.data_ptr()
        else:
            assert c3.d.res == c1.d.in_ and c3.d.res_stride == unit['stride']   # identity shortcut: the raw unit input
        H = Ho
    assert plan.tail[0].data_ptr() == stats[-1].scale.data_ptr() and stats[-1].x.data_ptr() == plan.final.data_ptr()
    assert stats[-1].rows == n * plan.final_hw
    # the inference packing is shared, not changed: conv1 / conv2 keep their folded epilogues for ResNetPlan
    assert packed.units[0]['conv1'].post_scale is not None and packed.units[0]['conv2'].post_relu


def test_train_plan_refuses_weights_without_batch_norm(fake_device):
    nets = fake_device
    from human_dynamics_b200 import _lib, synthetic
    w = synthetic.make_resnet_weights(seed=1)
    del w['resnet_v2_50/block2/unit_3/bottleneck_v2/conv2/BatchNorm/moving_variance']
    with pytest.raises(_lib.HDError, match='block2/unit_3/bottleneck_v2/conv2/BatchNorm/moving_variance'):
        nets.ResNetBatchNorm(w, 'cpu')


def test_train_config_flags():
    from human_dynamics_b200.objective import TrainConfig
    c = TrainConfig()
    assert c.precomputed_phi is True and c.freeze_phi is True


def test_bn_stats_argument_checks():
    """Every argument error returns HD_ERR_INVALID before any launch (no device is touched: the pointers are never read)."""
    import ctypes as C
    from human_dynamics_b200._lib import lib
    p = C.c_void_p(1 << 20)
    ws = lib.hd_bn_stats_workspace_bytes(1000, 64)
    assert ws > 0 and lib.hd_bn_stats_workspace_bytes(1, 64) == 0 and lib.hd_bn_stats_workspace_bytes(1000, 66) == 0

    def call(x=p, rows=1000, Cc=64, ld=64, g=p, b=p, sc=p, sh=p, mm=None, mv=None, decay=0.997, w=p, wsb=ws):
        return lib.hd_bn_batch_stats(x, rows, Cc, ld, g, b, 1e-5, sc, sh, None, None, mm, mv, decay, w, wsb, None)
    for kw in (dict(x=None), dict(g=None), dict(b=None), dict(sc=None), dict(sh=None), dict(w=None), dict(rows=1), dict(Cc=66),
               dict(Cc=0), dict(ld=32), dict(ld=66), dict(x=C.c_void_p((1 << 20) + 4)), dict(w=C.c_void_p((1 << 20) + 8)),
               dict(mm=p), dict(mv=p), dict(mm=p, mv=p, decay=1.5), dict(wsb=ws - 1)):
        assert call(**kw) == 1, kw
    assert lib.hd_bn_moving_update(None, p, 10, 64, 0.997, p, p, None) == 1
    assert lib.hd_bn_moving_update(p, p, 1, 64, 0.997, p, p, None) == 1
    assert lib.hd_bn_moving_update(p, p, 10, 64, -0.1, p, p, None) == 1
