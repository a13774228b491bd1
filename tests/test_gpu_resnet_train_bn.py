"""GPU: the training-mode ResNet (batch statistics, precomputed_phi=False).  hd_bn_batch_stats / hd_bn_moving_update against float64
numpy, a padded strided 3x3 with a batch-norm prologue, ResNetTrainPlan against the float64 oracle (oracle/nets_train_ref.py) and the
reference's own training trunk (resnet_train_bn_v1.npz), HMMRTrainer from images, and the encoder_resnet(is_training=True) drop-in."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'resnet_train_bn_v1.npz')
DECAY = 0.997


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stats(x2d, rows, Cc, ld, gamma, beta, eps=1e-5, moving=None, decay=DECAY):
    """One hd_bn_batch_stats call -> (scale, shift, mean, var) device tensors (moving: (mean, var) stepped in place)."""
    from human_dynamics_b200._lib import lib, check
    dev = 'cuda'
    out = [torch.empty(Cc, device=dev) for _ in range(4)]
    wsb = lib.hd_bn_stats_workspace_bytes(rows, Cc)
    ws = torch.empty(max(16, wsb), dtype=torch.uint8, device=dev)
    mm, mv = moving if moving is not None else (None, None)
    check(lib.hd_bn_batch_stats(_vp(x2d), rows, Cc, ld, _vp(gamma), _vp(beta), eps, *[_vp(t) for t in out], _vp(mm), _vp(mv), decay,
                                _vp(ws), ws.numel(), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "hd_bn_batch_stats")
    return out


def _np_stats(x, gamma, beta, eps=1e-5):
    x = x.astype(np.float64)
    m, v = x.mean(0), x.var(0)
    sc = gamma.astype(np.float64) / np.sqrt(v + eps)
    return sc, beta - m * sc, m, v


@pytest.mark.parametrize('rows,Cc,ld,mean,std', [
    (1000, 64, 64, 0., 1.), (4097, 128, 128, 0.5, 2.), (12345, 256, 264, 0., 1.), (3001, 512, 512, -3., 0.5), (777, 1024, 1024, 0., 1.),
    (50001, 2048, 2048, 0.1, 1.), (8191, 64, 96, 1e3, 1.), (2, 2048, 2048, 0., 1.), (100003, 192, 192, 1e3, 1.), (3, 4, 8, 5., 1.)])
def test_stats_kernel_against_float64(rows, Cc, ld, mean, std):
    rng = np.random.RandomState(rows % 1000 + Cc)
    base = rng.normal(mean, std, size=(rows, ld)).astype(np.float32)
    base[:, :Cc] += rng.normal(0, std, size=Cc).astype(np.float32)             # per-channel offsets
    gamma = rng.uniform(0.5, 1.5, Cc).astype(np.float32)
    beta = rng.normal(0, 0.3, Cc).astype(np.float32)
    mm0 = rng.normal(0, 1, Cc).astype(np.float32)
    mv0 = rng.uniform(0.5, 2, Cc).astype(np.float32)
    x = torch.from_numpy(base).cuda()
    g, b = torch.from_numpy(gamma).cuda(), torch.from_numpy(beta).cuda()
    mm, mv = torch.from_numpy(mm0).cuda(), torch.from_numpy(mv0).cuda()
    sc, sh, m, v = _stats(x, rows, Cc, ld, g, b, moving=(mm, mv))
    rsc, rsh, rm, rv = _np_stats(base[:, :Cc], gamma, beta)
    tol = 1e-6
    assert np.abs(m.cpu().numpy() - rm).max() <= tol * (np.abs(rm).max() + std)
    assert np.abs(v.cpu().numpy() - rv).max() <= tol * rv.max()
    assert np.abs(sc.cpu().numpy() - rsc).max() <= tol * np.abs(rsc).max()
    assert np.abs(sh.cpu().numpy() - rsh).max() <= tol * (np.abs(rm * rsc).max() + 1)
    rmm = mm0 - (mm0 - rm) * (1 - DECAY)
    rmv = mv0 - (mv0 - rv * rows / (rows - 1)) * (1 - DECAY)
    assert np.abs(mm.cpu().numpy() - rmm).max() <= 1e-6 * (np.abs(rmm).max() + 1)
    assert np.abs(mv.cpu().numpy() - rmv).max() <= 1e-6 * (np.abs(rmv).max() + 1)
    # repeats are bit-identical; the separate moving-average step equals the one the stats call takes
    again = _stats(x, rows, Cc, ld, g, b)
    for a, c in zip((sc, sh, m, v), again):
        assert torch.equal(a, c)
    from human_dynamics_b200._lib import lib, check
    mm2, mv2 = torch.from_numpy(mm0).cuda(), torch.from_numpy(mv0).cuda()
    check(lib.hd_bn_moving_update(_vp(m), _vp(v), rows, Cc, DECAY, _vp(mm2), _vp(mv2), None), 'hd_bn_moving_update')
    assert torch.equal(mm2, mm) and torch.equal(mv2, mv)
    # a row permutation changes the chunking of the sums, not the result beyond rounding
    perm = torch.from_numpy(rng.permutation(rows)).cuda()
    psc, psh, pm, pv = _stats(x[perm].contiguous(), rows, Cc, ld, g, b)
    assert torch.allclose(pm, m, rtol=0, atol=1e-6 * (abs(mean) + std)) and torch.allclose(pv, v, rtol=1e-6, atol=0)


def test_stats_kernel_argument_errors():
    """Every argument error returns HD_ERR_INVALID and launches nothing."""
    from human_dynamics_b200._lib import lib
    x = torch.zeros((100, 64), device='cuda')
    v = [torch.ones(64, device='cuda') for _ in range(6)]
    wsb = lib.hd_bn_stats_workspace_bytes(100, 64)
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
    ok = dict(x=_vp(x), rows=100, Cc=64, ld=64, g=_vp(v[0]), b=_vp(v[1]), sc=_vp(v[2]), sh=_vp(v[3]), mm=None, mv=None, decay=DECAY,
              ws=_vp(ws), wsb=wsb)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.hd_bn_batch_stats(a['x'], a['rows'], a['Cc'], a['ld'], a['g'], a['b'], 1e-5, a['sc'], a['sh'], None, None, a['mm'],
                                     a['mv'], a['decay'], a['ws'], a['wsb'], None)
    lib.hd_launch_count_reset()
    bad = [dict(x=None), dict(g=None), dict(b=None), dict(sc=None), dict(sh=None), dict(ws=None), dict(rows=1), dict(Cc=62),
           dict(ld=60), dict(ld=66), dict(x=C.c_void_p(x.data_ptr() + 4)), dict(ws=C.c_void_p(ws.data_ptr() + 8)), dict(mm=_vp(v[4])),
           dict(mv=_vp(v[5])), dict(mm=_vp(v[4]), mv=_vp(v[5]), decay=1.5), dict(wsb=wsb - 1)]
    for kw in bad:
        assert call(**kw) == 1, kw
    assert lib.hd_bn_moving_update(None, _vp(v[0]), 100, 64, DECAY, _vp(v[4]), _vp(v[5]), None) == 1
    assert lib.hd_bn_moving_update(_vp(v[0]), _vp(v[1]), 1, 64, DECAY, _vp(v[4]), _vp(v[5]), None) == 1
    assert lib.hd_launch_count() == 0
    assert call() == 0 and lib.hd_launch_count() == 2


@pytest.mark.parametrize('H,stride', [(15, 2), (14, 2), (13, 1)])
def test_padded_strided_3x3_with_prologue(H, stride):
    """conv2 of a training-mode unit: relu(x * scale + shift) in the A producer of a padded (strided) 3x3, no epilogue vectors.  The
    padding must stay zero after the prologue (shift > 0 here, so an activated pad would show)."""
    from human_dynamics_b200.nets import PackedConv
    from oracle.nets_ref import conv2d_same
    rng = np.random.RandomState(H * 10 + stride)
    n, Cin, Cout = 3, 64, 64
    w = rng.normal(0, 0.05, size=(3, 3, Cin, Cout)).astype(np.float32)
    x = rng.normal(0, 1, size=(n, H, H, Cin)).astype(np.float32)
    sc = rng.uniform(0.5, 1.5, Cin).astype(np.float32)
    sh = rng.uniform(0.2, 1.0, Cin).astype(np.float32)
    conv = PackedConv(w, 'cuda', post_scale=np.ones(Cout, np.float32), post_shift=np.ones(Cout, np.float32), post_relu=True,
                      stride=stride, pad=(1, 1), tc='auto')
    Ho = (H - 1) // stride + 1
    xt = torch.from_numpy(x).cuda()
    out = torch.empty((n, Ho, Ho, Cout), device='cuda')
    op = conv.bind(xt, n, H, H, out, pre=(torch.from_numpy(sc).cuda(), torch.from_numpy(sh).cuda(), 0, 1), post=(None, None, False))
    assert op.d.impl == 3 and not op.d.post_scale and not op.d.post_shift
    op.run(C.c_void_p(torch.cuda.current_stream().cuda_stream))
    a = torch.relu(torch.from_numpy(x).double() * torch.from_numpy(sc).double() + torch.from_numpy(sh).double())
    ref = conv2d_same(a, torch.from_numpy(w).double(), stride).numpy()
    got = out.cpu().numpy()
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-5


@pytest.fixture(scope='module')
def golden_weights():
    from human_dynamics_b200 import synthetic
    return synthetic.make_synthetic_weights(seed=1)


def _trunk(w, n, size, images):
    from human_dynamics_b200.nets import PackedResNet, ResNetBatchNorm, ResNetTrainPlan
    packed = PackedResNet(w, 'cuda', tc='auto')
    bn = ResNetBatchNorm(w, 'cuda')
    plan = ResNetTrainPlan(packed, bn, n, size)
    phi = torch.empty((n, 2048), device='cuda')
    plan.run(images, phi)
    return plan, bn, phi


def _check_trunk(plan, bn, phi, ref, tol=1e-4):
    rphi, rmom, rmov = ref
    assert np.abs(phi.cpu().numpy() - rphi).max() / np.abs(rphi).max() < tol
    mom = plan.moments()
    for s in bn.scopes:
        m, v = (t.cpu().numpy() for t in mom[s])
        rm, rv = rmom[s]
        assert np.abs(m - rm).max() <= tol * (np.abs(rm).max() + np.sqrt(rv.max())), s
        assert np.abs(v - rv).max() <= tol * rv.max(), s
    plan.apply_moving_update()
    got = bn.moving()
    for k, want in rmov.items():
        assert np.abs(got[k] - want).max() <= 1e-6 * (np.abs(want).max() + 1), k


@pytest.mark.parametrize('n', [2, 5, 16, 160])
def test_trunk_against_oracle(golden_weights, n):
    from human_dynamics_b200 import synthetic
    from oracle import nets_train_ref
    img = synthetic.make_images(n, seed=90 + n, size=224)
    plan, bn, phi = _trunk(golden_weights, n, 224, torch.from_numpy(img).cuda())
    ref = nets_train_ref.encoder_resnet_train(img, golden_weights, device='cuda')
    _check_trunk(plan, bn, phi, ref)
    if n == 16:                                      # bit-identical repeats
        phi2 = torch.empty_like(phi)
        m0 = plan.mean.clone()
        plan.run(torch.from_numpy(img).cuda(), phi2)
        assert torch.equal(phi, phi2) and torch.equal(plan.mean, m0)


def test_trunk_against_reference_fixture(golden_weights):
    """The reference's encoder_resnet(is_training=True) + UPDATE_OPS over the TF stand-in (float32)."""
    from human_dynamics_b200 import synthetic
    g = np.load(GOLDEN)
    n, size = int(g['frames']), int(g['size'])
    img = synthetic.make_images(n, seed=int(g['seed']), size=size)
    plan, bn, phi = _trunk(golden_weights, n, size, torch.from_numpy(img).cuda())
    assert list(g['scopes']) == bn.scopes
    rmom = {s: (g['mean_%d' % i], g['var_%d' % i]) for i, s in enumerate(bn.scopes)}
    rmov = {}
    for i, s in enumerate(bn.scopes):
        rmov[s + '/moving_mean'], rmov[s + '/moving_variance'] = g['moving_mean_%d' % i], g['moving_variance_%d' % i]
    _check_trunk(plan, bn, phi, (g['phi'], rmom, rmov))


# ------------------------------------------------------------------------------------------------------------------------------------
# the trainer from images
# ------------------------------------------------------------------------------------------------------------------------------------
def _batch(B, T, S, seed, with_images=True):
    from human_dynamics_b200 import synthetic
    rng = np.random.RandomState(seed)
    b = {'labels': torch.from_numpy(np.concatenate([rng.uniform(-1, 1, (B, T, 25, 2)), np.ones((B, T, 25, 1))], -1).astype(np.float32)).cuda(),
         'poses': torch.from_numpy(rng.normal(0, 0.3, (B, T, 72)).astype(np.float32)).cuda(),
         'shape': torch.from_numpy(rng.normal(0, 0.5, (B, 10)).astype(np.float32)).cuda(),
         'gt3ds': torch.from_numpy(rng.normal(0, 0.3, (B, T, 14, 3)).astype(np.float32)).cuda(),
         'has_3d': torch.ones((B, 2), device='cuda')}
    if with_images:
        b['images'] = torch.from_numpy(synthetic.make_images(B * T, seed=seed, size=S).reshape(B, T, S, S, 3)).cuda()
    return b


def _mocap(n, seed):
    from human_dynamics_b200.smpl import batch_rodrigues
    aa = torch.from_numpy(np.random.RandomState(seed).normal(0, 0.3, size=(n * 24, 3)).astype(np.float32)).cuda()
    return batch_rodrigues(aa).reshape(n, 216)


def test_trainer_from_images(weights, smpl_model):
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.engine import HMMREngine, load_weights
    from human_dynamics_b200.nets import PackedResNet
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from oracle import nets_ref
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    B, T, S = 2, 6, 64
    batch = _batch(B, T, S, 5)
    tr = HMMRTrainer(TrainConfig(precomputed_phi=False), weights, smpl)
    phis, _ = tr.trunk(batch['images'])
    mocap = _mocap(tr.n_fake(B, T), 6)
    # image mode == phi mode fed the training-mode trunk's phis, bit for bit
    ref_tr = HMMRTrainer(TrainConfig(), weights, smpl)
    pb = {k: v for k, v in batch.items() if k != 'images'}
    pb['phis'] = phis.clone()
    w_conv = tr.trunk.packed.units[3]['conv2'].w_kn.clone()
    mm0, mv0 = tr.trunk.bn.moving_mean.clone(), tr.trunk.bn.moving_variance.clone()
    named, e_loss, _ = tr.forward(batch, mocap)
    assert torch.equal(tr.trunk.bn.moving_mean, mm0) and torch.equal(tr.trunk.bn.moving_variance, mv0)   # forward moves nothing
    a, b = tr.step(batch, mocap), ref_tr.step(pb, mocap)
    assert torch.equal(named['e_kp'].detach(), a['e_kp'])
    for k in b:
        assert torch.equal(a[k], b[k]), k
    # exactly one moving-average step per step, from this iteration's moments
    plan = tr.trunk.plan(B * T, S)
    mom = (1.0 - DECAY)
    for i, op in enumerate(plan.stats):
        v = tr.trunk.bn.view
        m_exp = v(mm0, i) - (v(mm0, i) - op.mean) * torch.tensor(mom, dtype=torch.float32)
        var_u = (op.var.double() * op.rows / (op.rows - 1)).float()
        v_exp = v(mv0, i) - (v(mv0, i) - var_u) * torch.tensor(mom, dtype=torch.float32)
        assert torch.equal(v(tr.trunk.bn.moving_mean, i), m_exp) and torch.equal(v(tr.trunk.bn.moving_variance, i), v_exp), i
    mm1 = tr.trunk.bn.moving_mean.clone()
    tr.step(batch, mocap)
    assert not torch.equal(tr.trunk.bn.moving_mean, mm1)
    # the ResNet itself is frozen
    assert torch.equal(tr.trunk.packed.units[3]['conv2'].w_kn, w_conv)
    tv = tr.tf_variables()
    for k, val in weights.items():
        if k.startswith('resnet_v2_50/') and 'moving_' not in k:
            assert np.array_equal(tv[k], val), k
    # the checkpoint carries the trained moving statistics: HMMREngine's inference trunk on it == the oracle's with those statistics
    moving = tr.trunk.bn.moving()
    with tempfile.TemporaryDirectory() as d:
        prefix = tr.save_checkpoint(os.path.join(d, 'model.ckpt-2'))
        w2 = load_weights(prefix)
    for k, val in moving.items():
        assert np.array_equal(w2[k], val) and not np.array_equal(val, weights[k]), k
    img = batch['images'].reshape(B * T, S, S, 3)
    eng = HMMREngine(w2, smpl_model)
    phi_inf = eng.encode_images(img).cpu().numpy()
    ref = nets_ref.encoder_resnet(img.cpu().numpy(), w2, torch.float64).numpy()
    assert np.abs(phi_inf - ref).max() / np.abs(ref).max() < 1e-4
    with pytest.raises(_lib.HDError, match='freeze_phi'):
        HMMRTrainer(TrainConfig(freeze_phi=False), weights, smpl)
    no_resnet = {k: v for k, v in weights.items() if k != 'resnet_v2_50/block3/unit_2/bottleneck_v2/conv3/weights'}
    with pytest.raises(_lib.HDError, match='block3/unit_2/bottleneck_v2/conv3/weights'):
        HMMRTrainer(TrainConfig(precomputed_phi=False), no_resnet, smpl)
    assert PackedResNet is not None


def test_trainer_end_to_end_from_uint8_frames(weights, smpl_model):
    """uint8 frames -> TubeAugmentor (seeded) -> HMMRTrainer(precomputed_phi=False).step: shapes, finite losses, repeatable."""
    from human_dynamics_b200.augment import TubeAugmentor
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    B, T, S = 2, 5, 64
    rng = np.random.RandomState(12)
    frames = rng.randint(0, 256, size=(B * T, 96, 120, 3)).astype(np.uint8)
    lab = np.stack([rng.uniform(0, 120, (B * T, 25)), rng.uniform(0, 96, (B * T, 25)), np.ones((B * T, 25))], 1).astype(np.float32)
    cen = np.stack([rng.randint(40, 80, B * T), rng.randint(30, 60, B * T)], 1).astype(np.int32)
    pose = rng.normal(0, 0.3, (B * T, 72)).astype(np.float32)
    g3 = rng.normal(0, 0.3, (B * T, 14, 3)).astype(np.float32)
    outs = []
    for _ in range(2):
        aug = TubeAugmentor(img_size=S, seed=7)
        r = aug(frames, lab, cen, pose, g3, tube_lengths=[T] * B)
        assert r['images'].shape == (B * T, S, S, 3)
        batch = {'images': r['images'].view(B, T, S, S, 3), 'labels': r['labels'].transpose(1, 2).reshape(B, T, 25, 3).contiguous(),
                 'poses': r['poses'].reshape(B, T, 72), 'shape': torch.zeros((B, 10), device='cuda'),
                 'gt3ds': r['gt3ds'].reshape(B, T, 14, 3), 'has_3d': torch.ones((B, 2), device='cuda')}
        tr = HMMRTrainer(TrainConfig(precomputed_phi=False), weights, smpl)
        out = tr.step(batch, _mocap(tr.n_fake(B, T), 3))
        assert all(v.shape == () and torch.isfinite(v) for v in out.values())
        outs.append((out, tr.trunk.bn.moving_variance.clone()))
    for k in outs[0][0]:
        assert torch.equal(outs[0][0][k], outs[1][0][k]), k
    assert torch.equal(outs[0][1], outs[1][1])


def test_encoder_resnet_drop_in_training_mode(weights, smpl_model):
    from human_dynamics_b200 import runtime as rt
    from human_dynamics_b200.engine import HMMREngine
    from human_dynamics_b200.nets import PackedResNet, ResNetBatchNorm, ResNetTrainPlan
    from human_dynamics_b200 import synthetic
    from src import models as M
    eng = HMMREngine(weights, smpl_model)
    rt.set_default_engine(eng)
    n, S = 6, 64
    x = torch.from_numpy(synthetic.make_images(n, seed=4, size=S)).cuda()
    phi, scope = M.encoder_resnet(x, is_training=True)
    assert scope == 'resnet_v2_50' and phi.shape == (n, 2048)
    bn = ResNetBatchNorm(weights, 'cuda')
    plan = ResNetTrainPlan(PackedResNet(weights, 'cuda', tc='auto'), bn, n, S)
    ref = torch.empty((n, 2048), device='cuda')
    plan.run(x, ref)
    assert torch.equal(phi, ref)
    phi2, _ = M.encoder_resnet(x, is_training=True)
    assert torch.equal(phi2, phi)
    assert torch.equal(eng._train_trunk.bn.moving_mean, bn.moving_mean)          # untouched: no update ops run
    inf, _ = M.encoder_resnet(x, is_training=False)
    assert not torch.equal(inf, phi)
