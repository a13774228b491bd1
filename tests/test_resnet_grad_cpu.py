"""The trunk's backward without a GPU: the float64 autograd oracle (oracle/nets_train_grad_ref.py) against nets_train_ref and against
central finite differences for every kind of trainable variable, the argument checks of the new entry points, and the trainer's
freeze_phi wiring."""
import ctypes as C

import numpy as np
import pytest
import torch

from human_dynamics_b200 import synthetic
from oracle import nets_train_grad_ref as G
from oracle import nets_train_ref

BLOCKS = ((4, 2, 2), (8, 1, 1))          # a conv shortcut, a strided identity unit, a stride-1 identity unit, at a few dozen pixels


def test_oracle_matches_the_training_forward():
    w = synthetic.make_resnet_weights(seed=1, blocks=BLOCKS)
    x = synthetic.make_images(3, seed=0, size=16)
    ref = nets_train_ref.encoder_resnet_train(x, w, blocks=BLOCKS)[0]
    phi = G.encoder_resnet_train(torch.as_tensor(x, dtype=torch.float64), G.leaves(w, BLOCKS), BLOCKS).detach().numpy()
    assert np.abs(phi - ref).max() <= 1e-12 * np.abs(ref).max()
    wf = synthetic.make_resnet_weights(seed=1)
    xf = synthetic.make_images(2, seed=1, size=64)
    ref = nets_train_ref.encoder_resnet_train(xf, wf)[0]
    phi = G.encoder_resnet_train(torch.as_tensor(xf, dtype=torch.float64), G.leaves(wf)).detach().numpy()
    assert np.abs(phi - ref).max() <= 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize('name', [
    'resnet_v2_50/conv1/weights',                                              # 7x7 stride 2, through the max pool
    'resnet_v2_50/block1/unit_1/bottleneck_v2/shortcut/weights',               # 1x1 conv shortcut
    'resnet_v2_50/block1/unit_1/bottleneck_v2/conv2/weights',                  # SAME 3x3
    'resnet_v2_50/block1/unit_2/bottleneck_v2/conv2/weights',                  # conv2d_same 3x3 stride 2 (strided identity unit)
    'resnet_v2_50/block1/unit_2/bottleneck_v2/conv3/weights',
    'resnet_v2_50/block1/unit_2/bottleneck_v2/preact/gamma',                   # batch norm in front of the subsampled shortcut
    'resnet_v2_50/block2/unit_1/bottleneck_v2/conv1/BatchNorm/beta',
    'resnet_v2_50/postnorm/gamma', 'resnet_v2_50/postnorm/beta',
    'resnet_v2_50/block2/unit_1/bottleneck_v2/conv3/biases', 'resnet_v2_50/conv1/biases'])
def test_oracle_against_finite_differences(name):
    w = synthetic.make_resnet_weights(seed=3, blocks=BLOCKS)
    x = synthetic.make_images(2, seed=4, size=16)
    dphi = np.random.RandomState(5).normal(0, 1, (2, 32))
    g, _ = G.trunk_gradients(x, w, dphi, BLOCKS)
    xt = torch.as_tensor(x, dtype=torch.float64)
    L = G.leaves(w, BLOCKS)
    rng = np.random.RandomState(6)
    flat = L[name].detach().reshape(-1)
    h = 1e-5
    for i in rng.choice(flat.numel(), min(6, flat.numel()), replace=False):
        vals = []
        for sgn in (1, -1):
            Lp = {k: v.detach().clone() for k, v in L.items()}
            Lp[name].view(-1)[i] += sgn * h
            vals.append(float((G.encoder_resnet_train(xt, Lp, BLOCKS) * torch.as_tensor(dphi)).sum()))
        fd = (vals[0] - vals[1]) / (2 * h)
        an = float(g[name].reshape(-1)[i])
        scale = float(g[name].abs().max()) + (float(g[name[:-len('biases')] + 'weights'].abs().max()) if name.endswith('biases') else 0.)
        assert abs(fd - an) <= 1e-6 * scale + 1e-9, (name, i, fd, an)


def test_max_pool_gradient_goes_to_the_first_maximum():
    x = torch.zeros((1, 4, 4, 1), dtype=torch.float64, requires_grad=True)      # all ties
    y = G.max_pool_3x3_s2(x)
    g, = torch.autograd.grad(y.sum(), x)
    # windows start at rows / columns 0 and 2 (SAME: pad 0 before, 1 after): each sends its gradient to its top-left cell
    want = np.zeros((4, 4))
    want[0, 0] = want[0, 2] = want[2, 0] = want[2, 2] = 1
    assert np.array_equal(g[0, :, :, 0].numpy(), want)


def test_argument_checks():
    """Every argument error returns HD_ERR_INVALID before any launch (the pointers are never read)."""
    from human_dynamics_b200._lib import lib
    p = C.c_void_p(1 << 20)
    ws = lib.hd_conv_wgrad_workspace_bytes(1000, 64, 64, 1)
    assert ws == 1 * 65 * 64 * 4 and lib.hd_conv_wgrad_workspace_bytes(0, 64, 64, 0) == 0

    def wg(x=p, n=1, H=10, Cin=64, Ho=10, K=1, s=1, pad=0, pre=(None, None), dy=p, Cout=64, dw=p, db=None, w=p, wsb=ws, x_ld=64):
        return lib.hd_conv_wgrad(x, x_ld, n, H, H, Cin, Ho, Ho, K, K, s, pad, pad, pre[0], pre[1], dy, Cout, Cout, dw, db, w, wsb, None)
    for kw in (dict(x=None), dict(dy=None), dict(dw=None), dict(w=None), dict(n=0), dict(Cin=0), dict(Cout=0), dict(K=0), dict(s=0),
               dict(pad=-1), dict(x_ld=32), dict(pre=(p, None)), dict(Ho=12), dict(wsb=0), dict(db=p, wsb=ws - 1)):
        assert wg(**kw) == 1, kw
    wb = lib.hd_bn_relu_backward_workspace_bytes(1000, 64)
    assert wb > 0 and lib.hd_bn_relu_backward_workspace_bytes(1, 64) == 0 and lib.hd_bn_relu_backward_workspace_bytes(1000, 66) == 0
    q = C.c_void_p((1 << 20) + 4096)

    def bb(x=p, dz=p, group=1, rows=1000, Cc=64, addend=None, aH=0, aW=0, s=0, dx=q, w=p, wsb=wb):
        return lib.hd_bn_relu_backward(x, dz, group, rows, Cc, p, p, p, p, 1e-5, addend, aH, aW, s, dx, p, p, w, wsb, None)
    for kw in (dict(x=None), dict(dz=None), dict(dx=None), dict(w=None), dict(rows=1), dict(Cc=66), dict(group=0), dict(group=3),
               dict(x=C.c_void_p((1 << 20) + 4)), dict(dx=p), dict(s=2), dict(s=2, addend=q, aH=7, aW=7), dict(wsb=wb - 1)):
        assert bb(**kw) == 1, kw
    assert lib.hd_maxpool3x3s2_same_backward(p, q, p, 1, 8, 8, 64, None) == 1                     # din aliases in
    assert lib.hd_maxpool3x3s2_same_backward(p, q, None, 1, 8, 8, 64, None) == 1
    assert lib.hd_zero_insert(p, p, 1, 4, 4, 64, 2, 8, 8, None) == 1
    assert lib.hd_zero_insert(p, q, 1, 4, 4, 64, 0, 8, 8, None) == 1
    assert lib.hd_version() >= 107


def test_trainer_wiring():
    """freeze_phi=False needs image input; the trunk's names are the reference's trainable resnet_v2_50 variables."""
    from human_dynamics_b200.trunk import conv_names
    names = G.trunk_names()
    convs = conv_names()
    assert len([n for n in convs if n.endswith('/weights')]) == 53 and len([n for n in convs if n.endswith('/biases')]) == 21
    assert names[:len(convs)] == convs and len(names) == 53 + 21 + 2 * 49
    w = synthetic.make_resnet_weights(seed=1)
    assert all(n in w for n in names)
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    with pytest.raises(HDError, match='freeze_phi=False'):
        HMMRTrainer(TrainConfig(freeze_phi=False), w, None)               # precomputed phis: no trunk to train


@pytest.fixture
def stub_device(monkeypatch):
    """No GPU: library calls return 0 without running, so the host-side wiring runs on 'cpu' tensors."""
    from human_dynamics_b200 import nets

    class FakeLib(object):
        def __getattr__(self, name):
            return lambda *a, **k: 0
    monkeypatch.setattr(nets, 'lib', FakeLib())
    return nets


def test_trunk_and_trainer_wiring_on_a_stub_device(stub_device, monkeypatch, tmp_path):
    """The trunk's 172 parameters join e_params; gamma / beta share storage with what the plans read; conv weights are read in place
    by their packs; tf_variables / save_checkpoint carry the current values; the keep-mode plan's backward descriptors read and write
    the buffers the walk expects (strided conv2 over the zero-inserted map, the shortcut's data gradient added in conv1's epilogue)."""
    from torch import nn
    from human_dynamics_b200 import adversarial, trainable
    from human_dynamics_b200.engine import load_weights
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    w = synthetic.make_resnet_weights(seed=1)

    class StubModel(nn.Module):
        def __init__(self, weights, config=None, device=None):
            super().__init__()
            self._source, self.device = weights, torch.device('cpu')
            self.p = nn.Parameter(torch.zeros(3))

        def tf_variables(self):
            return {'stub/p': self.p.detach().numpy().copy()}

    class StubDisc(StubModel):
        def __init__(self, *a, **k):
            super().__init__(None)

        def tf_variables(self):
            return {'stub/d': np.zeros(2, np.float32)}
    monkeypatch.setattr(trainable, 'TemporalModel', StubModel)
    monkeypatch.setattr(adversarial, 'PoseDiscriminator', StubDisc)

    class Smpl(object):
        consts = None
    tr = HMMRTrainer(TrainConfig(precomputed_phi=False, freeze_phi=False), w, Smpl())
    net = tr.trunk.net
    assert len(tr.e_params) == 1 + 53 + 21 + 2 * 49 and all(any(p is q for q in tr.e_params) for p in net.parameters())
    bn = net.bn
    for i, s in enumerate(bn.scopes):
        assert net.param(s + '/gamma').data_ptr() == bn.view(bn.gamma, i).data_ptr()
        assert net.param(s + '/beta').data_ptr() == bn.view(bn.beta, i).data_ptr()
    q = 'resnet_v2_50/block2/unit_1/bottleneck_v2'
    unit = net.packed.units[3]
    assert unit['conv2'].w_kn.data_ptr() == net.param(q + '/conv2/weights').data_ptr()
    assert unit['conv3'].post_shift.data_ptr() == net.param(q + '/conv3/biases').data_ptr()
    assert unit['conv2'].bwd.src.data_ptr() == net.param(q + '/conv2/weights').data_ptr()
    with torch.no_grad():
        net.param(q + '/conv2/weights').add_(1.0)
        net.param(q + '/preact/gamma').mul_(2.0)
    tv = tr.tf_variables()
    assert np.array_equal(tv[q + '/conv2/weights'], w[q + '/conv2/weights'] + 1.0)
    assert np.array_equal(tv[q + '/preact/gamma'], np.float32(w[q + '/preact/gamma']) * 2)
    assert all(n in tv for n in net.names) and 'stub/p' in tv and 'stub/d' in tv
    assert np.array_equal(tv[q + '/preact/moving_mean'], np.float32(w[q + '/preact/moving_mean']))
    w2 = load_weights(tr.save_checkpoint(str(tmp_path / 'model.ckpt-1')))
    assert np.array_equal(w2[q + '/conv2/weights'], tv[q + '/conv2/weights'])
    # the keep-mode plan and its backward descriptors
    n = 2
    plan = net.plan(n, 64)
    assert plan.keep and plan.num_backward_launches == 3 + 1 + 2 + 16 * 18 + 4 * 3 + 3
    S = plan._backward_state()
    U = len(net.packed.units)
    for ui, (unit, u) in enumerate(zip(net.packed.units, S['units'])):
        k = U - 1 - ui
        assert u['gy'] is S['G'][k % 2] and u['gx'] is S['G'][(k + 1) % 2]
        assert u['conv3'].d.in_ == u['gy'].data_ptr() and u['conv3'].d.out == S['D1'].data_ptr()
        assert u['conv2'].d.in_ == (S['Z'] if unit['stride'] > 1 else S['D2']).data_ptr() and u['conv2'].d.KH == 3
        assert u['conv1'].d.in_ == S['D2'].data_ptr() and u['conv1'].d.out == S['P'].data_ptr()
        assert u['conv1'].d.impl == u['conv3'].d.impl == 1                                   # 3xTF32
        if 'shortcut' in unit:
            assert u['shortcut'].d.in_ == u['gy'].data_ptr() and u['conv1'].d.res == S['P'].data_ptr()
        else:
            assert not u['conv1'].d.res
    assert plan.stats[-1].x is plan.final and plan.root_buf is plan.root_out
