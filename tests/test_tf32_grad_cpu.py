"""The TF32 gradient mode (grad_precision='tf32') checked WITHOUT a GPU: argument checks, the host emulation of the kernels' TF32 rounding
against hand-worked bit patterns, and the mode's reach on a stubbed library -- every backward hd_conv_gemm of the trunk, the temporal
model and D_pose runs 1xTF32 on heads alone and every trunk weight gradient is hd_conv_wgrad_ex(impl 2), while 'fp32' keeps the
3xTF32 descriptors and calls."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from tf32_emulation import rn_tf32


# ------------------------------------------------------------------------------------------------------------------------------------
# argument checks
# ------------------------------------------------------------------------------------------------------------------------------------
BAD = ['bf16', 'fp16', 'TF32', 'tf32 ', '', None, 1]


@pytest.mark.parametrize('bad', BAD)
def test_bad_grad_precision_is_refused(bad):
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200.adversarial import PoseDiscriminator
    from human_dynamics_b200.objective import TrainConfig
    from human_dynamics_b200.trunk import TrainableResNet
    with pytest.raises(HDError, match='grad_precision'):
        TrainConfig(grad_precision=bad)
    with pytest.raises(HDError, match='grad_precision'):
        TrainableResNet({}, grad_precision=bad)
    with pytest.raises(HDError, match='grad_precision'):
        PoseDiscriminator(grad_precision=bad)


def test_modes_and_tc1h_still_refused():
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200.nets import GRAD_PRECISIONS, grad_one_pass
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    assert GRAD_PRECISIONS == ('fp32', 'tf32') and TrainConfig().grad_precision == 'fp32'
    assert grad_one_pass('tf32', 'x') and not grad_one_pass('fp32', 'x')
    for gp in GRAD_PRECISIONS:
        with pytest.raises(HDError, match='tc1h'):
            HMMRTrainer(TrainConfig(impl='tc1h', grad_precision=gp), synthetic.make_resnet_weights(seed=1), None)


def test_wgrad_ex_refuses_a_bad_impl_before_any_launch():
    """Checked against the real library: the impl is refused before anything reaches the device."""
    from human_dynamics_b200._lib import lib, HD_IMPL_TC_1XF16, HD_IMPL_TC_3XF16, HD_IMPL_SIMT
    p = C.c_void_p(16)
    ws = lib.hd_conv_wgrad_workspace_bytes(100, 64, 64, 0)
    for impl in (HD_IMPL_SIMT, HD_IMPL_TC_3XF16, HD_IMPL_TC_1XF16, -1, 5):
        rc = lib.hd_conv_wgrad_ex(p, 64, 1, 10, 10, 64, 10, 10, 1, 1, 1, 0, 0, None, None, p, 64, 64, p, None, p, ws, impl, None)
        assert rc == 1, impl                                    # HD_ERR_INVALID
    assert 'impl' in lib.hd_last_error().decode()
    # the head-only TF32 transpose is mode 1 alone: mode 2 (fp16) still needs its remainder
    assert lib.hd_transpose_split(p, 32, 32, 32, 2, p, None, 32, 64, 32, None) == 1


# ------------------------------------------------------------------------------------------------------------------------------------
# the host emulation of rn_tf32
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bits,want', [
    (0x3F800000, 0x3F800000),           # 1.0: already TF32
    (0x3F800FFF, 0x3F800000),           # below half an ulp: down
    (0x3F801000, 0x3F802000),           # exactly half, retained lsb 0: away from zero (round-half-even would keep 0x3F800000)
    (0x3F803000, 0x3F804000),           # exactly half, retained lsb 1: up
    (0x3F805000, 0x3F806000),           # exactly half, retained lsb 0: away (even would give 0x3F804000)
    (0x3F801001, 0x3F802000),           # above half: up
    (0x3FFFF000, 0x40000000),           # the carry reaches the exponent: 2.0
    (0xBF801000, 0xBF802000),           # negative tie: away from zero in magnitude, -(1 + 2^-10)
    (0xBF800FFF, 0xBF800000),           # negative, below half: toward zero
    (0xC2C81FFF, 0xC2C82000),           # -100.0625 - a hair: up in magnitude
    (0x00000000, 0x00000000), (0x80000000, 0x80000000),     # +0, -0
    (0x00001000, 0x00002000),           # a subnormal tie
    (0x7F7FFFFF, 0x7F800000)])          # FLT_MAX's last ulp rounds to +inf, as the kernels do
def test_rn_tf32_bit_patterns(bits, want):
    a = np.array([bits], np.uint32).view(np.float32)
    got = rn_tf32(a).view(np.uint32)[0]
    assert got == want, (hex(bits), hex(int(got)), hex(want))


def test_rn_tf32_is_the_nearest_tf32_value():
    rng = np.random.RandomState(0)
    x = (rng.normal(0, 1, 20000) * 10.0 ** rng.uniform(-6, 6, 20000)).astype(np.float32)
    h = rn_tf32(x)
    assert np.all(h.view(np.uint32) & 0x1FFF == 0)
    ulp = np.abs(np.spacing(h)) * 8192                           # TF32 spacing at h
    assert np.all(np.abs(h.astype(np.float64) - x) <= ulp / 2 * (1 + 1e-12))
    assert np.array_equal(rn_tf32(-x), -h)                       # symmetric: ties go away from zero on both sides


# ------------------------------------------------------------------------------------------------------------------------------------
# the mode reaches every backward descriptor (stubbed library)
# ------------------------------------------------------------------------------------------------------------------------------------
class RecLib(object):
    """Library stub: every call returns 0 without running and is recorded as (name, args)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*a):
            self.calls.append((name, a))
            return 0
        return f

    def gemm_descs(self):
        return [a[0]._obj for n, a in self.calls if n == 'hd_conv_gemm']

    def named(self, name):
        return [a for n, a in self.calls if n == name]


@pytest.fixture
def rec_device(monkeypatch):
    """nets / trainable / adversarial with one recording library stub, a null stream and host pointers: host-side wiring on 'cpu'
    tensors."""
    from human_dynamics_b200 import adversarial, nets, trainable
    rec = RecLib()
    for m in (nets, trainable, adversarial):
        monkeypatch.setattr(m, 'lib', rec)
        monkeypatch.setattr(m, 'current_stream', lambda: None)
        monkeypatch.setattr(m, 'fptr', lambda t: C.c_void_p(t.data_ptr()) if t is not None else None)
    return rec


def _check_descs(descs, one_pass):
    assert descs
    for d in descs:
        assert d.w_nk_hi and d.tmap_hi and d.in_ and d.out
        assert not d.in_hi and not d.in_lo and not d.out_hi and not d.out_lo and not d.tmap_lo_n64
        if one_pass:
            assert d.impl == 2 and not d.w_nk_lo and not d.tmap_lo, (d.impl, d.w_nk_lo, d.tmap_lo)
        else:
            assert d.impl == 1 and d.w_nk_lo and d.tmap_lo


@pytest.mark.parametrize('gp', ['fp32', 'tf32'])
def test_trunk_backward_descriptors(rec_device, monkeypatch, gp):
    from torch import nn
    from human_dynamics_b200 import adversarial, synthetic, trainable
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    rec = rec_device
    w = synthetic.make_resnet_weights(seed=1)

    class StubModel(nn.Module):
        def __init__(self, weights, config=None, device=None):
            super().__init__()
            self._source, self.device = weights, torch.device('cpu')
            self.p = nn.Parameter(torch.zeros(3))

    seen = {}

    class StubDisc(StubModel):
        def __init__(self, *a, **k):
            super().__init__(None)
            seen.update(k)
    monkeypatch.setattr(trainable, 'TemporalModel', StubModel)
    monkeypatch.setattr(adversarial, 'PoseDiscriminator', StubDisc)

    class Smpl(object):
        consts = None
    tr = HMMRTrainer(TrainConfig(precomputed_phi=False, freeze_phi=False, grad_precision=gp), w, Smpl())
    assert seen['grad_precision'] == gp
    net = tr.trunk.net
    assert net.grad_precision == gp
    n = 2
    plan = net.plan(n, 64)
    assert plan.one_pass == (gp == 'tf32') and plan.grad_precision == gp
    rec.calls.clear()
    grads = plan.backward(torch.zeros((n, 2048)), torch.zeros((n, 64, 64, 3)), stream=None)
    descs = rec.gemm_descs()
    units = net.packed.units
    assert len(descs) == sum(4 if 'shortcut' in u else 3 for u in units)
    _check_descs(descs, gp == 'tf32')
    if gp == 'fp32':                                             # each descriptor reads its own pack's remainder and map
        S = plan._backward_state()
        for unit, u in zip(units, S['units']):
            for c in u:
                if c in ('conv1', 'conv2', 'conv3', 'shortcut'):
                    bwd = unit[c].bwd
                    assert u[c].d.w_nk_lo == bwd.w_nk_lo.data_ptr() and u[c].d.tmap_lo == C.cast(bwd.tmap_lo, C.c_void_p).value
    assert len(rec.named('hd_zero_insert')) == sum(1 for u in units if u['stride'] > 1)
    ex, old = rec.named('hd_conv_wgrad_ex'), rec.named('hd_conv_wgrad')
    weights = [k for k in grads if k.endswith('/weights')]
    assert len(weights) == 53
    if gp == 'tf32':
        assert not old and len(ex) == 53 and all(a[-2] == 2 for a in ex)
    else:
        assert not ex and len(old) == 53


def _pack(shape, KH, Cin, Cout):
    from human_dynamics_b200.trainable import BackwardDataPack
    return BackwardDataPack(torch.zeros(shape), KH, Cin, Cout)


@pytest.mark.parametrize('gp', ['fp32', 'tf32'])
def test_temporal_and_dpose_backward_descriptors_from_layer_packs(rec_device, gp):
    """f_movie, an IEF head, fc2_res and D_pose: every backward GEMM (data gradients and weight gradients) in the model's mode, and the
    weight gradients' B operand written as a TF32 head alone (hd_transpose_split mode 1, lo NULL) under 'tf32'."""
    from human_dynamics_b200 import adversarial, trainable
    from human_dynamics_b200.synthetic import make_dpose_weights
    rec = rec_device
    one = gp == 'tf32'
    B, T, Cc, N = 2, 4, 64, 8

    def transposes():
        return [a for a in rec.named('hd_transpose_split') if a[4] == 1]

    def check(expect_gemms):
        descs = rec.gemm_descs()
        assert len(descs) == expect_gemms
        _check_descs(descs, one)
        tr = transposes()
        assert tr and all((a[6] is None) == one for a in tr)
        rec.calls.clear()
    # f_movie (3 blocks of two 3x1 convs): per conv one weight gradient and one data gradient
    z = lambda *s: torch.zeros(s)                                # noqa: E731
    layer = lambda bwd: types.SimpleNamespace(bwd=bwd)           # noqa: E731
    blocks = [{'gn1': (z(Cc), z(Cc)), 'gn2': (z(Cc), z(Cc)), 'conv1': layer(_pack((3, 1, Cc, Cc), 3, Cc, Cc)),
               'conv2': layer(_pack((3, 1, Cc, Cc), 3, Cc, Cc))} for _ in range(3)]
    model = types.SimpleNamespace(one_pass=one, fmovie=types.SimpleNamespace(blocks=blocks))
    rec.calls.clear()
    trainable.fmovie_backward(model, [(z(B, T, Cc), z(B, T, Cc))] * 3, z(B, T, Cc))
    check(3 * 2 * 2)
    # one IEF head: fc2's and fc1's data gradients, four weight-gradient GEMMs
    feat, d = 64, 85
    head = types.SimpleNamespace(d=d, feat=feat, fc1_phi=layer(_pack((feat, 1024), 1, feat, 1024)),
                                 fc1_theta=layer(types.SimpleNamespace(dst=z(1024, d))), fc2=layer(_pack((1024, 1024), 1, 1024, 1024)),
                                 fc3=layer(types.SimpleNamespace(dst=z(d, 1024))))
    model = types.SimpleNamespace(one_pass=one, _zeros=z(96))
    trainable.ief_head_backward(model, head, z(N, feat), N, (z(3, N, 1024), z(3, N, 1024), z(N, d), d, z(N, d), z(N, d)), z(N, d), d,
                                None, None)
    check(3 + 1 + 4)
    # fc2_res: three weight gradients, three data gradients
    model = types.SimpleNamespace(one_pass=one, hal=types.SimpleNamespace(**{'fc%d' % i: layer(_pack((2048, 2048), 1, 2048, 2048))
                                                                            for i in (1, 2, 3)}))
    trainable.hal_backward(model, z(N, 2048), z(N, 2048), z(N, 2048), z(N, 2048))
    check(6)
    # D_pose: fc2's and fc1's data gradients and weight gradients
    w = make_dpose_weights(0)
    P = []
    for name in adversarial.PARAM_NAMES:
        if 'pose_out_j/' in name:
            P.append(z(23, 32) if name.endswith('weights') else z(23))
        else:
            P.append(torch.from_numpy(np.asarray(w[name], np.float32)))
    disc = types.SimpleNamespace(one_pass=one, _p=P, fc1_bwd=_pack((736, 1024), 1, 736, 1024), fc2_bwd=_pack((1024, 1024), 1, 1024, 1024))
    adversarial.dpose_backward(disc, z(N, 23, 9), (z(N, 736), z(N, 736), z(N, 1024), z(N, 1024)), z(N, 24), True, True)
    check(4)
