"""Host-side wiring of the half-precision inference mode (impl 'tc1h', HD_IMPL_TC_1XF16) checked WITHOUT a GPU: device allocations and
library calls of the plans are stubbed, the descriptors they fill are real.  Every conv of a 'tc1h' plan reads and writes fp16 heads only
(no remainder pointer anywhere), its activation memory is the parity plan's minus the remainder buffers, and the training entries refuse
the mode.  The C-ABI's own refusals are checked against the real library (they return before any launch)."""
import ctypes as C

import numpy as np
import pytest
import torch


@pytest.fixture
def fake_device(monkeypatch):
    """nets with a stub library and device allocations on the CPU; `allocs` records every tensor torch.empty / zeros make."""
    from human_dynamics_b200 import nets

    class FakeLib(object):
        def __getattr__(self, name):
            return lambda *a, **k: 0
    monkeypatch.setattr(nets, 'lib', FakeLib())
    monkeypatch.setattr(nets, '_dev', lambda a, device, dtype=np.float32: torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)))
    monkeypatch.setattr(torch.Tensor, 'to', lambda self, *a, **k: self)
    e, z = torch.empty, torch.zeros
    allocs = []

    def rec(fn):
        def f(*a, **k):
            t = fn(*a, **{kk: v for kk, v in k.items() if kk != 'device'})
            allocs.append(t)
            return t
        return f
    monkeypatch.setattr(torch, 'empty', rec(e))
    monkeypatch.setattr(torch, 'zeros', rec(z))
    return nets, allocs


REMAINDERS = ('in_lo', 'out_lo', 'w_nk_lo', 'tmap_lo', 'tmap_lo_n64', 'tmap_out_lo')


def _conv_descs(ops):
    return [o.d for o in ops if getattr(o, 'd', None) is not None]


def _assert_heads_only(d):
    assert d.impl == 4, d.impl
    assert d.in_hi and d.w_nk_hi and d.tmap_hi
    for f in REMAINDERS:
        assert not getattr(d, f), f


def _nbytes(tensors):
    return sum(t.numel() * t.element_size() for t in {id(t): t for t in tensors}.values())


def _plan_allocs(allocs, build):
    n0 = len(allocs)
    plan = build()
    return plan, list(allocs[n0:])


def _resnet_remainders(plan):
    """The remainder halves of every fp16 pair a parity ResNet plan reads or writes (conv1 planes included)."""
    out = [plan.planes[1]] if plan.planes is not None else []
    for op in plan.ops:
        keep = getattr(op, 'keep', None)
        if not keep or len(keep) < 7:
            continue
        for pair in (keep[5], keep[6]):                 # inp_split, out_split
            if pair is not None:
                out.append(pair[1])
    return out


def test_resnet_plan_tc1h_is_heads_only(fake_device):
    nets, allocs = fake_device
    from human_dynamics_b200 import synthetic
    w = synthetic.make_resnet_weights(seed=1)
    packed = nets.PackedResNet(w, 'cpu', tc='tc1h')
    packed3 = nets.PackedResNet(w, 'cpu', tc='tc3h')
    fast, a1 = _plan_allocs(allocs, lambda: nets.ResNetPlan(packed, 2, 64, 'tc1h'))
    ref, a3 = _plan_allocs(allocs, lambda: nets.ResNetPlan(packed3, 2, 64, 'tc3h'))
    assert fast.split and fast.planes is not None and fast.planes[1] is None and fast.pool_split[2][1] is None
    _assert_heads_only(fast.conv1_op.d)
    assert fast.conv1_op.d.flags & 2                                           # HD_CONV_INPUT_PLANES
    convs, convs3 = _conv_descs(fast.ops), _conv_descs(ref.ops)
    assert len(convs) == len(convs3) == 52 and fast.num_launches == ref.num_launches
    for d, d3 in zip(convs, convs3):
        _assert_heads_only(d)
        assert d3.impl == 3 and d3.in_lo and d3.w_nk_lo
        # same layer geometry and epilogue as the parity plan, only the remainders are gone
        for f in ('n_img', 'H', 'W', 'Cin', 'Ho', 'Wo', 'KH', 'KW', 'stride', 'Cout', 'post_relu', 'post2_relu', 'out_subsample'):
            assert getattr(d, f) == getattr(d3, f), f
        for f in ('out', 'res', 'out_hi', 'tmap_out_hi', 'tmap_out'):
            assert bool(getattr(d, f)) == bool(getattr(d3, f)), f
    # activation memory: the parity plan's minus its remainder buffers, counted from shapes
    rem = _resnet_remainders(ref)
    assert len(rem) > 4 and all(t.dtype == torch.float16 for t in rem)
    assert _nbytes(a1) == _nbytes(a3) - _nbytes(rem)


def test_stage_plans_tc1h_rebind_heads_only(fake_device):
    """The engine's two trunk stages in 'tc1h': the stage boundary carries the head alone (set_output / set_input)."""
    nets, _ = fake_device
    from human_dynamics_b200 import synthetic
    packed = nets.PackedResNet(synthetic.make_resnet_weights(seed=1), 'cpu', tc='tc1h')
    nxt = packed.units[7]
    pa = nets.ResNetPlan(packed, 2, 64, 'tc1h', units=(0, 7), root=True, tail=False, next_pre=nxt['pre'],
                         next_has_shortcut='shortcut' in nxt)
    pb = nets.ResNetPlan(packed, 2, 64, 'tc1h', units=(7, 16), root=False, tail=True)
    mid = torch.empty((2, 4, 4, 512))
    hi = torch.empty((2, 4, 4, 512), dtype=torch.float16)
    pa.set_output(mid, (hi, None))
    pb.set_input(mid, (hi, None))
    assert _conv_descs(pa.ops)[-1].out_hi == hi.data_ptr()
    assert all(f != 'in_lo' for _, f, _ in pb.in_refs)
    for d in _conv_descs(pa.ops) + _conv_descs(pb.ops):
        _assert_heads_only(d)
    assert sum(1 for d in _conv_descs(pb.ops) if d.in_hi == hi.data_ptr()) == 2        # block 3's shortcut conv and conv1


def test_fmovie_and_ief_plans_tc1h(fake_device):
    nets, _ = fake_device
    from human_dynamics_b200 import synthetic
    w = synthetic.make_synthetic_weights(seed=1)
    B, T = 2, 20
    N = B * T
    sizes = {}
    for impl in ('tc1h', 'tc3h'):
        fm = nets.FMoviePlan(nets.PackedFMovie(w, 'cpu', 3, tc=impl), B, T, impl)
        ief = nets.IEFPlan(nets.PackedIEF(w, 'cpu', tc=impl), N, 3, None, impl)
        fm._bind(torch.zeros((B, T, 2048)))
        ief._bind(torch.zeros((N, 2048)), torch.zeros((N, 85)))
        convs = [s[1].d for s in fm.steps if s[0] == 'conv'] + [op[1].d for ops in [ief.main_ops] + list(ief.delta_ops.values())
                                                                for op in ops if op[0] == 'conv']
        assert [s[0] for s in fm.steps] == ['gns', 'conv'] * 6 and ief.fast and ief.num_launches == 33
        assert len(convs) == 6 + 3 * 4
        if impl == 'tc1h':
            assert fm.act[1] is None and ief.phi_split[1] is None and ief.h1_split[1] is None
            for d in convs:
                _assert_heads_only(d)
        else:
            assert all(d.impl == 3 and d.in_lo and d.w_nk_lo for d in convs)
        pairs = (fm.act, ief.phi_split, ief.h1_split)
        sizes[impl] = _nbytes([t for pair in pairs for t in pair if t is not None])
    assert sizes['tc1h'] * 2 == sizes['tc3h'] == 2 * 2 * (N * 2048 + N * 2048 + N * 1024)


def test_hallucinator_binds_impl4(fake_device):
    """fc2_res reads its fp32 input through the register-staged producer: under 'tc1h' it is impl 4 with the weight heads alone."""
    nets, _ = fake_device
    pc = nets.PackedConv(np.zeros((2048, 2048), np.float32), 'cpu', post_relu=True, tc='tc1h')
    x, out = torch.zeros((40, 2048)), torch.zeros((40, 2048))
    d = pc.bind(x, 40, 1, 1, out, impl='tc1h').d
    assert d.impl == 4 and d.in_ and not d.in_hi and d.w_nk_hi and d.tmap_hi
    for f in REMAINDERS:
        assert not getattr(d, f), f


def test_training_entries_refuse_tc1h(fake_device):
    nets, _ = fake_device
    from human_dynamics_b200 import _lib, synthetic
    from human_dynamics_b200.config import HMMRConfig
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from human_dynamics_b200.trainable import TemporalModel
    packed = nets.PackedResNet(synthetic.make_resnet_weights(seed=1), 'cpu', tc='auto')
    with pytest.raises(_lib.HDError, match='tc1h'):
        nets.ResNetTrainPlan(packed, None, 2, 64, impl='tc1h')
    with pytest.raises(_lib.HDError, match='tc1h'):
        TemporalModel({}, HMMRConfig(impl='tc1h'))
    with pytest.raises(_lib.HDError, match='tc1h'):
        HMMRTrainer(TrainConfig(impl='tc1h'), {}, None)


def test_impl4_abi_refusals():
    """hd_conv_gemm with impl 4 refuses any remainder pointer (before any launch); the pair writers refuse a remainder without a head."""
    from human_dynamics_b200 import _lib
    lib = _lib.lib
    assert _lib.IMPL_BY_NAME['tc1h'] == _lib.HD_IMPL_TC_1XF16 == 4 and lib.hd_version() >= 108
    fake = 1 << 20                                          # never dereferenced: the descriptor is refused first
    tm = (C.c_ubyte * 128)()

    def desc(**kw):
        d = _lib.ConvDesc()
        d.n_img, d.H, d.W, d.Cin, d.Ho, d.Wo, d.KH, d.KW, d.stride = 1, 8, 8, 64, 8, 8, 1, 1, 1
        d.in_ld, d.Cout, d.K_pad, d.out_ld, d.out2_ld = 64, 64, 64, 64, 64
        d.in_hi, d.out_hi, d.w_nk_hi, d.tmap_hi, d.impl = fake, fake, fake, C.cast(tm, C.c_void_p), 4
        for k, v in kw.items():
            setattr(d, k, v)
        return d
    for f in ('in_lo', 'out_lo', 'w_nk_lo'):
        d = desc(**{f: fake})
        assert lib.hd_conv_gemm(C.byref(d), None) == 1, f
        assert b'impl 4' in lib.hd_last_error()
    for f in ('tmap_lo', 'tmap_lo_n64'):
        d = desc(**{f: C.cast(tm, C.c_void_p)})
        assert lib.hd_conv_gemm(C.byref(d), None) == 1, f
    d = desc(in_hi=None)                                    # no input at all
    assert lib.hd_conv_gemm(C.byref(d), None) == 1
    v = C.c_void_p(fake)
    assert lib.hd_maxpool3x3s2_same(v, None, 1, 8, 8, 64, v, v, None, v, None) == 1
    assert lib.hd_ief_fc1_theta(v, v, 85, v, 85, 1024, None, v, v, 8, None) == 1
    assert lib.hd_process_image(v, 1, 8, 8, v, v, 8, None, v, 16, None) == 1
    assert lib.hd_pack_conv1_planes(v, None, v, 1, 8, 8, 16, None) == 1
    assert lib.hd_groupnorm_relu_split(v, v, v, None, v, 1, 20, 2048, 32, 1e-6, None) == 1
    assert lib.hd_split_f16(v, None, v, 16, None) == 1
