"""Which conv pairs the ResNet plans run as one hd_conv_gemm_chain launch, checked WITHOUT a GPU: device allocations and launches are
stubbed, the descriptors the plans fill are real, and the eligibility rule is the library's own (hd_conv_gemm_chain_supported looks
at shapes and pointers only).  Stage A (blocks 1-2) chains block 1's two identity transitions; stage B (blocks 3-4) chains none.  The
library refuses pairs outside the rule with HD_ERR_UNSUPPORTED before any launch."""
import numpy as np
import pytest
import torch

HD_ERR_UNSUPPORTED = 4


@pytest.fixture
def chain_device(monkeypatch):
    from human_dynamics_b200 import nets, _lib

    class FakeLib(object):
        def __getattr__(self, name):
            if name == 'hd_conv_gemm_chain_supported':
                return _lib.lib.hd_conv_gemm_chain_supported
            return lambda *a, **k: 0
    monkeypatch.setattr(nets, 'lib', FakeLib())
    monkeypatch.setattr(nets, '_dev', lambda a, device, dtype=np.float32: torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)))
    monkeypatch.setattr(torch.Tensor, 'to', lambda self, *a, **k: self)
    e, z = torch.empty, torch.zeros
    monkeypatch.setattr(torch, 'empty', lambda *a, **k: e(*a, **{kk: v for kk, v in k.items() if kk != 'device'}))
    monkeypatch.setattr(torch, 'zeros', lambda *a, **k: z(*a, **{kk: v for kk, v in k.items() if kk != 'device'}))
    return nets


def _stages(nets, packed, impl):
    nxt = packed.units[7]
    pa = nets.ResNetPlan(packed, 2, 64, impl, units=(0, 7), root=True, tail=False, next_pre=nxt['pre'], next_has_shortcut='shortcut' in nxt)
    pb = nets.ResNetPlan(packed, 2, 64, impl, units=(7, 16), root=False, tail=True)
    return pa, pb


@pytest.mark.parametrize('impl', ['auto', 'tc1h'])
def test_stage_a_chains_block_1_transitions_and_stage_b_none(chain_device, impl):
    nets = chain_device
    from human_dynamics_b200 import synthetic
    packed = nets.PackedResNet(synthetic.make_resnet_weights(seed=1), 'cpu', tc=impl)
    pa, pb = _stages(nets, packed, impl)
    chains = [o for o in pa.ops if isinstance(o, nets.ChainOp)]
    assert not any(isinstance(o, nets.ChainOp) for o in pb.ops)
    # unit 1 -> 2 (the shortcut's output as residual, full fp32 output), unit 2 -> 3 (identity residual, x[:, ::2, ::2] alone)
    assert [(c.d.Cin, c.d.Cout, c.second.d.Cout, c.d.out_subsample) for c in chains] == [(64, 256, 64, 0), (64, 256, 64, 2)]
    assert chains[0].d.res == pa.bufS.data_ptr() and chains[1].d.out == pa.bufS.data_ptr()
    for c in chains:
        assert c.d.out and c.d.res and not c.d.out_hi and not c.d.out_lo and c.d.post2_relu == 1
        assert not c.second.d.in_hi and not c.second.d.in_lo and c.second.d.out_hi
    # the same plan when the library runs no pair as one launch: the two launches each chain replaces, with the pair between them
    nets.lib.hd_conv_gemm_chain_supported = lambda *a: 0
    unchained = nets.ResNetPlan(packed, 2, 64, impl, units=(0, 7), root=True, tail=False, next_pre=packed.units[7]['pre'],
                                next_has_shortcut=True)
    assert len(unchained.ops) == len(pa.ops) + 2
    assert unchained.num_launches == pa.num_launches + 2
    i3 = [i for i, o in enumerate(unchained.ops) if o.d is not None and o.d.Cout == 256 and o.d.KH == 1 and o.d.res and o.d.out_hi]
    pairs = [(unchained.ops[i].d, unchained.ops[i + 1].d) for i in i3[:2]]
    for c, (d3, d1) in zip(chains, pairs):
        assert d3.out_hi == d1.in_hi and d1.Cout == 64
        for f in ('n_img', 'H', 'Ho', 'Cout', 'out_subsample', 'post2_relu'):
            assert getattr(c.d, f) == getattr(d3, f), f


def test_whole_plan_chains_the_same_pairs(chain_device):
    nets = chain_device
    from human_dynamics_b200 import synthetic
    packed = nets.PackedResNet(synthetic.make_resnet_weights(seed=1), 'cpu', tc='auto')
    whole = nets.ResNetPlan(packed, 2, 64, 'auto')
    assert sum(isinstance(o, nets.ChainOp) for o in whole.ops) == 2
    assert sum(1 for o in whole.ops if getattr(o, 'd', None) is not None) == 50


def test_library_refuses_pairs_outside_the_rule(chain_device):
    nets = chain_device
    from human_dynamics_b200 import _lib, synthetic
    packed = nets.PackedResNet(synthetic.make_resnet_weights(seed=1), 'cpu', tc='auto')
    pa, _ = _stages(nets, packed, 'auto')
    c = next(o for o in pa.ops if isinstance(o, nets.ChainOp))
    d3, d1 = c.first.d, c.second.d
    lib = _lib.lib
    assert lib.hd_conv_gemm_chain_supported(c.first.ref, c.second.ref) == 1
    for desc, field, bad in ((d3, 'res', None), (d3, 'res_stride', 2), (d3, 'out_hi', d1.out_hi), (d1, 'in_hi', d3.in_hi),
                             (d3, 'KH', 3), (d1, 'Cout', 128), (d3, 'Cout', 512), (d1, 'n_img', 3), (d3, 'post_relu', 1),
                             (d1, 'impl', 4), (d3, 'impl', 1), (d1, 'res', d3.res)):
        keep = getattr(desc, field)
        setattr(desc, field, bad)
        assert lib.hd_conv_gemm_chain_supported(c.first.ref, c.second.ref) == 0, field
        assert lib.hd_conv_gemm_chain(c.first.ref, c.second.ref, None) == HD_ERR_UNSUPPORTED, field
        assert lib.hd_last_error().startswith(b'hd_conv_gemm_chain: ')
        setattr(desc, field, keep)
    assert lib.hd_conv_gemm_chain(None, c.second.ref, None) == HD_ERR_UNSUPPORTED
