"""hd_conv_gemm_chain (conv_tc.cu, conv_chain_tc_kernel): conv3 of a bottleneck unit and conv1 of the identity unit after it in one
launch, bit for bit against the two hd_conv_gemm launches it replaces, in impl 3 (tc3h) and impl 4 (tc1h).  The transitions the
ResNet plans chain: block 1 unit 1 -> 2 (the shortcut's output as residual, the full fp32 output) and unit 2 -> 3 (identity residual,
out_subsample = 2); small maps with M below one tile and not a multiple of it, odd maps under the subsample, and tile counts of several
tiles per CTA.  Outputs are pre-filled with NaN in buffers with extra rows, so a write outside the output rows is seen."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CASES = [  # (n, H, out_subsample)
    (2, 56, 0), (3, 56, 0), (2, 56, 2), (20, 56, 0), (20, 56, 2), (1, 7, 0), (1, 13, 2), (2, 5, 2),
]


def _pair(t, heads):
    hi = t.half()
    return (hi, None) if heads else (hi, ((t - hi.float()) * 2048).half())


def _nan(shape, dtype, dev):
    return torch.full(shape, float('nan'), dtype=dtype, device=dev)


def _transition(n, H, sub, impl, seed):
    """Both ways of running conv3 (64 -> 256, bias, residual, post2 = the next unit's pre-activation) and conv1 (256 -> 64, BN + ReLU)."""
    from human_dynamics_b200.nets import PackedConv, ChainOp
    dev = torch.device('cuda')
    heads = impl == 'tc1h'
    rng = np.random.RandomState(seed)
    M, extra = n * H * H, 5
    Hs = (H + sub - 1) // sub if sub > 1 else H
    Mo = n * Hs * Hs
    f = lambda a: torch.from_numpy(np.asarray(a, np.float32)).to(dev)          # noqa: E731
    conv3 = PackedConv((rng.normal(0, 1, size=(1, 1, 64, 256)) / 8).astype(np.float32), dev,
                       post_shift=rng.normal(0, 0.2, size=256).astype(np.float32), tc=impl)
    conv1 = PackedConv((rng.normal(0, 1, size=(1, 1, 256, 64)) / 16).astype(np.float32), dev,
                       rng.uniform(0.5, 1.5, size=64).astype(np.float32), rng.normal(0, 0.3, size=64).astype(np.float32), True, tc=impl)
    post2 = (f(rng.uniform(0.5, 1.5, size=256)), f(rng.normal(0, 0.3, size=256)), 1)
    xin = _pair(torch.relu(f(rng.normal(0, 1, size=(M, 64)))), heads)
    res = f(rng.normal(0, 1, size=(M, 256)))
    outs = []
    for chained in (False, True):
        out = _nan((Mo + extra, 256), torch.float32, dev)
        x_pair = (_nan((M + extra, 256), torch.float16, dev), None if heads else _nan((M + extra, 256), torch.float16, dev))
        r1 = (_nan((M + extra, 64), torch.float16, dev), None if heads else _nan((M + extra, 64), torch.float16, dev))
        op3 = conv3.bind(None, n, H, H, out, inp_split=xin, out_split=x_pair, post2=post2, res=res, res_geom=(256, H, H, 1),
                         out_subsample=sub, impl=impl)
        op1 = conv1.bind(None, n, H, H, None, inp_split=x_pair, out_split=r1, impl=impl)
        st = torch.cuda.current_stream().cuda_stream
        if chained:
            chain = ChainOp.bind(op3, op1)
            assert chain is not None
            for _ in range(2):
                chain.run(st)
        else:
            op3.run(st)
            op1.run(st)
        torch.cuda.synchronize()
        o = {'out': out.cpu().numpy(), 'r1_hi': r1[0].cpu().numpy()}
        if not heads:
            o['r1_lo'] = r1[1].cpu().numpy()
        for k, rows in (('out', Mo), ('r1_hi', M), ('r1_lo', M)):
            if k in o:
                assert np.isnan(o[k][rows:]).all(), k + ' written past its rows'
                assert not np.isnan(o[k][:rows]).any(), k + ' not written everywhere'
        outs.append(o)
    return outs


@pytest.mark.parametrize('impl', ['tc3h', 'tc1h'])
@pytest.mark.parametrize('n,H,sub', CASES)
def test_chain_equals_two_launches_bit_for_bit(impl, n, H, sub):
    two, one = _transition(n, H, sub, impl, seed=n * 977 + H * 31 + sub)
    assert sorted(two) == sorted(one)
    for k in two:
        a, b = two[k], one[k]
        assert np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint16),
                              b.view(np.uint32) if b.dtype == np.float32 else b.view(np.uint16)), k
