"""Pre-split conv_gemm_tc layers write their outputs through shared memory with TMA bulk-tensor stores (the fp32 output over the
residual slot, everything else through a staging buffer), except a pair whose row pitch is not a multiple of 16 bytes, which
leaves from registers.  Every output is pre-filled with NaN in a buffer with extra rows and padded pitches: nothing outside
[0, M) x [0, Cout) may be written and everything inside must be.  Both tile widths, with and without a residual, each output
alone and together, several tiles per CTA and ragged M, against an fp64 reference of the same arithmetic; the staged and the
register-stored pair are bit-identical."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    b = np.asarray(b, np.float64)
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


def _run(n, H, Cin, Cout, res, fp32_out, split_out, out_pad, pair_pad, extra_rows, affine_relu):
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.nets import PackedConv
    rng = np.random.RandomState(n * 7919 + H * 131 + Cin + Cout + 2 * res + 4 * fp32_out + 8 * split_out + 16 * affine_relu)
    dev = torch.device('cuda')
    M = n * H * H
    x = np.maximum(rng.normal(0, 1, size=(n, H, H, Cin)), 0).astype(np.float32)          # already pre-activated
    w = (rng.normal(0, 1, size=(1, 1, Cin, Cout)) / np.sqrt(Cin)).astype(np.float32)
    bias = rng.normal(0, 0.2, size=Cout).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32) if affine_relu else None
    s2 = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32); b2 = rng.normal(0, 0.3, size=Cout).astype(np.float32)
    r = rng.normal(0, 1, size=(M, Cout)).astype(np.float32) if res else None
    pc = PackedConv(w, dev, post_scale=scale, post_shift=bias, post_relu=affine_relu, tc='tc3h')
    xt = torch.from_numpy(x).to(dev)
    hi = xt.half(); lo = ((xt - hi.float()) * 2048).half()
    out = torch.full((M + extra_rows, Cout + out_pad), np.nan, device=dev) if fp32_out else None
    oh = torch.full((M + extra_rows, Cout + pair_pad), np.nan, dtype=torch.float16, device=dev) if split_out else None
    ol = torch.full_like(oh, np.nan) if split_out else None
    op = pc.bind(None, n, H, H, out, out_ld=Cout + out_pad, inp_split=(hi, lo), out_split=(oh, ol) if split_out else None,
                 res=torch.from_numpy(r).to(dev) if res else None, res_geom=(Cout, H, H, 1) if res else None,
                 post2=(torch.from_numpy(s2).to(dev), torch.from_numpy(b2).to(dev), 1), impl='tc3h')
    assert op.d.impl == _lib.HD_IMPL_TC_3XF16
    if split_out:
        op.d.out2_ld = Cout + pair_pad
        op.encode_act_maps()
    op.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()

    v = torch.from_numpy(x).double().reshape(M, Cin) @ torch.from_numpy(w).double().reshape(Cin, Cout)
    if scale is not None:
        v = v * torch.from_numpy(scale).double()
    v = v + torch.from_numpy(bias).double()
    if res:
        v = v + torch.from_numpy(r).double()
    if affine_relu:
        v = torch.relu(v)
    got = {}
    if fp32_out:
        o = out.cpu().numpy()
        assert np.isnan(o[M:]).all() and np.isnan(o[:M, Cout:]).all(), 'fp32 output written outside [0, M) x [0, Cout)'
        assert not np.isnan(o[:M, :Cout]).any(), 'fp32 output not written everywhere'
        assert rel_err(o[:M, :Cout], v.numpy()) < 2e-5
        got['out'] = o[:M, :Cout].copy()
    if split_out:
        h, l = oh.cpu().numpy(), ol.cpu().numpy()
        for a in (h, l):
            assert np.isnan(a[M:]).all() and np.isnan(a[:M, Cout:]).all(), 'pair written outside [0, M) x [0, Cout)'
            assert not np.isnan(a[:M, :Cout]).any(), 'pair not written everywhere'
        y = torch.relu(v * torch.from_numpy(s2).double() + torch.from_numpy(b2).double())
        pair = h[:M, :Cout].astype(np.float64) + l[:M, :Cout].astype(np.float64) / 2048.0      # the pair represents y to ~2^-22
        assert rel_err(pair, y.numpy()) < 2e-5
        got['hi'], got['lo'] = h[:M, :Cout].copy(), l[:M, :Cout].copy()
    return got


SHAPES = [
    # n, H, Cin, Cout, res, fp32_out, split_out, out_pad, pair_pad, extra_rows, affine_relu
    (300, 14, 64, 256, False, True, False, 0, 0, 0, False),     # shortcut conv: fp32 only, 128-wide tile, ~7 tiles per CTA, ragged M
    (41, 14, 64, 256, False, True, False, 12, 0, 37, True),     # fp32 only, padded pitch, scale + ReLU
    (350, 14, 64, 64, False, True, False, 4, 0, 7, False),      # fp32 only, 64-wide tile, ~4 tiles per CTA
    (7, 14, 64, 64, False, False, True, 0, 8, 5, False),        # pair only, 64-wide tile, out2_ld = Cout + 8
    (350, 14, 64, 64, False, False, True, 0, 8, 3, True),       # pair only, 64-wide tile, several tiles per CTA
    (300, 14, 64, 256, False, False, True, 0, 8, 3, False),     # pair only, 128-wide tile, several tiles per CTA
    (300, 14, 64, 256, False, False, True, 0, 4, 3, False),     # same, out2_ld = Cout + 4: the pair leaves from registers
    (5, 14, 64, 96, False, True, True, 4, 8, 9, False),         # both outputs, Cout = 96: the second pass has one fp32 box
    (3, 14, 512, 2048, False, True, True, 0, 8, 2, False),      # both outputs, K = 512 (8 chunks), 16 N tiles
    (4, 14, 64, 256, True, True, True, 8, 8, 11, False),        # residual: fp32 over the residual slot, padded pitches
    (4, 14, 64, 256, True, True, True, 8, 4, 11, False),        # residual, out2_ld = Cout + 4
    (300, 14, 64, 256, True, True, True, 0, 0, 0, True),        # residual, 128-wide tile, several tiles per CTA
    (300, 14, 64, 256, True, False, True, 0, 4, 1, False),      # residual, pair only from registers, several tiles per CTA
    (350, 14, 64, 64, True, True, True, 4, 8, 2, False),        # residual, 64-wide tile (3 stages), several tiles per CTA
    (1, 9, 64, 256, True, True, True, 0, 8, 3, False),          # M = 81: the second warpgroup's rows are all past M
]


@pytest.mark.parametrize('shape', SHAPES)
def test_staged_epilogue_bounds(shape):
    _run(*shape)


@pytest.mark.parametrize('shape', [
    (300, 14, 64, 256, True, True, True, 0, 8, 0, True),
    (350, 14, 64, 64, False, True, True, 0, 8, 0, False),
])
def test_staged_pair_matches_register_pair(shape):
    """out2_ld = Cout + 8 (TMA stores) and Cout + 4 (register stores) compute the same bits, and a rerun repeats them."""
    staged = _run(*shape)
    regs = _run(*(shape[:8] + (4,) + shape[9:]))
    again = _run(*shape)
    for k in staged:
        assert np.array_equal(staged[k], regs[k]), k
        assert np.array_equal(staged[k], again[k]), k
