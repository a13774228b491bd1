"""Pre-split conv_gemm_tc layers with a residual row-aligned with the output: the residual tile reaches the epilogue through
shared memory (TMA, 32-column boxes of 64 rows per warpgroup).  Ragged M and Cout (partial and skipped boxes), both tile widths,
one and eight K chunks, every output combination, a padded residual pitch, the strided subsample output, several tiles per CTA
(slot reuse, barrier phases) and run-to-run bit-identity, against an fp64 reference of the same arithmetic."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    b = np.asarray(b, np.float64)
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


def _case(n, H, Cin, Cout, res_pad, fp32_out, split_out, sub, affine_relu):
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.nets import PackedConv
    rng = np.random.RandomState(n * 7919 + H * 131 + Cin + Cout + res_pad + 2 * fp32_out + 4 * split_out + 8 * sub + 16 * affine_relu)
    dev = torch.device('cuda')
    x = np.maximum(rng.normal(0, 1, size=(n, H, H, Cin)), 0).astype(np.float32)          # already pre-activated
    w = (rng.normal(0, 1, size=(1, 1, Cin, Cout)) / np.sqrt(Cin)).astype(np.float32)
    bias = rng.normal(0, 0.2, size=Cout).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32) if affine_relu else None
    s2 = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32); b2 = rng.normal(0, 0.3, size=Cout).astype(np.float32)
    res_ld = Cout + res_pad
    r = rng.normal(0, 1, size=(n, H, H, res_ld)).astype(np.float32)
    pc = PackedConv(w, dev, post_scale=scale, post_shift=bias, post_relu=affine_relu, tc='tc3h')
    xt = torch.from_numpy(x).to(dev)
    hi = xt.half(); lo = ((xt - hi.float()) * 2048).half()
    Hs = (H + sub - 1) // sub if sub > 1 else H
    out = torch.full((n, Hs, Hs, Cout), np.nan, device=dev) if fp32_out else None
    oh = torch.zeros((n, H, H, Cout), dtype=torch.float16, device=dev) if split_out else None
    ol = torch.zeros_like(oh) if split_out else None
    rt = torch.from_numpy(r).to(dev)
    op = pc.bind(None, n, H, H, out, inp_split=(hi, lo), out_split=(oh, ol) if split_out else None, res=rt,
                 res_geom=(res_ld, H, H, 1), post2=(torch.from_numpy(s2).to(dev), torch.from_numpy(b2).to(dev), 1),
                 out_subsample=sub if sub > 1 else 0, impl='tc3h')
    assert op.d.impl == _lib.HD_IMPL_TC_3XF16

    def run():
        op.run(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return (out.cpu().numpy().copy() if fp32_out else None,
                (oh.cpu().numpy().copy(), ol.cpu().numpy().copy()) if split_out else None)

    got32, got2 = run()
    v = torch.from_numpy(x).double().reshape(-1, Cin) @ torch.from_numpy(w).double().reshape(Cin, Cout)
    if scale is not None:
        v = v * torch.from_numpy(scale).double()
    v = (v + torch.from_numpy(bias).double() + torch.from_numpy(r).double().reshape(-1, res_ld)[:, :Cout]).reshape(n, H, H, Cout)
    if affine_relu:
        v = torch.relu(v)
    if fp32_out:
        assert rel_err(got32, v[:, ::sub, ::sub].numpy() if sub > 1 else v.numpy()) < 2e-5
    if split_out:
        y = torch.relu(v * torch.from_numpy(s2).double() + torch.from_numpy(b2).double())
        pair = got2[0].astype(np.float64) + got2[1].astype(np.float64) / 2048.0      # the pair represents y to ~2^-22
        assert rel_err(pair, y.numpy()) < 2e-5
    again32, again2 = run()
    if fp32_out:
        assert np.array_equal(got32, again32)
    if split_out:
        assert np.array_equal(got2[0], again2[0]) and np.array_equal(got2[1], again2[1])


@pytest.mark.parametrize('shape', [
    # n, H, Cin, Cout, res_pad, fp32_out, split_out, sub, affine_relu
    (1, 9, 64, 256, 0, True, True, 1, False),        # M = 81 < 128: the second warpgroup's rows are all past M (no box)
    (3, 14, 512, 2048, 0, False, True, 1, False),    # K = 512 (8 chunks), M = 588 ragged, 16 N tiles
    (3, 14, 512, 2048, 0, True, False, 1, True),     # same with scale + ReLU and the fp32 output only
    (5, 14, 64, 96, 0, True, True, 1, False),        # Cout = 96: the last N tile has one 32-column box
    (40, 14, 64, 160, 0, True, True, 1, False),      # Cout = 160, 128-wide tiles: one box of four, three not loaded
    (7, 14, 64, 64, 0, True, True, 1, True),         # Cout = 64: 64-wide tile
    (4, 14, 64, 256, 32, True, True, 1, False),      # res_ld = Cout + 32
    (2, 28, 512, 256, 4, False, True, 1, False),     # res_ld = Cout + 4, K = 512
    (6, 14, 64, 256, 0, True, True, 2, False),       # residual + out_subsample (strided fp32 rows, pair dense)
    (5, 9, 128, 512, 0, True, True, 3, False),       # odd map, subsample 3
    (300, 14, 64, 256, 0, True, True, 1, False),     # ~7 tiles per CTA (128-wide): slot reuse across barrier phases
    (350, 14, 64, 64, 0, False, True, 1, False),     # ~4 tiles per CTA through the 64-wide tile
    (100, 7, 512, 2048, 0, True, True, 1, False),    # block 4 conv3 shape, 39 x 16 tiles
])
def test_presplit_residual_epilogue(shape):
    _case(*shape)
