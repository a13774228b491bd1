"""The short-K pre-split 1x1 layers of conv_gemm_tc (conv_tc.cu, SHORT: K <= 128, 64-wide tiles, two CTAs per SM, one running-sum
flush per tile done in the accumulator itself, the residual slot doubling as the output staging).  K = 64 and 128, Cout = 64 / 96 /
256 / 512, ragged M, M < 64, four or more tiles per CTA with tile counts that are not a multiple of twice the SM count (132 SMs),
with and without a residual, each output alone and together, and the strided subsample (the fp32 output alone without a
residual stays on the one-CTA kernels, so there the cases check that dispatch).  In the style of
test_gpu_conv_residual_shapes.py: outputs pre-filled with NaN in buffers with extra rows and padded pitches.  Checked against fp64 of
the same arithmetic and, bit for bit, against the same layer with the input and the weights zero-padded by 128 channels (K > 128
runs the kernels with the running sums; the zero products leave both accumulator fragments unchanged); a rerun repeats the bits."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    b = np.asarray(b, np.float64)
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


def _layer(n, H, Cin, Cout, res, fp32_out, split_out, sub=0, zero_ch=0, runs=1, out_pad=4, pair_pad=8, extra_rows=3):
    """One 1x1 layer over n images of H x H.  Returns the outputs of every run, cropped to their rows and [0, Cout), and the fp64
    reference of the fp32 output (before any subsample) and of the pair."""
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.nets import PackedConv
    rng = np.random.RandomState(n * 7919 + H * 131 + Cin * 7 + Cout)
    dev = torch.device('cuda')
    M = n * H * H
    x = np.maximum(rng.normal(0, 1, size=(n, H, H, Cin)), 0).astype(np.float32)
    w = (rng.normal(0, 1, size=(1, 1, Cin, Cout)) / np.sqrt(Cin)).astype(np.float32)
    bias = rng.normal(0, 0.2, size=Cout).astype(np.float32)
    sc = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32)
    s2 = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32); b2 = rng.normal(0, 0.3, size=Cout).astype(np.float32)
    r = rng.normal(0, 1, size=(M, Cout)).astype(np.float32)
    xp = np.concatenate([x, np.zeros((n, H, H, zero_ch), np.float32)], axis=3)
    wp = np.concatenate([w, np.zeros((1, 1, zero_ch, Cout), np.float32)], axis=2)
    pc = PackedConv(wp, dev, post_scale=sc, post_shift=bias, post_relu=False, tc='tc3h')
    xt = torch.from_numpy(xp).to(dev)
    hi = xt.half(); lo = ((xt - hi.float()) * 2048).half()
    Hs = (H + sub - 1) // sub if sub > 1 else H
    Mo = n * Hs * Hs
    out = torch.empty((Mo + extra_rows, Cout + out_pad), device=dev) if fp32_out else None
    oh = torch.empty((M + extra_rows, Cout + pair_pad), dtype=torch.float16, device=dev) if split_out else None
    ol = torch.empty_like(oh) if split_out else None
    rt = torch.from_numpy(r).to(dev) if res else None
    op = pc.bind(None, n, H, H, out, out_ld=Cout + out_pad, inp_split=(hi, lo), out_split=(oh, ol) if split_out else None,
                 res=rt, res_geom=(Cout, H, H, 1) if res else None,
                 post2=(torch.from_numpy(s2).to(dev), torch.from_numpy(b2).to(dev), 1), out_subsample=sub, impl='tc3h')
    assert op.d.impl == _lib.HD_IMPL_TC_3XF16
    if split_out:
        op.d.out2_ld = Cout + pair_pad
        op.encode_act_maps()
    got = []
    for _ in range(runs):
        for t in (out, oh, ol):
            if t is not None:
                t.fill_(float('nan'))
        op.run(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        g = {}
        for k, t, rows in (('out', out, Mo), ('hi', oh, M), ('lo', ol, M)):
            if t is None:
                continue
            a = t.cpu().numpy()
            assert np.isnan(a[rows:]).all() and np.isnan(a[:rows, Cout:]).all(), k + ' written outside its rows x [0, Cout)'
            assert not np.isnan(a[:rows, :Cout]).any(), k + ' not written everywhere'
            g[k] = a[:rows, :Cout].copy()
        got.append(g)
    v = torch.from_numpy(x).double().reshape(M, Cin) @ torch.from_numpy(w).double().reshape(Cin, Cout)
    v = v * torch.from_numpy(sc).double() + torch.from_numpy(bias).double()
    if res:
        v = v + torch.from_numpy(r).double()
    y = torch.relu(v * torch.from_numpy(s2).double() + torch.from_numpy(b2).double())
    return got, v.numpy(), y.numpy()


def _check(n, H, Cin, Cout, res, fp32_out, split_out, sub=0):
    got, v, y = _layer(n, H, Cin, Cout, res, fp32_out, split_out, sub=sub, runs=2)
    for k in got[0]:
        assert np.array_equal(got[0][k], got[1][k]), k + ': a rerun on the same buffers differs'
    g = got[0]
    if fp32_out:
        ref = v.reshape(n, H, H, Cout)[:, ::sub, ::sub].reshape(-1, Cout) if sub > 1 else v
        assert rel_err(g['out'], ref) < 2e-5
    if split_out:
        assert rel_err(g['hi'].astype(np.float64) + g['lo'].astype(np.float64) / 2048.0, y) < 2e-5
    long_k = _layer(n, H, Cin, Cout, res, fp32_out, split_out, sub=sub, zero_ch=128)[0][0]
    for k in g:
        assert np.array_equal(g[k], long_k[k]), k + ': differs from the same layer over K + 128 zero channels'


SHAPES = [
    # n, H, Cin, Cout: M = n H^2; tiles of 128 x 64 against 2 x 132 CTAs
    (690, 14, 64, 64),       # 1057 tiles: four per CTA, one CTA a fifth
    (345, 14, 128, 96),      # 529 x 2 tiles, the second column tile has one 32-column box of two
    (196, 14, 64, 256),      # 301 x 4 tiles, M = 300 x 128 + 16
    (196, 14, 128, 256),
    (87, 14, 128, 512),      # 134 x 8 tiles, M = 133 x 128 + 28
    (87, 14, 64, 512),
    (3, 9, 128, 96),         # M = 243: the second warpgroup of the last row tile has 51 rows
    (1, 7, 64, 256),         # M = 49 < 64: no second warpgroup rows at all
]


@pytest.mark.parametrize('n,H,Cin,Cout', SHAPES)
@pytest.mark.parametrize('res', [False, True])
def test_short_k_outputs(n, H, Cin, Cout, res):
    """Both outputs, the fp32 output alone and the pair alone: the pair is staged in the slot once the fp32 stores have read it."""
    _check(n, H, Cin, Cout, res, True, True)
    _check(n, H, Cin, Cout, res, True, False)
    _check(n, H, Cin, Cout, res, False, True)


@pytest.mark.parametrize('n,H,Cin,Cout', [(40, 14, 64, 256), (41, 15, 128, 96), (180, 14, 64, 64)])
@pytest.mark.parametrize('res', [False, True])
def test_short_k_subsample(n, H, Cin, Cout, res):
    """out_subsample: the fp32 rows x[:, ::2, ::2] stored from registers, the pair staged."""
    _check(n, H, Cin, Cout, res, True, True, sub=2)
    _check(n, H, Cin, Cout, res, True, False, sub=2)
