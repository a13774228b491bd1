"""The residual layers of conv_gemm_tc (conv_tc.cu, RES: the fp32 residual arrives by TMA in a shared-memory slot per consumer
warpgroup, the fp32 output is staged over it) at the shapes that turn the slot over many times and hit its edges: K = 64 .. 512,
five or six tiles per CTA with a tile count that is not a multiple of the SM count, ragged M, M < 64, Cout = 96 / 192 (a partial
and an absent second half of the slot), both tile widths, each output alone and together.  In the style of
test_gpu_conv_staged_epilogue.py: outputs pre-filled with NaN in buffers with extra rows and padded pitches.  Checked against fp64
of the same arithmetic and, bit for bit, against the same layer without a residual followed by a float32 add (ResNet's conv3 has
no ReLU after the add, so that is the identical sequence of operations); a rerun on the same buffers repeats the bits."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    b = np.asarray(b, np.float64)
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


def _layer(M, Cin, Cout, res, fp32_out, split_out, scale, out_pad=4, pair_pad=8, extra_rows=3, runs=1):
    """One 1x1 layer over M rows (M images of one pixel).  Returns the outputs of every run, cropped to [0, M) x [0, Cout)."""
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.nets import PackedConv
    rng = np.random.RandomState(M * 31 + Cin * 7 + Cout)
    dev = torch.device('cuda')
    x = np.maximum(rng.normal(0, 1, size=(M, 1, 1, Cin)), 0).astype(np.float32)
    w = (rng.normal(0, 1, size=(1, 1, Cin, Cout)) / np.sqrt(Cin)).astype(np.float32)
    bias = rng.normal(0, 0.2, size=Cout).astype(np.float32)
    sc = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32) if scale else None
    s2 = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32); b2 = rng.normal(0, 0.3, size=Cout).astype(np.float32)
    r = rng.normal(0, 1, size=(M, Cout)).astype(np.float32)
    pc = PackedConv(w, dev, post_scale=sc, post_shift=bias, post_relu=False, tc='tc3h')
    xt = torch.from_numpy(x).to(dev)
    hi = xt.half(); lo = ((xt - hi.float()) * 2048).half()
    out = torch.empty((M + extra_rows, Cout + out_pad), device=dev) if fp32_out else None
    oh = torch.empty((M + extra_rows, Cout + pair_pad), dtype=torch.float16, device=dev) if split_out else None
    ol = torch.empty_like(oh) if split_out else None
    rt = torch.from_numpy(r).to(dev) if res else None
    op = pc.bind(None, M, 1, 1, out, out_ld=Cout + out_pad, inp_split=(hi, lo), out_split=(oh, ol) if split_out else None,
                 res=rt, res_geom=(Cout, 1, 1, 1) if res else None,
                 post2=(torch.from_numpy(s2).to(dev), torch.from_numpy(b2).to(dev), 1), impl='tc3h')
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
        for k, t in (('out', out), ('hi', oh), ('lo', ol)):
            if t is None:
                continue
            a = t.cpu().numpy()
            assert np.isnan(a[M:]).all() and np.isnan(a[:M, Cout:]).all(), k + ' written outside [0, M) x [0, Cout)'
            assert not np.isnan(a[:M, :Cout]).any(), k + ' not written everywhere'
            g[k] = a[:M, :Cout].copy()
        got.append(g)
    v = torch.from_numpy(x).double().reshape(M, Cin) @ torch.from_numpy(w).double().reshape(Cin, Cout)
    if sc is not None:
        v = v * torch.from_numpy(sc).double()
    v = v + torch.from_numpy(bias).double()
    if res:
        v = v + torch.from_numpy(r).double()
    y = torch.relu(v * torch.from_numpy(s2).double() + torch.from_numpy(b2).double())
    return got, v.numpy(), y.numpy(), r


def _check(M, Cin, Cout, fp32_out, split_out, scale=False, pair_pad=8):
    got, v, y, r = _layer(M, Cin, Cout, True, fp32_out, split_out, scale, pair_pad=pair_pad, runs=2)
    for k in got[0]:
        assert np.array_equal(got[0][k], got[1][k]), k + ': a rerun on the same buffers differs'
    g = got[0]
    if fp32_out:
        assert rel_err(g['out'], v) < 2e-5
        plain = _layer(M, Cin, Cout, False, True, False, scale)[0][0]['out']
        assert np.array_equal(g['out'], plain + r), 'differs from the layer without a residual + a float32 add'
    if split_out:
        assert rel_err(g['hi'].astype(np.float64) + g['lo'].astype(np.float64) / 2048.0, y) < 2e-5
    return g


# 132 SMs: 331 row tiles x 2 column tiles = 662 tiles of 128 x 128, five or six per CTA, not a multiple of the SM count
RAGGED = [330 * 128 + 1, 330 * 128 + 63, 330 * 128 + 64, 330 * 128 + 65]


@pytest.mark.parametrize('M,Cin', [(RAGGED[0], 64), (RAGGED[1], 128), (RAGGED[2], 256), (RAGGED[3], 512), (RAGGED[1], 64)])
def test_residual_many_tiles_wide(M, Cin):
    """128-wide tiles, both outputs; the pair alone, staged or stored from registers, is the same pair."""
    both = _check(M, Cin, 256, True, True)
    pair = _check(M, Cin, 256, False, True)
    regs = _check(M, Cin, 256, False, True, pair_pad=4)      # a pitch TMA cannot store: nothing staged, the slot is free once read
    for k in ('hi', 'lo'):
        assert np.array_equal(both[k], pair[k]) and np.array_equal(both[k], regs[k]), k


@pytest.mark.parametrize('M,Cin,Cout', [
    (RAGGED[3], 64, 96),          # one column tile, the slot's second half has a single box
    (RAGGED[0], 128, 96),
    (50 * 128 + 1, 64, 192),      # 128-wide (one wave of 100 tiles): odd tiles have no second half and no second weight box
    (50 * 128 + 63, 256, 192),
    (662 * 128 + 65, 64, 64),     # 64-wide tiles, five or six tiles per CTA
    (662 * 128 + 1, 128, 64),
    (3 * 128 + 64, 512, 256),     # small M: 64-wide tiles, the last tile's second warpgroup has no rows
    (63, 64, 256),                # M < 64
    (1, 256, 1024),
])
def test_residual_edges(M, Cin, Cout):
    _check(M, Cin, Cout, True, True, scale=True)
    _check(M, Cin, Cout, True, False)


def test_residual_fp32_only_many_tiles():
    """fp32 output only: the slot's own store group is the last one committed when the slot is reloaded."""
    _check(RAGGED[2], 64, 256, True, False, scale=True)
    _check(RAGGED[0], 256, 256, True, False)
