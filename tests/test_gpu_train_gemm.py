"""GPU: the backward GEMMs of f_movie, the IEF heads, fc2_res and D_pose, one at a time, and the operand builders behind them.

Each GEMM runs through the production helpers (trainable._xt / _stack_t / _bt_operand / _wgrad, nets.dgrad_op over a
BackwardDataPack) with the call shape of its site in trainable.py / adversarial.py, in both gradient precisions:
  'tf32'  against a float64 emulation of the operands as the kernels round them (the A operand rn_tf32 of the fp32 input, as the
          register-staged producer rounds it; the B operand the TF32 head of hd_transpose_split mode 1 / hd_pack_weight), products
          and sums in float64; and against plain float64;
  'fp32'  (3xTF32) against plain float64.
Every result is checked as a whole and on its ragged parts (the last partial 64-row and 64-column tile, the d columns), and the memory
the helpers allocate is poisoned with NaN first, so a padding row or column that is not written as zero shows up.  Then the operand
builders of csrc/net_grad.cu against float64 (or bit for bit where they only copy, round or add in a fixed order), hd_conv_gemm with
`out` == `res` against separate buffers, and hd_ief_fc3 at every D it accepts."""
import ctypes as C

import numpy as np
import pytest
import torch

from tf32_emulation import rn_tf32

pytestmark = pytest.mark.gpu

# Bars, per-tensor relative L2 (of a whole result or of one ragged part of it), from measurements on an NVIDIA H100 80GB HBM3
# (700 W); the worst measured value is next to each bar.  Every kernel here is deterministic, so a rerun measures the same values.
EMU_BAR = 1e-5            # 'tf32' against the float64 emulation of the operand rounding, fp32 accumulation noise alone: 7.1e-7
TF32_F64_BAR = 1e-3       # 'tf32' against plain float64: 3.5e-4
FP32_BAR = 1e-6           # 'fp32' (3xTF32) against plain float64 (the trunk's 3xTF32 tests: 2e-6): 2.7e-7
SMALL_BAR = 1e-6          # fp32 CUDA-core sums (hd_fc_small_dgrad, hd_ief_fc3, dbeta_part) against float64: 1.8e-7 (hd_fc_small_dgrad)
GN_BAR = 1e-6             # hd_groupnorm_relu_backward's dx and dgamma_part against float64: 1.3e-7 (dgamma_part)

NAN = float('nan')
MODES = [False, True]     # one_pass: 'fp32' (3xTF32), 'tf32' (1xTF32)


def _vp(t, off=0):
    return C.c_void_p(t.data_ptr() + off) if t is not None else None


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from human_dynamics_b200._lib import lib, check
    return lib, check


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _round(x, m):
    return (x + m - 1) // m * m


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, NAN, dtype=dtype, device='cuda')


def _mm(a, b):
    """float64 product of two host arrays, on the device."""
    return (torch.from_numpy(np.asarray(a, np.float64)).cuda() @ torch.from_numpy(np.asarray(b, np.float64)).cuda()).cpu().numpy()


@pytest.fixture(autouse=True)
def _poison():
    """Fill the memory the caching allocator hands out next with NaN: the helpers' torch.empty operands (_xt, _bt_operand) then start
    as NaN, so any element of their padding that the builders do not write reaches the GEMM as NaN."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    big = torch.full((96 << 20,), NAN, device='cuda')                      # 384 MiB: the large pool
    small = [torch.full((1 << 18,), NAN, device='cuda') for _ in range(32)]   # 1 MiB blocks: the small pool
    torch.cuda.synchronize()
    del big, small
    yield


def _regions(M, N):
    """The parts of an [M, N] result checked on their own: the whole, the last (partial) 64-row tile, the last 64-column tile."""
    r0, c0 = 64 * ((M - 1) // 64), 64 * ((N - 1) // 64)
    return {'all': (slice(None), slice(None)), 'rows %d:' % r0: (slice(r0, None), slice(None)),
            'cols %d:' % c0: (slice(None), slice(c0, None))}


def _check(tag, got, one_pass, emu, f64):
    """got against the emulation ('tf32') and float64, as a whole and per ragged part; returns the worst errors."""
    assert np.isfinite(got).all(), tag
    worst = [0.0, 0.0]
    for name, sl in _regions(*got.shape).items():
        g = got[sl]
        if one_pass:
            e, f = _rel(g, emu[sl]), _rel(g, f64[sl])
            assert e < EMU_BAR and f < TF32_F64_BAR, (tag, name, e, f)
        else:
            e, f = 0.0, _rel(g, f64[sl])
            assert f < FP32_BAR, (tag, name, f)
        worst = [max(worst[0], e), max(worst[1], f)]
    print('%s %s: vs emulation %.2e, vs float64 %.2e' % (tag, 'tf32' if one_pass else 'fp32', worst[0], worst[1]))
    return worst


def _guarded(rows, cols):
    """A NaN buffer with 64 spare rows: (the [rows, cols] output view, the spare rows that must stay NaN)."""
    buf = _nan((rows + 64, cols))
    return buf[:rows], buf[rows:]


def _untouched(spare, tag):
    assert bool(torch.isnan(spare).all()), '%s: written outside the output' % tag


# ------------------------------------------------------------------------------------------------------------------------------------
# weight gradients of the FC layers: out[M, cols] = X^T . G, X = rows of the layer input, G = rows of its output gradient, K = rows
# ------------------------------------------------------------------------------------------------------------------------------------
# site: (M = the layer's fan-in, cols = its fan-out, rows per N: 1 = N (phi part, fc2_res, D_pose), 3 = 3N (the IEF stages))
WGRAD_SITES = {'ief_fc1_phi': (2048, 1024, 1), 'ief_fc2': (1024, 1024, 3), 'ief_fc3_main': (1024, 85, 3), 'ief_fc3_delta': (1024, 72, 3),
               'hal_fc': (2048, 2048, 1), 'dpose_fc1': (736, 1024, 1), 'dpose_fc2': (1024, 1024, 1)}
# N: 1; 7 (kp = 32, K % 64 == 32; 3N = 21 likewise); 11 (3N = 33, just past 32); 33; 40; 640 (B*T of the C3 window); D_pose's
# batches of 800 and 3200
WGRAD_CASES = [(site, N) for site in sorted(WGRAD_SITES) for N in [1, 7, 11, 33, 40, 640] + ([800, 3200] if site.startswith('dpose') else [])]


@pytest.mark.parametrize('one_pass', MODES)
@pytest.mark.parametrize('site,N', WGRAD_CASES)
def test_fc_weight_gradient(site, N, one_pass):
    """`_wgrad(_xt([(x, R, M)], M, kp, st), M, kp, [(g, R, cols)], cols, W, st, one_pass)` as every FC site calls it."""
    from human_dynamics_b200.trainable import _wgrad, _xt
    M, cols, per = WGRAD_SITES[site]
    R = per * N
    kp = _round(R, 32)
    rng = np.random.RandomState(R * 7 + M + cols)
    x = np.maximum(rng.normal(0.2, 1, (R, M)), 0).astype(np.float32)       # a ReLU output, as every site's layer input
    g = (rng.normal(0, 1, (R, cols)) * 1e-3).astype(np.float32)
    xt, gt = torch.from_numpy(x).cuda(), torch.from_numpy(g).cuda()
    W, spare = _guarded(M, cols)
    st = _st()
    _wgrad(_xt([(xt, R, M)], M, kp, st), M, kp, [(gt, R, cols)], cols, W, st, one_pass)
    got = W.cpu().numpy()
    _untouched(spare, site)
    _check('%s N=%d' % (site, N), got, one_pass, _mm(rn_tf32(x).T, rn_tf32(g)), _mm(x.T, g))


def _theta_inputs(d, N, rng):
    """The IEF theta part's row blocks as ief_head_backward stacks them: the head's start, then the outputs of stages 0 and 1.  The main
    head's start is [N, 85]; a delta head's is the pose columns 3:75 of the main head's output, read in place at row stride 85."""
    theta = rng.normal(0, 1, (N, 85)).astype(np.float32)
    mids = [rng.normal(0, 1, (N, d)).astype(np.float32) for _ in range(2)]
    th = torch.from_numpy(theta).cuda()
    if d == 85:
        start, start_np = th, theta
    else:
        start, start_np = torch.as_strided(th, (N, 72), (85, 1), th.storage_offset() + 3), theta[:, 3:75]
    ms = [torch.from_numpy(m).cuda() for m in mids]
    return th, [(start, 85), (ms[0], d), (ms[1], d)], [start_np] + mids


@pytest.mark.parametrize('one_pass', MODES)
@pytest.mark.parametrize('N', [1, 7, 11, 40, 640])
@pytest.mark.parametrize('d', [85, 72])
def test_ief_theta_weight_gradient(d, N, one_pass):
    """The theta part of the IEF fc1 weight gradient: three row blocks stacked along K at column offsets 0, N, 2N (K = roundup32(3N)),
    M = d rows, less than one tile, written into the W1[feat:] view of the whole weight gradient."""
    from human_dynamics_b200.trainable import _wgrad, _xt
    rng = np.random.RandomState(d * 1000 + N)
    feat = 2048
    kp3 = _round(3 * N, 32)
    _keep, ins, blocks = _theta_inputs(d, N, rng)
    dp1 = (rng.normal(0, 1, (3 * N, 1024)) * 1e-3).astype(np.float32)
    DP1 = torch.from_numpy(dp1).cuda()
    W1, spare = _guarded(feat + d, 1024)
    st = _st()
    _wgrad(_xt([(t, N, ld) for t, ld in ins], d, kp3, st), d, kp3, [(DP1, 3 * N, 1024)], 1024, W1[feat:], st, one_pass)
    full = W1.cpu().numpy()
    assert np.isnan(full[:feat]).all(), 'the phi rows W1[:feat] were written'
    _untouched(spare, 'theta part')
    a = np.concatenate(blocks, 0)                                           # [3N, d]: the stacked K rows
    _check('ief theta d=%d N=%d' % (d, N), full[feat:], one_pass, _mm(rn_tf32(a).T, rn_tf32(dp1)), _mm(a.T, dp1))


FMOVIE_BT = [(1, 1), (1, 7), (3, 11), (2, 20), (1, 25), (32, 20)]        # B*T = 1, 7, 33, 40, 25, 640


def _fmovie_input(B, T, Cc, seed):
    rng = np.random.RandomState(seed)
    x = (rng.normal(0.1, 1, (B, T, Cc)) + rng.normal(0, 0.3, (B, 1, Cc))).astype(np.float32)
    gam = rng.uniform(0.5, 1.5, Cc).astype(np.float32)
    bet = rng.normal(0, 0.3, Cc).astype(np.float32)
    return x, gam, bet


def _gn_affine(xt, gt, bt, B, T, Cc):
    from human_dynamics_b200.nets import GN_EPS, GN_GROUPS
    lib, check = _lib()
    gain, offset = torch.empty((B, Cc), device='cuda'), torch.empty((B, Cc), device='cuda')
    check(lib.hd_groupnorm_stats(_vp(xt), _vp(gt), _vp(bt), _vp(gain), _vp(offset), B, T, Cc, GN_GROUPS, GN_EPS, _st()),
          'hd_groupnorm_stats')
    return gain, offset


def _act(x, gain, offset):
    """relu(x * gain + offset) as im2col_t computes it: one fused multiply-add (exact in float64, rounded once to fp32)."""
    v = (x.astype(np.float64) * gain[:, None].astype(np.float64) + offset[:, None].astype(np.float64)).astype(np.float32)
    return np.maximum(v, np.float32(0))


def _im2col_ref(a, KH, pad, out_cols):
    """hd_im2col_t's contract on a host array a [B, T, C]: [KH*C, out_cols]."""
    B, T, Cc = a.shape
    out = np.zeros((KH * Cc, out_cols), np.float32)
    for kh in range(KH):
        sh = np.zeros_like(a)
        lo, hi = max(0, pad - kh), min(T, T + pad - kh)
        if hi > lo:
            sh[:, lo:hi] = a[:, lo + kh - pad:hi + kh - pad]
        out[kh * Cc:(kh + 1) * Cc, :B * T] = sh.reshape(B * T, Cc).T
    return out


@pytest.mark.parametrize('one_pass', MODES)
@pytest.mark.parametrize('B,T', FMOVIE_BT)
def test_fmovie_weight_gradient(B, T, one_pass):
    """f_movie's dW as fmovie_backward computes it: hd_groupnorm_stats, hd_im2col_t of relu(gn(x)) into [3*Cc, kp], then
    _wgrad(xt, 3*Cc, kp, [(gin, B*T, Cc)], Cc, dW): M = 6144, N = 2048, K = kp = roundup32(B*T)."""
    from human_dynamics_b200.trainable import _wgrad
    lib, check = _lib()
    Cc, BT = 2048, B * T
    kp = _round(BT, 32)
    x, gam, bet = _fmovie_input(B, T, Cc, 10 * B + T)
    g = (np.random.RandomState(B + 100 * T).normal(0, 1, (BT, Cc)) * 1e-3).astype(np.float32)
    xt, gt, bt, gint = (torch.from_numpy(v).cuda() for v in (x, gam, bet, g))
    gain, offset = _gn_affine(xt, gt, bt, B, T, Cc)
    st = _st()
    col = _nan((3 * Cc, kp))
    check(lib.hd_im2col_t(_vp(xt), B, T, Cc, 3, 1, _vp(gain), _vp(offset), 1, _vp(col), kp, kp, st), 'hd_im2col_t')
    dW, spare = _guarded(3 * Cc, Cc)
    _wgrad(col, 3 * Cc, kp, [(gint, BT, Cc)], Cc, dW, st, one_pass)
    got = dW.cpu().numpy()
    _untouched(spare, 'f_movie dW')
    a = _im2col_ref(_act(x, gain.cpu().numpy(), offset.cpu().numpy()), 3, 1, BT)    # [3*Cc, B*T], built on the host
    _check('f_movie dW B=%d T=%d' % (B, T), got, one_pass, _mm(rn_tf32(a), rn_tf32(g)), _mm(a, g))


# ------------------------------------------------------------------------------------------------------------------------------------
# data gradients: dX = dY . W^T through the BackwardDataPack of each layer
# ------------------------------------------------------------------------------------------------------------------------------------
# site: (rows of the weight W [in, out] (the IEF fc1: feat + d, of which the pack reads the first feat), Cin = the pack's output
# width, Cout = K, the residual: None, 'sep' (fc2_res fc1: + g) or 'alias' (IEF fc1 of every head after the first: out = res = dphi))
DGRAD_SITES = {'ief_fc2': (1024, 1024, 1024, None), 'ief_fc1_first': (2048 + 85, 2048, 1024, None),
               'ief_fc1_accumulate': (2048 + 72, 2048, 1024, 'alias'), 'hal_fc3': (2048, 2048, 2048, None),
               'hal_fc1': (2048, 2048, 2048, 'sep'), 'dpose_fc2': (1024, 1024, 1024, None), 'dpose_fc1': (736, 736, 1024, None)}
# N: 1, 7, 33, 40, 640 everywhere; D_pose's batches of 800 and 3200 too
DGRAD_CASES = [(site, N) for site in sorted(DGRAD_SITES) for N in [1, 7, 33, 40, 640] + ([800, 3200] if site.startswith('dpose') else [])]


@pytest.mark.parametrize('one_pass', MODES)
@pytest.mark.parametrize('site,N', DGRAD_CASES)
def test_fc_data_gradient(site, N, one_pass):
    """dgrad_op(BackwardDataPack(W, 1, Cin, Cout), dY, N, 1, 1, 1, 1, out[, res]) as each site calls it.  With the residual aliased
    (ief_head_backward: out = res = dphi) the result is also bit-identical to the same call with separate buffers."""
    from human_dynamics_b200.nets import BackwardDataPack, dgrad_op
    rows, Cin, Cout, res = DGRAD_SITES[site]
    rng = np.random.RandomState(N + rows + Cin)
    w = (rng.normal(0, 1, (rows, Cout)) / np.sqrt(Cout)).astype(np.float32)
    dy = (rng.normal(0, 1, (N, Cout)) * 1e-3).astype(np.float32)
    r = (rng.normal(0, 1, (N, Cin)) * 1e-3).astype(np.float32) if res else None
    wt, dyt = torch.from_numpy(w).cuda(), torch.from_numpy(dy).cuda()
    pack = BackwardDataPack(wt, 1, Cin, Cout)
    pack.repack(_st())
    out, spare = _guarded(N, Cin)
    st = _st()
    if res == 'alias':
        out.copy_(torch.from_numpy(r))
        sep_res, sep_out = torch.from_numpy(r).cuda(), _nan((N, Cin))
        dgrad_op(pack, dyt, N, 1, 1, 1, 1, sep_out, res=sep_res, one_pass=one_pass).run(st)
        dgrad_op(pack, dyt, N, 1, 1, 1, 1, out, res=out, one_pass=one_pass).run(st)
        assert torch.equal(out, sep_out), 'out == res differs from separate buffers'
    else:
        rt = torch.from_numpy(r).cuda() if res else None
        dgrad_op(pack, dyt, N, 1, 1, 1, 1, out, res=rt, one_pass=one_pass).run(st)
    got = out.cpu().numpy()
    _untouched(spare, site)
    wc = w[:Cin]
    emu, f64 = _mm(rn_tf32(dy), rn_tf32(wc).T), _mm(dy, wc.T)
    if res:
        emu, f64 = emu + r, f64 + r
    _check('%s N=%d' % (site, N), got, one_pass, emu, f64)


@pytest.mark.parametrize('one_pass', MODES)
@pytest.mark.parametrize('B,T', FMOVIE_BT)
def test_fmovie_data_gradient(B, T, one_pass):
    """dgrad_op(fm_bwd, gin, B, T, 1, 3, 1, dact): the 3x1 SAME conv over T of the output gradient with the tap-flipped, transposed
    weight, clip by clip (no frame reads across a clip's ends)."""
    from human_dynamics_b200.nets import BackwardDataPack, dgrad_op
    Cc = 2048
    rng = np.random.RandomState(B * 31 + T)
    w = (rng.normal(0, 1, (3, Cc, Cc)) / np.sqrt(3 * Cc)).astype(np.float32)
    g = rng.normal(0, 1, (B, T, Cc)).astype(np.float32)
    wt, gt = torch.from_numpy(w).cuda(), torch.from_numpy(g).cuda()
    pack = BackwardDataPack(wt, 3, Cc, Cc)
    pack.repack(_st())
    out, spare = _guarded(B * T, Cc)
    dgrad_op(pack, gt, B, T, 1, 3, 1, out, one_pass=one_pass).run(_st())
    got = out.cpu().numpy()
    _untouched(spare, 'f_movie dX')

    def ref(wv, gv):                 # forward y[t] = sum_kh x[t + kh - 1] W[kh]  =>  dx[t] = sum_kh dy[t + 1 - kh] W[kh]^T
        a = _im2col_ref(gv[:, :, :], 3, 1, B * T)                      # rows kh*Cc + co: gv[b, t + kh - 1, co]
        wf = wv[::-1].transpose(0, 2, 1).reshape(3 * Cc, Cc)           # row k'*Cc + co: W[2 - k', :, co] (the pack's K order)
        return _mm(a.T, wf)
    _check('f_movie dX B=%d T=%d' % (B, T), got, one_pass, ref(rn_tf32(w), rn_tf32(g)), ref(w, g))


# ------------------------------------------------------------------------------------------------------------------------------------
# hd_conv_gemm with out == res (impl 1 and 2)
# ------------------------------------------------------------------------------------------------------------------------------------
# the IEF fc1 dX (N rows, Cin = 2048, K = 1024) and the trunk's bottleneck conv1 in a unit with a conv shortcut (n = 2 frames at 224²:
# the first unit of each block, dX of the 1x1 conv Cin -> Cout over H x H pixels, accumulated into the shortcut's dX P)
ALIAS_SHAPES = [(1, 1, 2048, 1024), (7, 1, 2048, 1024), (40, 1, 2048, 1024), (640, 1, 2048, 1024),
                (2, 56, 64, 64), (2, 28, 256, 128), (2, 14, 512, 256), (2, 7, 1024, 512)]


@pytest.mark.parametrize('one_pass', MODES)
@pytest.mark.parametrize('n,H,Cin,Cout', ALIAS_SHAPES)
def test_conv_gemm_out_aliasing_res(n, H, Cin, Cout, one_pass):
    """hd_conv_gemm in impl 1 / 2 with out == res gives the bits of the same call with a separate residual buffer: every element of the
    residual row-aligned with the output is read by the thread that writes it, before it writes it."""
    from human_dynamics_b200.nets import BackwardDataPack, dgrad_op
    rng = np.random.RandomState(n * H + Cin)
    w = (rng.normal(0, 1, (Cin, Cout)) / np.sqrt(Cout)).astype(np.float32)
    d2 = rng.normal(0, 1, (n, H, H, Cout)).astype(np.float32)
    p0 = rng.normal(0, 1, (n, H, H, Cin)).astype(np.float32)
    wt, d2t = torch.from_numpy(w).cuda(), torch.from_numpy(d2).cuda()
    pack = BackwardDataPack(wt, 1, Cin, Cout)
    pack.repack(_st())
    P = torch.from_numpy(p0).cuda()
    res, sep = torch.from_numpy(p0).cuda(), _nan((n, H, H, Cin))
    st = _st()
    dgrad_op(pack, d2t, n, H, H, 1, 1, sep, res=res, one_pass=one_pass).run(st)
    dgrad_op(pack, d2t, n, H, H, 1, 1, P, res=P, one_pass=one_pass).run(st)
    assert torch.equal(P, sep)
    assert torch.equal(res, torch.from_numpy(p0).cuda())
    a, b = d2.reshape(-1, Cout), w.T
    f64 = _mm(rn_tf32(a), rn_tf32(b)) if one_pass else _mm(a, b)
    e = _rel(P.cpu().numpy().reshape(-1, Cin).astype(np.float64) - p0.reshape(-1, Cin), f64)
    assert e < (EMU_BAR if one_pass else FP32_BAR), e


# ------------------------------------------------------------------------------------------------------------------------------------
# operand builders (csrc/net_grad.cu)
# ------------------------------------------------------------------------------------------------------------------------------------
def _split_ref(v, mode):
    """store_split on host float32 values: (hi, lo) with the kernels' roundings."""
    if mode == 0:
        return v, None
    if mode == 1:
        h = rn_tf32(v)
        return h, rn_tf32((v - h).astype(np.float32))
    h = v.astype(np.float16)
    return h, ((v - h.astype(np.float32)) * np.float32(2048)).astype(np.float16)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


@pytest.mark.parametrize('mode,with_lo', [(0, False), (1, True), (1, False), (2, True)])
@pytest.mark.parametrize('rows,cols,out_rows,out_cols', [(1, 85, 128, 32), (21, 72, 128, 32), (33, 1024, 1024, 64), (640, 2048, 2048, 640),
                                                         (100, 40, 64, 100), (70, 64, 64, 96)])
def test_transpose_split_contract(mode, with_lo, rows, cols, out_rows, out_cols):
    """hi[r, off + k] = split(x[k, r]) for r < cols, k < rows; exactly 0 on [cols, out_rows) and [rows, out_cols); nothing written
    outside out_rows x out_cols (the buffer has a column offset, spare columns in its pitch and spare rows, all NaN)."""
    lib, check = _lib()
    rng = np.random.RandomState(rows + cols + 3 * mode)
    ld = cols + 5
    x = (rng.normal(0, 1, (rows, ld)) * np.exp2(rng.randint(-8, 8, (rows, ld)))).astype(np.float32)
    b = x.reshape(-1).view(np.uint32)
    b[::3] = (b[::3] & np.uint32(0xFFFFE000)) | np.uint32(0x1000)          # every third value a TF32 tie
    off, pitch = 7, out_cols + 7 + 9
    dt = torch.float16 if mode == 2 else torch.float32
    hi, lo = _nan((out_rows + 5, pitch), dt), (_nan((out_rows + 5, pitch), dt) if with_lo else None)
    before = hi.cpu().numpy()
    esz = hi.element_size()
    xt = torch.from_numpy(x).cuda()
    check(lib.hd_transpose_split(_vp(xt), rows, cols, ld, mode, _vp(hi, off * esz),
                                 _vp(lo, off * esz) if with_lo else None, pitch, out_rows, out_cols, _st()), 'hd_transpose_split')
    h, lo_ref = _split_ref(x[:, :cols].T.copy(), mode)
    for got, ref in ((hi, h), (lo, lo_ref)) if with_lo else ((hi, h),):
        want = before.copy()
        want[:out_rows, off:off + out_cols] = 0
        want[:cols, off:off + rows] = ref
        assert np.array_equal(_bits(got.cpu().numpy()), _bits(want))


@pytest.mark.parametrize('KH,pad', [(1, 0), (3, 1), (3, 0)])
@pytest.mark.parametrize('B,T,Cc,extra', [(1, 1, 64, 31), (3, 7, 40, 11), (2, 20, 2048, 24), (4, 1, 96, 0)])
@pytest.mark.parametrize('affine', ['none', 'affine', 'affine_relu'])
def test_im2col_t_contract(KH, pad, B, T, Cc, extra, affine):
    """out[(kh*C + c), b*T + t] = a[b, t + kh - pad, c] (0 outside the clip), zero columns [B*T, out_cols), nothing else written;
    bit for bit against a host restatement (a = x, x*gain + offset, or relu of it)."""
    lib, check = _lib()
    rng = np.random.RandomState(B * T + Cc + KH)
    x = rng.normal(0, 1, (B, T, Cc)).astype(np.float32)
    gain = rng.uniform(0.5, 1.5, (B, Cc)).astype(np.float32)
    offset = rng.normal(0, 0.5, (B, Cc)).astype(np.float32)
    out_cols = B * T + extra
    out_ld = out_cols + 3
    out = _nan((KH * Cc + 2, out_ld))
    xt = torch.from_numpy(x).cuda()
    g, o = (torch.from_numpy(gain).cuda(), torch.from_numpy(offset).cuda()) if affine != 'none' else (None, None)
    check(lib.hd_im2col_t(_vp(xt), B, T, Cc, KH, pad, _vp(g), _vp(o), int(affine == 'affine_relu'), _vp(out), out_ld, out_cols, _st()),
          'hd_im2col_t')
    a = x
    if affine != 'none':
        a = (x.astype(np.float64) * gain[:, None].astype(np.float64) + offset[:, None].astype(np.float64)).astype(np.float32)
        if affine == 'affine_relu':
            a = np.maximum(a, np.float32(0))
    want = np.full((KH * Cc + 2, out_ld), np.nan, np.float32)
    want[:KH * Cc, :out_cols] = _im2col_ref(a, KH, pad, out_cols)
    assert np.array_equal(_bits(out.cpu().numpy()), _bits(want))


def _col_sum_ref(x, rows, cols):
    """col_sum_kernel's order in float32: per column 8 slices (rows slice, slice + 8, ...), each summed in row order from +0, then the
    slices in order from +0."""
    nb = (rows + 7) // 8
    pad = np.zeros((nb * 8, cols), np.float32)
    pad[:rows] = x[:rows, :cols]
    pad = pad.reshape(nb, 8, cols)
    s = np.zeros((8, cols), np.float32)
    for i in range(nb):
        s = s + pad[i]
    t = np.zeros(cols, np.float32)
    for k in range(8):
        t = t + s[k]
    return t


@pytest.mark.parametrize('rows,cols,ld', [(1, 85, 85), (7, 1024, 1030), (8 * 403 + 3, 85, 96), (8 * 80 + 3, 2048, 2048),
                                          (1920, 72, 85), (3, 45, 50)])
def test_col_sum_bit_exact(rows, cols, ld):
    lib, check = _lib()
    x = np.random.RandomState(rows + cols).normal(0, 1, (rows, ld)).astype(np.float32)
    out = _nan((cols + 40,))
    xt = torch.from_numpy(x).cuda()
    check(lib.hd_col_sum(_vp(xt), rows, cols, ld, _vp(out), _st()), 'hd_col_sum')
    got = out.cpu().numpy()
    assert np.array_equal(_bits(got[:cols]), _bits(_col_sum_ref(x, rows, cols)))
    assert np.isnan(got[cols:]).all()


@pytest.mark.parametrize('D,K,N,g_ld,g_off,masked', [(1, 1024, 13, 24, 23, True), (1, 1024, 800, 24, 23, True), (72, 1024, 21, 85, 3, True),
                                                     (85, 1024, 7, 85, 0, True), (85, 1000, 9, 90, 0, False), (96, 2052, 33, 96, 0, True),
                                                     (72, 1024, 640, 72, 0, False)])
def test_fc_small_dgrad(D, K, N, g_ld, g_off, masked):
    """out[n, k] = (mask > 0) * sum_j g[n, j] Wt[j, k] against float64: D = 1 (D_pose, g[:, 23] at stride 24), 72 / 85 (the IEF fc3,
    the delta heads' g at offset 3 of rows of 85), 96; K not a multiple of 1024; rows past N are not written."""
    lib, check = _lib()
    rng = np.random.RandomState(D * 7 + K + N)
    g = rng.normal(0, 1, (N, g_ld)).astype(np.float32)
    wt = rng.normal(0, 1, (D, K)).astype(np.float32)
    mask = np.maximum(rng.normal(0, 1, (N, K)), 0).astype(np.float32) if masked else None
    out = _nan((N + 8, K))
    gt = torch.from_numpy(g).cuda()
    mt = torch.from_numpy(mask).cuda() if masked else None
    wtt = torch.from_numpy(wt).cuda()
    check(lib.hd_fc_small_dgrad(_vp(gt, 4 * g_off), g_ld, _vp(wtt), K, D, _vp(mt), _vp(out), N, _st()),
          'hd_fc_small_dgrad')
    got = out.cpu().numpy()
    assert np.isnan(got[N:]).all()
    ref = g[:, g_off:g_off + D].astype(np.float64) @ wt.astype(np.float64)
    if masked:
        ref = ref * (mask > 0)
        assert (got[:N][mask <= 0] == 0).all()
    e = _rel(got[:N], ref)
    print('fc_small_dgrad D=%d K=%d N=%d: %.2e' % (D, K, N, e))
    assert e < SMALL_BAR


@pytest.mark.parametrize('relu', [1, 0])
@pytest.mark.parametrize('with_addend', [True, False])
@pytest.mark.parametrize('B,T,Cc,groups', [(2, 7, 2048, 32), (3, 40, 96, 4), (1, 1, 200, 8), (2, 13, 192, 6), (4, 20, 2048, 32)])
def test_groupnorm_relu_backward(B, T, Cc, groups, with_addend, relu):
    """hd_groupnorm_relu_backward against float64 (the ReLU mask taken from the GPU forward), and its mask equal to the one hd_im2col_t
    recomputes from hd_groupnorm_stats: with dy = 1, dbeta_part counts the frames with relu(x*gain + offset) > 0."""
    from human_dynamics_b200.nets import GN_EPS
    lib, check = _lib()
    rng = np.random.RandomState(B * T + Cc + groups)
    x = (rng.normal(0.2, 1, (B, T, Cc)) + rng.normal(0, 0.5, (B, 1, Cc))).astype(np.float32)
    gam = rng.uniform(0.5, 1.5, Cc).astype(np.float32)
    bet = rng.normal(0, 0.5, Cc).astype(np.float32)
    dy = rng.normal(0, 1, (B, T, Cc)).astype(np.float32)
    add = rng.normal(0, 1, (B, T, Cc)).astype(np.float32) if with_addend else None
    xt, gt, bt, dyt = (torch.from_numpy(v).cuda() for v in (x, gam, bet, dy))
    at = torch.from_numpy(add).cuda() if with_addend else None
    st = _st()
    gain, offset = torch.empty((B, Cc), device='cuda'), torch.empty((B, Cc), device='cuda')
    check(lib.hd_groupnorm_stats(_vp(xt), _vp(gt), _vp(bt), _vp(gain), _vp(offset), B, T, Cc, groups, GN_EPS, st), 'hd_groupnorm_stats')
    z = torch.empty((Cc, B * T), device='cuda')
    check(lib.hd_im2col_t(_vp(xt), B, T, Cc, 1, 0, _vp(gain), _vp(offset), 1, _vp(z), B * T, B * T, st), 'hd_im2col_t')
    mask = (z.t() > 0).reshape(B, T, Cc).cpu().numpy()

    def run(dyv, addv):
        dx, pg, pb = _nan((B, T, Cc)), _nan((B, Cc)), _nan((B, Cc))
        check(lib.hd_groupnorm_relu_backward(_vp(xt), _vp(gt), _vp(bt), _vp(dyv), _vp(addv), _vp(dx), _vp(pg), _vp(pb), B, T, Cc, groups,
                                             GN_EPS, relu, st), 'hd_groupnorm_relu_backward')
        return dx.cpu().numpy(), pg.cpu().numpy(), pb.cpu().numpy()
    if relu:
        _, _, cnt = run(torch.ones_like(dyt), None)
        assert np.array_equal(cnt, mask.sum(1).astype(np.float32)), 'the backward ReLU mask is not the forward one'
    dx, pg, pb = run(dyt, at)
    cg = Cc // groups
    xd = x.astype(np.float64).reshape(B, T, groups, cg)
    mu = xd.mean((1, 3), keepdims=True)
    rstd = 1 / np.sqrt(xd.var((1, 3), keepdims=True) + GN_EPS)
    xh = ((xd - mu) * rstd).reshape(B, T, Cc)
    gp = dy.astype(np.float64) * (mask if relu else 1)
    ghat = (gp * gam).reshape(B, T, groups, cg)
    m1 = ghat.mean((1, 3), keepdims=True)
    m2 = (ghat * xh.reshape(B, T, groups, cg)).mean((1, 3), keepdims=True)
    want = (rstd * (ghat - m1 - xh.reshape(B, T, groups, cg) * m2)).reshape(B, T, Cc) + (add if with_addend else 0)
    e = (_rel(dx, want), _rel(pg, (gp * xh).sum(1)), _rel(pb, gp.sum(1)))
    print('groupnorm_relu_backward %s: dx %.2e, dgamma %.2e, dbeta %.2e' % ((B, T, Cc, groups, relu), *e))
    assert e[0] < GN_BAR and e[1] < GN_BAR and e[2] < SMALL_BAR


@pytest.mark.parametrize('alias', ['a', 'b'])
def test_add_strided_in_place(alias):
    """out = a + b bit for bit with out aliasing a (ief_head_backward's dP and gm) or b, at the strides the IEF glue uses."""
    lib, check = _lib()
    rng = np.random.RandomState(5)
    N = 37
    a = rng.normal(0, 1, (N, 85)).astype(np.float32)
    b = rng.normal(0, 1, (N, 72)).astype(np.float32)
    want = a.copy()
    want[:, 3:75] = a[:, 3:75] + b
    at, bt = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    if alias == 'a':            # gm[:, 3:] += ds: a and out the same strided view
        check(lib.hd_add_strided(_vp(at, 12), 85, _vp(bt), 72, _vp(at, 12), 85, N, 72, _st()), 'hd_add_strided')
        got = at.cpu().numpy()
    else:                       # b and out the same dense [N, 72], a strided
        check(lib.hd_add_strided(_vp(at, 12), 85, _vp(bt), 72, _vp(bt), 72, N, 72, _st()), 'hd_add_strided')
        got, want = bt.cpu().numpy(), want[:, 3:75]
    assert np.array_equal(_bits(got), _bits(want))


# ------------------------------------------------------------------------------------------------------------------------------------
# hd_ief_fc3
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('D', [1, 17, 32, 33, 64, 72, 85, 96])
@pytest.mark.parametrize('N', [1, 13])
def test_ief_fc3_against_float64(D, N):
    """out[n, :D] = prev[n, :D] + h2[n] . W + bias for every D the entry accepts, prev / out at row strides above D; the columns of out
    past D stay as they were."""
    lib, check = _lib()
    rng = np.random.RandomState(D * 10 + N)
    K = 1024
    h2 = np.maximum(rng.normal(0, 1, (N, K)), 0).astype(np.float32)
    w = (rng.normal(0, 1, (K, D)) / 32).astype(np.float32)
    bias = rng.normal(0, 1, D).astype(np.float32)
    prev = rng.normal(0, 1, (N, D + 9)).astype(np.float32)
    out = _nan((N, D + 5))
    h2t, wt, bt, pt = (torch.from_numpy(v).cuda() for v in (h2, w, bias, prev))
    check(lib.hd_ief_fc3(_vp(h2t), _vp(wt), _vp(bt), _vp(pt), D + 9, _vp(out), D + 5, N, K, D, _st()), 'hd_ief_fc3')
    got = out.cpu().numpy()
    assert np.isnan(got[:, D:]).all()
    want = prev[:, :D] + h2.astype(np.float64) @ w + bias
    e = _rel(got[:, :D], want)
    print('ief_fc3 D=%d N=%d: %.2e' % (D, N, e))
    assert e < SMALL_BAR
