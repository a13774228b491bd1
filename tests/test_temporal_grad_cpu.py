"""CPU: the float64 gradient oracle of the trainable layers (oracle/nets_grad_ref.py) against oracle/nets_ref.py and finite
differences, the GroupNorm backward formula the GPU kernel implements, the backward-data repack index map, argument checking of the
new C entries and the TemporalModel parameter names.  No GPU needed."""
import ctypes

import numpy as np
import pytest
import torch

F64 = torch.float64


def _fm_weights(C, L, seed):
    from human_dynamics_b200 import synthetic
    return synthetic.make_fmovie_weights(seed, L, C=C)


def test_grad_oracle_equals_nets_ref():
    from oracle import nets_ref, nets_grad_ref as g
    from human_dynamics_b200 import synthetic
    rng = np.random.RandomState(0)
    w = _fm_weights(64, 2, 3)
    x = rng.normal(size=(2, 5, 64))
    L = g.leaves(w, list(w))
    got = g.fmovie(torch.from_numpy(x), g.fmovie_blocks(L, 2))
    ref = nets_ref.az_fc2_groupnorm(x, w, 2, F64)
    assert (got - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()
    wi = synthetic.make_ief_weights(5, (-5, 5), feat=32)
    wi['mean_param'] = synthetic.make_mean_param()
    phi = rng.normal(size=(4, 32))
    Li = g.leaves(wi, list(wi))
    start = torch.from_numpy(np.tile(wi['mean_param'].reshape(1, 85), (4, 1)).astype(np.float64))
    th, dl = g.call_hmr_ief(torch.from_numpy(phi), start, {dt: g.ief_params(Li, dt) for dt in (0, -5, 5)}, (-5, 5))
    th_r, dl_r = nets_ref.call_hmr_ief(phi, start.numpy(), wi, 'single_view_ief', 85, 3, (0, -5, 5), True, True, F64)
    assert (th - th_r).abs().max().item() <= 1e-12 * th_r.abs().max().item()
    for k in (-5, 5):
        assert (dl[k] - dl_r[k]).abs().max().item() <= 1e-12 * dl_r[k].abs().max().item()
    wh = synthetic.make_hal_weights(6, C=32)
    xh = rng.normal(size=(3, 32))
    Lh = g.leaves(wh, list(wh))
    got = g.fc2_res(torch.from_numpy(xh), tuple(Lh['fc2_res/fc%d/%s' % (i, k)] for i in (1, 2, 3) for k in ('weights', 'biases')))
    ref = nets_ref.fc2_res(xh, wh, F64)
    assert (got - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()


@pytest.mark.parametrize('T', [1, 3])
def test_gradcheck_fmovie(T):
    """C = 64 (2 channels per group), B = 2: finite differences pin every gradient of one block (input, gamma, beta, W, b)."""
    from oracle import nets_grad_ref as g
    w = _fm_weights(64, 1, 7)
    rng = np.random.RandomState(T)
    names = sorted(w)
    L = g.leaves(w, names)
    x = torch.from_numpy(rng.normal(size=(2, T, 64))).requires_grad_()
    U = torch.from_numpy(rng.normal(size=(2, T, 64)))

    def f(x, *ps):
        L2 = dict(zip(names, ps))
        return (g.fmovie(x, g.fmovie_blocks(L2, 1)) * U).sum()
    assert torch.autograd.gradcheck(f, (x,) + tuple(L[n] for n in names), eps=1e-6, atol=1e-5, rtol=1e-4)


def test_gradcheck_small_ief_and_hal():
    from oracle import nets_grad_ref as g
    from human_dynamics_b200 import synthetic
    rng = np.random.RandomState(2)
    wi = synthetic.make_ief_weights(5, (5,), feat=8)
    # shrink the hidden width for finite differences: the oracle is width-agnostic
    for k in list(wi):
        a = wi[k]
        if k.endswith('fc1/weights'):
            wi[k] = a[:, :16]
        elif k.endswith('fc1/biases'):
            wi[k] = a[:16]
        elif k.endswith('fc2/weights'):
            wi[k] = a[:16, :16]
        elif k.endswith('fc2/biases'):
            wi[k] = a[:16]
        elif k.endswith('fc3/weights'):
            wi[k] = a[:16]
    names = sorted(wi)
    L = g.leaves(wi, names)
    phi = torch.from_numpy(rng.normal(size=(2, 8))).requires_grad_()
    start = torch.from_numpy(rng.normal(0, 0.3, size=(2, 85))).requires_grad_()
    U = [torch.from_numpy(rng.normal(size=(2, 85))) for _ in range(2)]

    def f(phi, start, *ps):
        L2 = dict(zip(names, ps))
        th, dl = g.call_hmr_ief(phi, start, {0: g.ief_params(L2, 0), 5: g.ief_params(L2, 5)}, (5,))
        return (th * U[0]).sum() + (dl[5] * U[1]).sum()
    assert torch.autograd.gradcheck(f, (phi, start) + tuple(L[n] for n in names), eps=1e-6, atol=1e-5, rtol=1e-4)
    wh = synthetic.make_hal_weights(6, C=12)
    hn = sorted(wh)
    Lh = g.leaves(wh, hn)
    x = torch.from_numpy(rng.normal(size=(3, 12))).requires_grad_()

    def fh(x, *ps):
        L2 = dict(zip(hn, ps))
        return g.fc2_res(x, tuple(L2['fc2_res/fc%d/%s' % (i, k)] for i in (1, 2, 3) for k in ('weights', 'biases'))).sum()
    assert torch.autograd.gradcheck(fh, (x,) + tuple(Lh[n] for n in hn), eps=1e-6, atol=1e-5, rtol=1e-4)


def _gn_relu_backward_numpy(x, gamma, beta, dy, groups, eps):
    """The formula hd_groupnorm_relu_backward implements, per (clip, group), in float64."""
    B, T, C = x.shape
    cg = C // groups
    xg = x.reshape(B, T, groups, cg)
    mean = xg.mean(axis=(1, 3), keepdims=True)
    var = ((xg - mean) ** 2).mean(axis=(1, 3), keepdims=True)
    rstd = 1.0 / np.sqrt(var + eps)
    xh = (xg - mean) * rstd
    gm, bt = gamma.reshape(1, 1, groups, cg), beta.reshape(1, 1, groups, cg)
    z = xh * gm + bt
    gp = dy.reshape(B, T, groups, cg) * (z > 0)
    gh = gp * gm
    n = T * cg
    dx = rstd * (gh - gh.sum(axis=(1, 3), keepdims=True) / n - xh * (gh * xh).sum(axis=(1, 3), keepdims=True) / n)
    return dx.reshape(B, T, C), (gp * xh).sum(axis=(0, 1)).reshape(C), gp.sum(axis=(0, 1)).reshape(C)


def test_groupnorm_backward_formula_equals_autograd():
    from oracle.nets_ref import group_norm_tf
    rng = np.random.RandomState(4)
    for (B, T, C) in ((2, 1, 64), (3, 7, 64), (2, 4, 128)):
        x, dy = rng.normal(size=(B, T, C)), rng.normal(size=(B, T, C))
        gamma, beta = rng.uniform(0.5, 1.5, size=C), rng.normal(0, 0.3, size=C)
        xt = torch.from_numpy(x).requires_grad_()
        gt, bt = torch.from_numpy(gamma).requires_grad_(), torch.from_numpy(beta).requires_grad_()
        y = torch.relu(group_norm_tf(xt[:, :, None, :], gt, bt))[:, :, 0, :]
        ref = torch.autograd.grad(y, (xt, gt, bt), torch.from_numpy(dy))
        got = _gn_relu_backward_numpy(x, gamma, beta, dy, 32, 1e-6)
        for a, b in zip(got, ref):
            assert np.abs(a - b.numpy()).max() <= 1e-10 * max(1.0, np.abs(b.numpy()).max())


def _pack_bwd_data_numpy(w):
    """The index map of hd_pack_weight(HD_PACK_BACKWARD_DATA): dst[ci, k'*Cout + co] = W[KH-1-k', ci, co]."""
    KH, Cin, Cout = w.shape
    dst = np.zeros((Cin, KH * Cout))
    for kp in range(KH):
        dst[:, kp * Cout:(kp + 1) * Cout] = w[KH - 1 - kp]
    return dst


def test_backward_data_repack_is_the_adjoint():
    """<conv(x, W), y> = <x, conv(y, W')> in float64, SAME padding over T, with W' rebuilt from the packed K-major matrix."""
    from oracle.nets_ref import conv2d_nhwc
    rng = np.random.RandomState(5)
    for (B, T, Cin, Cout, KH) in ((2, 5, 6, 4, 3), (1, 1, 3, 5, 3), (3, 4, 7, 2, 1)):
        w = rng.normal(size=(KH, Cin, Cout))
        x, y = rng.normal(size=(B, T, 1, Cin)), rng.normal(size=(B, T, 1, Cout))
        packed = _pack_bwd_data_numpy(w)                                    # [Cin, KH*Cout]: row = output channel of the dX conv
        wp = packed.reshape(Cin, KH, Cout).transpose(1, 2, 0)[:, None]      # back to HWIO [KH, 1, Cout, Cin]
        lhs = (conv2d_nhwc(torch.from_numpy(x), torch.from_numpy(w[:, None])) * torch.from_numpy(y)).sum()
        rhs = (torch.from_numpy(x) * conv2d_nhwc(torch.from_numpy(y), torch.from_numpy(np.ascontiguousarray(wp)))).sum()
        assert abs(lhs.item() - rhs.item()) <= 1e-12 * max(1.0, abs(lhs.item()))


def test_new_entries_reject_bad_arguments_without_launch():
    from human_dynamics_b200 import _lib
    lib = _lib.lib
    lib.hd_launch_count_reset()
    assert lib.hd_pack_weight(None, 3, 64, 64, 0, 2, None, None, 64, 192, None) == 1
    buf = ctypes.c_void_p(16)                         # never dereferenced: the checks fail first
    assert lib.hd_pack_weight(buf, 3, 64, 64, 0, 2, buf, buf, 60, 192, None) == 1          # rows % 64
    assert lib.hd_pack_weight(buf, 3, 64, 64, 1, 4, buf, buf, 64, 100, None) == 1          # k_pad % 32
    assert lib.hd_pack_weight(buf, 3, 64, 128, 0, 2, buf, buf, 64, 192, None) == 1         # rows < Cout
    assert lib.hd_pack_weight(buf, 3, 64, 64, 2, 2, buf, buf, 64, 192, None) == 1          # mode
    assert lib.hd_transpose_split(buf, 10, 4, 4, 0, buf, buf, 32, 4, 32, None) == 1         # mode 0 with lo
    assert lib.hd_transpose_split(buf, 10, 4, 4, 1, buf, buf, 32, 4, 8, None) == 1          # out_cols < rows
    assert lib.hd_im2col_t(buf, 2, 3, 64, 3, 3, None, None, 0, buf, 32, 32, None) == 1      # pad >= KH
    assert lib.hd_im2col_t(buf, 2, 3, 64, 3, 1, buf, None, 1, buf, 32, 32, None) == 1       # gain without offset
    assert lib.hd_groupnorm_relu_backward(buf, buf, buf, buf, None, buf, buf, buf, 2, 3, 64, 32, 1e-6, 1, None) == 1   # dx aliases x
    assert lib.hd_groupnorm_relu_backward(buf, buf, buf, ctypes.c_void_p(32), None, ctypes.c_void_p(48), buf, buf, 2, 3, 66, 32,
                                          1e-6, 1, None) == 1                                # C % groups
    assert lib.hd_col_sum(buf, 4, 8, 4, buf, None) == 1                                      # ld < cols
    assert lib.hd_relu_backward(None, buf, buf, 4, None) == 1
    assert lib.hd_fc_small_dgrad(buf, 85, buf, 1024, 97, None, buf, 4, None) == 1           # D > 96
    assert lib.hd_add_strided(buf, 2, buf, 4, buf, 4, 3, 4, None) == 1                       # lda < cols
    assert b'hd_add_strided' in lib.hd_last_error()
    assert lib.hd_launch_count() == 0
    assert lib.hd_version() >= 103


def test_trainable_names_are_the_engine_keys(weights):
    """TemporalModel holds exactly the f_movie / IEF / mean_param / fc2_res variables HMMREngine's packers read."""
    from human_dynamics_b200.trainable import trainable_names
    names = trainable_names(weights)
    assert len(names) == len(set(names))
    assert set(names) <= set(weights)
    want = {k for k in weights if k.startswith(('AZ_FC_', 'single_view_ief', 'fc2_res/'))} | {'mean_param'}
    assert set(names) == want
    nohal = {k: v for k, v in weights.items() if not k.startswith('fc2_res/')}
    assert not any(n.startswith('fc2_res/') for n in trainable_names(nohal))
