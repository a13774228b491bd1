"""Training surface of the temporal model: f_movie ("az_fc2_groupnorm"), the IEF heads (main + delta), `mean_param` and the fc2_res
hallucinator as torch parameters, differentiable on the GPU.

This is what the reference trains in its default configuration (freeze_phi=True, precomputed_phi=True: src/config.py): everything
after the ResNet.  The model packs its parameters in place with the inference engine's packs (nets.PackedFMovie, PackedIEF, PackedHal)
and each forward runs the inference plans over them (nets.FMoviePlan and IEFPlan with keep=True, which hold what the backward reads, and
PackedHal.run), so its outputs are bit-identical to HMMREngine's; the weights are packed on the device (hd_pack_weight) and repacked
before a forward whenever a parameter was changed in place (optimizer.step()).  The backward (csrc/net_grad.cu + hd_conv_gemm in its
3xTF32 mode, or 1xTF32 with TrainConfig.grad_precision='tf32') is first-order, deterministic and follows the inference graph: dropout is the identity (is_training=False)
unless a call asks for the reference's training-mode IEF dropout explicitly (`regress(..., dropout=(seed, step, call, keep_prob))`).

All arithmetic goes through libhd_b200.so; torch provides buffers, streams and the autograd plumbing.  The user's loss and optimizer
are ordinary torch code:

    model = TemporalModel(weights)                     # anything engine.load_weights accepts
    opt = torch.optim.Adam(model.parameters(), 1e-5)
    out = model.predict_from_features(phi, smpl)       # phi (B,T,2048), smpl = src.tf_smpl.batch_smpl.SMPL
    loss = keypoint_loss(out['kps'], gt)               # any torch expression
    loss.backward(); opt.step(); opt.zero_grad()
    model.save_checkpoint('/path/model.ckpt-1000')     # HMMREngine / Tester load it unchanged
"""
from __future__ import annotations

import ctypes as C
import types

import numpy as np
import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import _lib
from ._lib import lib, check, fptr, current_stream
from .nets import (GN_EPS, GN_GROUPS, BackwardDataPack, FMoviePlan, IEFPlan, PackedFMovie, PackedHal, PackedIEF, dgrad_op, grad_one_pass,
                   require_training_impl, sync_packing, weight_tmap)

F32 = torch.float32


def _vp(t, off=0):
    return C.c_void_p(t.data_ptr() + off)


def _round(x, m):
    return (x + m - 1) // m * m


class TransposedCopy(object):
    """dst = src^T in fp32 on the device (src [rows, cols] row-major, dst [cols, rows]): a small layer's input-gradient operand."""

    def __init__(self, src, dst):
        self.src, self.dst = src, dst

    def repack(self, stream):
        src, dst = self.src, self.dst
        check(lib.hd_transpose_split(fptr(src), src.shape[0], src.shape[1], src.shape[1], 0, _vp(dst), None, dst.shape[1], dst.shape[0],
                                     dst.shape[1], stream), 'hd_transpose_split')


def _bt_operand(pieces, cols, k_pad, st, one_pass=False):
    """B operand of a weight-gradient GEMM, with a BackwardDataPack's fields for dgrad_op: the row blocks `pieces` = [(x, rows, ld)]
    of an upstream gradient stacked along K, transposed and TF32-split into w_nk_hi / w_nk_lo [roundup64(cols), k_pad] (zero past the
    real rows / columns).  one_pass: the round-to-nearest TF32 head alone (w_nk_lo and tmap_lo are None)."""
    rows = _round(cols, 64)
    hi = torch.empty((rows, k_pad), dtype=F32, device=pieces[0][0].device)
    lo = None if one_pass else torch.empty_like(hi)
    _stack_t(pieces, cols, k_pad, 1, hi, lo, rows, st)
    return types.SimpleNamespace(w_nk_hi=hi, w_nk_lo=lo, tmap_hi=weight_tmap(hi), tmap_lo=None if one_pass else weight_tmap(lo),
                                 Cout=cols, K=k_pad)


def _stack_t(pieces, cols, k_pad, mode, hi, lo, out_rows, st):
    off = 0
    for i, (x, n, ld) in enumerate(pieces):
        last = i == len(pieces) - 1
        check(lib.hd_transpose_split(fptr(x), n, cols, ld, mode, _vp(hi, off * 4), _vp(lo, off * 4) if lo is not None else None, k_pad,
                                     out_rows, (k_pad - off) if last else n, st), 'hd_transpose_split')
        off += n


def _xt(pieces, cols, k_pad, st):
    """A operand of a weight-gradient GEMM for an FC layer: input rows stacked along K, transposed to [cols, k_pad] fp32."""
    out = torch.empty((cols, k_pad), dtype=F32, device=pieces[0][0].device)
    _stack_t(pieces, cols, k_pad, 0, out, None, cols, st)
    return out


def _col_sum(x, rows, cols, ld, out, st):
    check(lib.hd_col_sum(fptr(x), rows, cols, ld, fptr(out), st), 'hd_col_sum')


def _wgrad(xt, M, k_pad, g_pieces, cols, out, st, one_pass=False):
    """out[M, cols] = xt . (stacked g) : the weight gradient, 3xTF32 (one_pass: 1xTF32)."""
    dgrad_op(_bt_operand(g_pieces, cols, k_pad, st, one_pass), xt, M, 1, 1, 1, 1, out, one_pass=one_pass).run(st)


# ------------------------------------------------------------------------------------------------------------------------------------
# f_movie
# ------------------------------------------------------------------------------------------------------------------------------------
def fmovie_backward(model, saved, g):
    """Gradients of f_movie: returns (dx, [per block: dgamma1, dbeta1, dW1, db1, dgamma2, dbeta2, dW2, db2])."""
    st = current_stream()
    B, T, Cc = g.shape
    BT = B * T
    kp = _round(BT, 32)
    dev = g.device
    xt = torch.empty((3 * Cc, kp), dtype=F32, device=dev)
    gain, offset = torch.empty((B, Cc), dtype=F32, device=dev), torch.empty((B, Cc), dtype=F32, device=dev)
    pg, pb = torch.empty((B, Cc), dtype=F32, device=dev), torch.empty((B, Cc), dtype=F32, device=dev)
    dact = torch.empty((B, T, Cc), dtype=F32, device=dev)
    blocks = model.fmovie.blocks
    grads = [None] * len(blocks)
    g = g.contiguous()
    for i in range(len(blocks) - 1, -1, -1):
        blk = blocks[i]
        x, mid = saved[i]
        gr = {}
        dmid = torch.empty((B, T, Cc), dtype=F32, device=dev)
        dx = torch.empty((B, T, Cc), dtype=F32, device=dev)
        for k, src, gin, gout, addend in ((2, mid, g, dmid, None), (1, x, dmid, dx, g)):
            gam, bet = blk['gn%d' % k]
            # dW = im2col(relu(gn(src)))^T . gin, db = colsum(gin)
            check(lib.hd_groupnorm_stats(fptr(src), fptr(gam), fptr(bet), fptr(gain), fptr(offset), B, T, Cc, GN_GROUPS, GN_EPS, st),
                  'hd_groupnorm_stats')
            check(lib.hd_im2col_t(fptr(src), B, T, Cc, 3, 1, fptr(gain), fptr(offset), 1, fptr(xt), kp, kp, st), 'hd_im2col_t')
            dW = torch.empty((3, 1, Cc, Cc), dtype=F32, device=dev)
            _wgrad(xt, 3 * Cc, kp, [(gin, BT, Cc)], Cc, dW, st, model.one_pass)
            db = torch.empty(Cc, dtype=F32, device=dev)
            _col_sum(gin, BT, Cc, Cc, db, st)
            # d relu(gn(src)) = conv(gin, W'); then the GroupNorm + ReLU backward (+ the block's residual gradient for gn1)
            dgrad_op(blk['conv%d' % k].bwd, gin, B, T, 1, 3, 1, dact, one_pass=model.one_pass).run(st)
            check(lib.hd_groupnorm_relu_backward(fptr(src), fptr(gam), fptr(bet), fptr(dact), fptr(addend) if addend is not None else None,
                                                 fptr(gout), fptr(pg), fptr(pb), B, T, Cc, GN_GROUPS, GN_EPS, 1, st),
                  'hd_groupnorm_relu_backward')
            dg, dbe = torch.empty(Cc, dtype=F32, device=dev), torch.empty(Cc, dtype=F32, device=dev)
            _col_sum(pg, B, Cc, Cc, dg, st)
            _col_sum(pb, B, Cc, Cc, dbe, st)
            gr[k] = (dg, dbe, dW, db)
        grads[i] = list(gr[1]) + list(gr[2])
        g = dx
    return g, grads


# ------------------------------------------------------------------------------------------------------------------------------------
# IEF heads
# ------------------------------------------------------------------------------------------------------------------------------------
def ief_head_backward(model, head, phi, N, saved, g, g_ld, dphi, st, p=None):
    """Backward of one hmr_ief head.  saved = (h1, h2, start, start_ld, stage-0 output, stage-1 output); g: gradient of the head's
    output (rows of d at stride g_ld).  Accumulates dL/dphi into `dphi`
    (None: written).  p: nn.dropout's float32 keep_prob when the forward ran the IEF dropout (h1 / h2 are then the masked
    activations, so h > 0 <=> kept and positive, and a kept element's gradient is divided by p), None for the identity.
    Returns (dstart [N, d], [dW1, db1, dW2, db2, dW3, db3], dphi)."""
    dev = phi.device
    d, feat = head.d, head.feat
    h1, h2, start, start_ld, mid0, mid1 = saved
    ins = [(start, start_ld), (mid0, d), (mid1, d)]
    G = torch.empty((3, N, d), dtype=F32, device=dev)
    DP2 = torch.empty((3, N, 1024), dtype=F32, device=dev)
    DP1 = torch.empty((3, N, 1024), dtype=F32, device=dev)
    dstart = torch.empty((N, d), dtype=F32, device=dev)
    for s in range(2, -1, -1):
        gs, gld = (g, g_ld) if s == 2 else (G[s], d)
        if s == 2:
            G[2].copy_(torch.as_strided(g, (N, d), (g_ld, 1)))
        # dpre2 = (g . W3^T) * (h2 > 0);  dpre1 = (dpre2 . W2^T) * (h1 > 0);  dprev = g + dpre1 . W1theta^T
        if p is None:
            check(lib.hd_fc_small_dgrad(fptr(gs), gld, fptr(head.fc3.bwd.dst), 1024, d, fptr(h2[s]), fptr(DP2[s]), N, st),
                  'hd_fc_small_dgrad')
        else:
            check(lib.hd_fc_small_dgrad_dropout(fptr(gs), gld, fptr(head.fc3.bwd.dst), 1024, d, fptr(h2[s]), p, fptr(DP2[s]), N, st),
                  'hd_fc_small_dgrad_dropout')
        dgrad_op(head.fc2.bwd, DP2[s], N, 1, 1, 1, 1, DP1[s], one_pass=model.one_pass).run(st)
        if p is None:
            check(lib.hd_relu_backward(fptr(h1[s]), fptr(DP1[s]), fptr(DP1[s]), N * 1024, st), 'hd_relu_backward')
        else:
            check(lib.hd_relu_dropout_backward(fptr(h1[s]), fptr(DP1[s]), fptr(DP1[s]), N * 1024, p, st), 'hd_relu_dropout_backward')
        dst = G[s - 1] if s > 0 else dstart
        check(lib.hd_ief_fc3(fptr(DP1[s]), fptr(head.fc1_theta.bwd.dst), fptr(model._zeros), fptr(gs), gld, fptr(dst), d, N, 1024, d, st),
              'hd_ief_fc3')
    kp3, kp1 = _round(3 * N, 32), _round(N, 32)
    W1, W2, W3 = (torch.empty(shape, dtype=F32, device=dev) for shape in ((feat + d, 1024), (1024, 1024), (1024, d)))
    b1, b2, b3 = (torch.empty(n, dtype=F32, device=dev) for n in (1024, 1024, d))
    # dP = sum over the stages (fixed order), then the phi part of fc1
    dP = torch.empty((N, 1024), dtype=F32, device=dev)
    check(lib.hd_add_strided(fptr(DP1[0]), 1024, fptr(DP1[1]), 1024, fptr(dP), 1024, N, 1024, st), 'hd_add_strided')
    check(lib.hd_add_strided(fptr(dP), 1024, fptr(DP1[2]), 1024, fptr(dP), 1024, N, 1024, st), 'hd_add_strided')
    _col_sum(dP, N, 1024, 1024, b1, st)
    _col_sum(DP2, 3 * N, 1024, 1024, b2, st)
    _col_sum(G, 3 * N, d, d, b3, st)
    op = model.one_pass
    _wgrad(_xt([(phi, N, feat)], feat, kp1, st), feat, kp1, [(dP, N, 1024)], 1024, W1, st, op)
    _wgrad(_xt([(t, N, ld) for t, ld in ins], d, kp3, st), d, kp3, [(DP1.view(3 * N, 1024), 3 * N, 1024)], 1024, W1[feat:], st, op)
    _wgrad(_xt([(h1.view(3 * N, 1024), 3 * N, 1024)], 1024, kp3, st), 1024, kp3, [(DP2.view(3 * N, 1024), 3 * N, 1024)], 1024, W2, st, op)
    _wgrad(_xt([(h2.view(3 * N, 1024), 3 * N, 1024)], 1024, kp3, st), 1024, kp3, [(G.view(3 * N, d), 3 * N, d)], d, W3, st, op)
    out = torch.empty((N, feat), dtype=F32, device=dev) if dphi is None else dphi
    dgrad_op(head.fc1_phi.bwd, dP, N, 1, 1, 1, 1, out, res=dphi, one_pass=op).run(st)
    return dstart, [W1, b1, W2, b2, W3, b3], out


def regress_plan(model, keys, tiled, phi, start, dropout=None):
    """call_hmr_ief over phi (N,2048) from start (N,85), or the tiled (1,85) when `tiled`, through a keep=True IEFPlan built for this
    call (with its `dropout`): the main head, then the delta heads `keys` from its pose.  Returns ((theta, deltas...), the start rows
    (N,85), the plan)."""
    N = phi.shape[0]
    s0 = start.expand(N, 85).contiguous() if tiled else start
    plan = IEFPlan(model.ief, N, 3, list(keys), keep=True, dropout=dropout)
    theta, deltas = plan.run(phi, s0)
    return (theta,) + tuple(deltas[k] for k in keys), s0, plan


# ------------------------------------------------------------------------------------------------------------------------------------
# fc2_res
# ------------------------------------------------------------------------------------------------------------------------------------
def hal_backward(model, x, h1, h2, g):
    N = x.shape[0]
    st = current_stream()
    dev = x.device
    kp = _round(N, 32)
    L = model.hal
    grads = []
    dh2, dh1, dx = (torch.empty((N, 2048), dtype=F32, device=dev) for _ in range(3))
    for inp, gin, name in ((h2, g, 'fc3'), (h1, dh2, 'fc2'), (x, dh1, 'fc1')):
        W, b = torch.empty((2048, 2048), dtype=F32, device=dev), torch.empty(2048, dtype=F32, device=dev)
        _wgrad(_xt([(inp, N, 2048)], 2048, kp, st), 2048, kp, [(gin, N, 2048)], 2048, W, st, model.one_pass)
        _col_sum(gin, N, 2048, 2048, b, st)
        grads = [W, b] + grads
        if name == 'fc3':
            dgrad_op(L.fc3.bwd, g, N, 1, 1, 1, 1, dh2, one_pass=model.one_pass).run(st)
            check(lib.hd_relu_backward(fptr(h2), fptr(dh2), fptr(dh2), N * 2048, st), 'hd_relu_backward')
        elif name == 'fc2':
            dgrad_op(L.fc2.bwd, dh2, N, 1, 1, 1, 1, dh1, one_pass=model.one_pass).run(st)
            check(lib.hd_relu_backward(fptr(h1), fptr(dh1), fptr(dh1), N * 2048, st), 'hd_relu_backward')
        else:
            dgrad_op(L.fc1.bwd, dh1, N, 1, 1, 1, 1, dx, res=g, one_pass=model.one_pass).run(st)
    return dx, grads


# ------------------------------------------------------------------------------------------------------------------------------------
# autograd
# ------------------------------------------------------------------------------------------------------------------------------------
class FMovieFunction(torch.autograd.Function):
    """phi (B,T,C) -> f_movie(phi); differentiable w.r.t. phi and every block's gamma / beta / weights / biases."""

    @staticmethod
    def forward(ctx, model, x, *params):
        plan = FMoviePlan(model.fmovie, x.shape[0], x.shape[1], keep=True)
        out = plan.run(x)
        ctx.model = model
        ctx.save_for_backward(*[t for pair in plan.saved for t in pair])
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        ctx.model.sync_bwd_packs()
        t = ctx.saved_tensors
        dx, grads = fmovie_backward(ctx.model, [(t[2 * i], t[2 * i + 1]) for i in range(len(t) // 2)], g)
        return (None, dx) + tuple(t for blk in grads for t in blk)


class RegressFunction(torch.autograd.Function):
    """call_hmr_ief as Tester wires it: phi (N,2048), start (N,85) or the tiled mean_param (1,85) -> (theta (N,85), deltas (N,85)...).
    The delta heads start from theta's pose and carry its beta, so their gradients flow back into the main head; a tiled start's
    gradient is its column sum.  dropout: IEFPlan's; the backward reads the masked activations the plan saved and the keep_prob."""

    @staticmethod
    def forward(ctx, model, keys, tiled, dropout, phi, start, *params):
        outs, s0, plan = regress_plan(model, keys, tiled, phi, start, dropout)
        # Everything the backward reads goes through save_for_backward (theta, an output, included): no tensor or view of one is held on
        # ctx, so an unused graph is freed with its outputs and retain_graph works.  The delta heads' start is theta's pose, rebuilt there.
        ctx.model, ctx.keys, ctx.tiled, ctx.p = model, keys, tiled, plan.dropout_p
        ctx.save_for_backward(phi, outs[0], s0, *[t for head in plan.saved for t in head])
        ctx.set_materialize_grads(False)
        return outs

    @staticmethod
    @once_differentiable
    def backward(ctx, dtheta, *ddeltas):
        model, keys = ctx.model, ctx.keys
        model.sync_bwd_packs()
        t = ctx.saved_tensors
        phi, theta, s0 = t[:3]
        N = phi.shape[0]
        pose = torch.as_strided(theta, (N, 72), (85, 1), theta.storage_offset() + 3)
        heads = [t[3 + 4 * j:7 + 4 * j] for j in range(1 + len(keys))]
        state = [(h1, h2, s0 if j == 0 else pose, 85, m0, m1) for j, (h1, h2, m0, m1) in enumerate(heads)]
        st = current_stream()
        dev = phi.device
        # gradient reaching the main head's output: its own upstream + each delta head's start (pose) and carried beta, ascending dt
        gm = torch.zeros((N, 85), dtype=F32, device=dev) if dtheta is None else dtheta.contiguous().clone()
        dphi = None
        head_grads = {}
        for i, k in enumerate(keys):
            dd = ddeltas[i]
            if dd is None:
                continue
            dd = dd.contiguous()
            ds, hg, dphi = ief_head_backward(model, model.ief.deltas[k], phi, N, state[1 + i],
                                             torch.as_strided(dd, (N, 72), (85, 1), dd.storage_offset() + 3), 85, dphi, st, ctx.p)
            head_grads[k] = hg
            check(lib.hd_add_strided(fptr(gm[:, 3:]), 85, fptr(ds), 72, fptr(gm[:, 3:]), 85, N, 72, st), 'hd_add_strided')
            check(lib.hd_add_strided(fptr(gm[:, 75:]), 85, fptr(dd[:, 75:]), 85, fptr(gm[:, 75:]), 85, N, 10, st), 'hd_add_strided')
        dstart, hg, dphi = ief_head_backward(model, model.ief.main, phi, N, state[0], gm, 85, dphi, st, ctx.p)
        head_grads['main'] = hg
        if ctx.tiled:
            ds = torch.empty((1, 85), dtype=F32, device=dev)
            _col_sum(dstart, N, 85, 85, ds, st)
            dstart = ds
        flat = []
        for k in ['main'] + list(keys):
            flat += head_grads.get(k, [None] * 6)
        return (None, None, None, None, dphi, dstart) + tuple(flat)


class HalFunction(torch.autograd.Function):
    """fc2_res: x (N,2048) -> x + fc3(relu(fc2(relu(fc1(x)))))."""

    @staticmethod
    def forward(ctx, model, x, *params):
        h1, h2, out = (torch.empty_like(x) for _ in range(3))
        model.hal.run(x, h1, h2, out)
        ctx.model = model
        ctx.save_for_backward(x, h1, h2)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        ctx.model.sync_bwd_packs()
        x, h1, h2 = ctx.saved_tensors
        dx, grads = hal_backward(ctx.model, x, h1, h2, g.contiguous())
        return (None, dx) + tuple(grads)


# ------------------------------------------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------------------------------------------
def fmovie_names(i):
    name = 'block_%d' % i
    return ['AZ_FC_block_preact_gn1%s/gamma' % name, 'AZ_FC_block_preact_gn1%s/beta' % name,
            'AZ_FC_block2_conv1%s/weights' % name, 'AZ_FC_block2_conv1%s/biases' % name,
            'AZ_FC_block_preact_gn2%s/gamma' % name, 'AZ_FC_block_preact_gn2%s/beta' % name,
            'AZ_FC_block2_conv2%s/weights' % name, 'AZ_FC_block2_conv2%s/biases' % name]


def ief_scope(dt, scope='single_view_ief'):
    return scope if dt == 0 else scope + ('_future%d' % dt if dt > 0 else '_past%d' % abs(dt))


def ief_names(dt):
    q = ief_scope(dt) + '/3D_module'
    return [q + '/fc%d/%s' % (i, k) for i in (1, 2, 3) for k in ('weights', 'biases')]


HAL_NAMES = ['fc2_res/fc%d/%s' % (i, k) for i in (1, 2, 3) for k in ('weights', 'biases')]


def trainable_names(w, num_conv_layers=3, delta_t_values=(-5, 5)):
    """TF variable names TemporalModel holds for a weight dict: exactly the f_movie / IEF / mean_param / fc2_res keys HMMREngine reads."""
    names = []
    if any(k.startswith('AZ_FC_block2_conv1') for k in w):
        for i in range(num_conv_layers):
            names += fmovie_names(i)
    for dt in [0] + sorted(int(d) for d in delta_t_values if int(d) != 0):
        names += ief_names(dt)
    names.append('mean_param')
    if 'fc2_res/fc1/weights' in w:
        names += HAL_NAMES
    return names


class TrainableModule(nn.Module):
    """fp32 parameters addressable by TF variable name (`param(name)`), and the device packs that read them in place, as (name, pack)
    pairs: `_fwd_packs` are written by their constructors, `_bwd_packs` by the first backward.  A pack is rewritten on the current
    stream when its parameter was changed in place (optimizer.step(), copy_), detected by the parameter's version counter."""

    def __init__(self):
        super().__init__()
        self._params = nn.ParameterDict()
        self._fwd_packs, self._bwd_packs = [], []
        self._seen, self._bwd_seen = {}, {}

    def param(self, name):
        return self._params[name]

    def _packs_written(self, device):
        """Wait for the packing the constructors of `_fwd_packs` queued on `device`, and record their parameters' versions: from here on
        only what changes is repacked."""
        sync_packing(device)
        self._seen = {n: self.param(n)._version for n, _ in self._fwd_packs}

    def _repack(self, packs, seen):
        st = current_stream()
        stale = {n for n, _ in packs if seen.get(n) != self.param(n)._version}
        for n, pk in packs:
            if n in stale:
                pk.repack(st)
        for n in stale:
            seen[n] = self.param(n)._version
        return len(stale)

    def sync_packs(self):
        """Repack every forward weight whose parameter changed since it was last packed (called by each forward).  Returns the count."""
        return self._repack(self._fwd_packs, self._seen)

    def sync_bwd_packs(self):
        """The same for the backward packs (called by each backward; the first one writes them all).  Returns the count."""
        return self._repack(self._bwd_packs, self._bwd_seen)

    def _grad_on(self, names, *inputs):
        """Whether a forward goes on the autograd graph: grad mode is on and an input or a parameter of `names` requires grad."""
        return torch.is_grad_enabled() and (any(x.requires_grad for x in inputs) or any(self.param(n).requires_grad for n in names))


class TemporalModel(TrainableModule):
    """The trainable part of HMMR (f_movie, the IEF heads, mean_param, fc2_res) as fp32 parameters on one CUDA device.

    Parameters are addressable by their TF variable names (`model.param('single_view_ief/3D_module/fc2/weights')`); `parameters()`
    feeds any torch optimizer.  A parameter changed in place (optimizer.step(), copy_) is repacked on the device before the next
    forward (detected by its version counter).  Under torch.no_grad(), or when nothing requires grad, the methods run the inference
    kernels and build no graph.

    The forward is HMMREngine's in its default configuration (impl 'auto'): the engine's packs (PackedFMovie, PackedIEF, PackedHal) over
    the parameters, run by FMoviePlan and IEFPlan built per call with keep=True (they keep the activations the backward reads) and by
    PackedHal.run, so it is bit-identical to the engine at every T.

    The backward's GEMMs follow `config.grad_precision` when the config has one (objective.TrainConfig): 'fp32' (3xTF32, the default)
    or 'tf32' (1xTF32, nets.GRAD_PRECISIONS)."""

    def __init__(self, weights, config=None, device=None):
        super().__init__()
        from .config import HMMRConfig
        from .engine import load_weights
        self.config = config or HMMRConfig()
        require_training_impl(self.config.impl, 'TemporalModel')
        self.one_pass = grad_one_pass(getattr(self.config, 'grad_precision', 'fp32'), 'TemporalModel')
        if not torch.cuda.is_available():
            raise _lib.HDError('TemporalModel needs a CUDA device: the hot path has no CPU fallback')
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        w = load_weights(weights)
        self._source = w                                       # frozen variables (the ResNet) for tf_variables / save_checkpoint
        self.num_conv_layers = int(self.config.num_conv_layers)
        self.delta_keys = sorted(int(d) for d in self.config.delta_t_values if int(d) != 0)
        self.names = trainable_names(w, self.num_conv_layers, self.delta_keys)
        for n in self.names:
            a = np.asarray(w[n], np.float32)
            if n == 'mean_param':
                a = a.reshape(1, 85)
            self._params[n] = nn.Parameter(torch.from_numpy(np.ascontiguousarray(a)).to(self.device))
        with torch.cuda.device(self.device):
            self._build()

    # ---------------------------------------------------------------- packing
    def _build(self):
        """The engine's packs over the parameters, read in place, each layer with its input-gradient operand `bwd` beside it."""
        w = {n: self.param(n).data for n in self.names}
        f32 = dict(dtype=F32, device=self.device)
        self.fmovie = PackedFMovie(w, self.device, self.num_conv_layers, tc='auto') if 'AZ_FC_block2_conv1block_0/weights' in w else None
        self.ief = PackedIEF(w, self.device, delta_t_values=self.delta_keys, tc='auto')
        self.hal = PackedHal(w, self.device, tc='auto') if 'fc2_res/fc1/weights' in w else None

        def layer(name, conv):                                 # a PackedConv whose input gradient is a BackwardDataPack
            conv.bwd = BackwardDataPack(conv.w_kn, conv.KH, conv.Cin, conv.Cout)
            self._fwd_packs.append((name, conv))
            self._bwd_packs.append((name, conv.bwd))
        for i, blk in enumerate(self.fmovie.blocks if self.fmovie is not None else []):
            layer(fmovie_names(i)[2], blk['conv1'])
            layer(fmovie_names(i)[6], blk['conv2'])
        for dt in [0] + self.delta_keys:
            n = ief_names(dt)
            h = self.ief.main if dt == 0 else self.ief.deltas[dt]
            layer(n[0], h.fc1_phi)
            layer(n[2], h.fc2)
            h.fc3.bwd = TransposedCopy(h.fc3.w_kn, torch.empty((h.d, 1024), **f32))                  # fc3^T  (input gradient of fc3)
            h.fc1_theta.bwd = TransposedCopy(h.fc1_theta.w_kn, torch.empty((1024, h.d), **f32))      # fc1's theta rows, transposed
            self._fwd_packs.append((n[4], h.fc3))
            self._bwd_packs += [(n[4], h.fc3.bwd), (n[0], h.fc1_theta.bwd)]
        if self.hal is not None:
            for i in (1, 2, 3):
                layer(HAL_NAMES[2 * i - 2], getattr(self.hal, 'fc%d' % i))
        self._zeros = torch.zeros(96, **f32)
        self._packs_written(self.device)

    # ---------------------------------------------------------------- forward API
    def _check_input(self, x, name, last=2048):
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise _lib.HDError('%s: a CUDA tensor is required (no CPU fallback exists)' % name)
        if x.dtype != F32 or x.shape[-1] != last:
            raise _lib.HDError('%s: expected float32 [..., %d], got %s %s' % (name, last, x.dtype, tuple(x.shape)))
        if x.device != self.device:
            raise _lib.HDError('%s: tensor is on %s, the model on %s' % (name, x.device, self.device))

    def temporal_encode(self, phi):
        """az_fc2_groupnorm ("f_movie"): (B,T,2048) -> (B,T,2048)."""
        self._check_input(phi, 'temporal_encode')
        if self.fmovie is None:
            raise _lib.HDError('no f_movie weights were loaded')
        self.sync_packs()
        phi = phi.contiguous()
        names = [n for i in range(self.num_conv_layers) for n in fmovie_names(i)]
        if self._grad_on(names, phi):
            return FMovieFunction.apply(self, phi, *[self.param(n) for n in names])
        with torch.no_grad():
            return FMoviePlan(self.fmovie, phi.shape[0], phi.shape[1]).run(phi.detach())

    def hallucinate(self, phi):
        """fc2_res: (B,T,2048) -> (B,T,2048)   (pred_mode='hal')."""
        self._check_input(phi, 'hallucinate')
        if self.hal is None:
            raise _lib.HDError('no fc2_res weights were loaded')
        self.sync_packs()
        x = phi.contiguous().reshape(-1, 2048)
        if self._grad_on(HAL_NAMES, x):
            return HalFunction.apply(self, x, *[self.param(n) for n in HAL_NAMES]).view(phi.shape)
        with torch.no_grad():
            x = x.detach()
            return self.hal.run(x, torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)).view(phi.shape)

    def regress(self, feats, omega_start=None, delta_keys=None, dropout=None):
        """call_hmr_ief: feats (N,2048) -> (omega (N,85), {dt: (N,85)}).  Starts from mean_param (tiled) unless omega_start (N,85) is
        given; the delta heads start from the main prediction (use_delta_from_pred=True, use_optcam=True, as Tester wires them).

        dropout=(seed, step, call, keep_prob): the reference's training-mode IEF (is_training=True): slim.dropout(keep_prob) after the
        ReLU of fc1 and fc2 at every stage of every head, forward and backward, with masks that are a function of (seed, step, call,
        head, stage, layer, row, column) alone (nets.IEFPlan, csrc/dropout.cuh).  call 0 = the pred strips, 1 = the hal strips.
        None (the default) or keep_prob 1: the inference graph.  Dropout is never implied by `training` or by grad mode."""
        self._check_input(feats, 'regress')
        keys = tuple(self.delta_keys) if delta_keys is None else tuple(sorted(int(k) for k in delta_keys if int(k) != 0))
        for k in keys:
            if k not in self.ief.deltas:
                raise _lib.HDError('no IEF head for delta_t %d' % k)
        self.sync_packs()
        feats = feats.contiguous().reshape(-1, 2048)
        tiled = omega_start is None
        start = self.param('mean_param') if tiled else omega_start
        if not tiled:
            self._check_input(start, 'regress(omega_start)', 85)
            start = start.contiguous()
        names = [n for dt in (0,) + keys for n in ief_names(dt)]
        if self._grad_on(names + ['mean_param'], feats, start):
            outs = RegressFunction.apply(self, keys, tiled, dropout, feats, start, *[self.param(n) for n in names])
        else:
            with torch.no_grad():
                outs = regress_plan(self, keys, tiled, feats.detach(), start.detach(), dropout)[0]
        return outs[0], {k: outs[1 + i] for i, k in enumerate(keys)}

    def predict_from_features(self, phi, smpl, single_frame=False):
        """Tester's fetch dict (tester.py:217-255) from features phi (B,T,2048) through f_movie (or fc2_res with pred_mode 'hal'), the IEF
        heads and the differentiable SMPL `smpl` (src.tf_smpl.batch_smpl.SMPL): cams, joints, kps, poses, shapes, verts, omegas and
        their *_delta stackings [B,T,D,...]; the delta heads' cameras are the main prediction's (tester.py:210-213)."""
        from src.tf_smpl.projection import batch_orth_proj_idrot
        B, T = phi.shape[0], phi.shape[1]
        N = B * T
        if single_frame:
            strips = phi
            keys = ()
        else:
            strips = self.temporal_encode(phi) if self.config.pred_mode == 'pred' else self.hallucinate(phi)
            keys = tuple(self.delta_keys)
        omega, deltas = self.regress(strips.reshape(N, 2048), delta_keys=keys)
        cams = omega[:, :3]

        def smpl_out(om, cam):
            verts, joints, Rs = smpl(om[:, 75:85], om[:, 3:75], get_skin=True)
            kps = batch_orth_proj_idrot(joints, cam)
            return {'cams': cam, 'joints': joints, 'kps': kps, 'poses': Rs, 'shapes': om[:, 75:85], 'verts': verts, 'omegas': om}
        o0 = smpl_out(omega, cams)
        out = {k: v.reshape((B, T) + tuple(v.shape[1:])) for k, v in o0.items()}
        if keys:
            per = [smpl_out(deltas[k], cams) for k in keys]
            for k in o0:
                out[k + '_delta'] = torch.stack([p[k] for p in per], 1).reshape((B, T, len(keys)) + tuple(per[0][k].shape[1:]))
        out['_movie_strips'] = strips
        return out

    def relu_masks(self, phi=None, feats=None, hal=None, omega_start=None, delta_keys=None):
        """The ReLU masks (pre-activation > 0) of the GPU forward, as CPU bool tensors keyed like oracle/nets_grad_ref's sites: f_movie
        over phi (B,T,2048) ('fm<i>.gn1' / '.gn2', [B,T,1,C]), the IEF heads over feats (N,2048) ('main.s<k>.fc1', 'd<dt>.s<k>.fc2', ...)
        and fc2_res over hal (N,2048) ('hal.fc1' / '.fc2').  An inspection aid for comparing against a float64 reference at near-tie
        sites; runs its own forward."""
        out = {}
        st = current_stream()
        with torch.no_grad():
            self.sync_packs()
            if phi is not None:
                B, T, Cc = phi.shape
                plan = FMoviePlan(self.fmovie, B, T, keep=True)
                plan.run(phi.contiguous())
                gain, offset = torch.empty((B, Cc), dtype=F32, device=self.device), torch.empty((B, Cc), dtype=F32, device=self.device)
                a = torch.empty((Cc, B * T), dtype=F32, device=self.device)
                for i, (x, mid) in enumerate(plan.saved):
                    for k, src in ((1, x), (2, mid)):
                        g, b = self.fmovie.blocks[i]['gn%d' % k]
                        check(lib.hd_groupnorm_stats(fptr(src), fptr(g), fptr(b), fptr(gain), fptr(offset), B, T, Cc, GN_GROUPS, GN_EPS, st),
                              'hd_groupnorm_stats')
                        check(lib.hd_im2col_t(fptr(src), B, T, Cc, 1, 0, fptr(gain), fptr(offset), 1, fptr(a), B * T, B * T, st), 'hd_im2col_t')
                        out['fm%d.gn%d' % (i, k)] = (a.t() > 0).reshape(B, T, 1, Cc).cpu()
            if feats is not None:
                keys = tuple(self.delta_keys) if delta_keys is None else tuple(sorted(int(k) for k in delta_keys if int(k) != 0))
                tiled = omega_start is None
                start = self.param('mean_param') if tiled else omega_start.contiguous()
                plan = regress_plan(self, keys, tiled, feats.contiguous(), start.detach())[2]
                for name, (h1, h2, _, _) in zip(['main'] + ['d%d' % k for k in keys], plan.saved):
                    for s in range(3):
                        out['%s.s%d.fc1' % (name, s)] = (h1[s] > 0).cpu()
                        out['%s.s%d.fc2' % (name, s)] = (h2[s] > 0).cpu()
            if hal is not None:
                x = hal.contiguous()
                h1, h2 = torch.empty_like(x), torch.empty_like(x)
                self.hal.run(x, h1, h2, torch.empty_like(x))
                out['hal.fc1'], out['hal.fc2'] = (h1 > 0).cpu(), (h2 > 0).cpu()
        return out

    # ---------------------------------------------------------------- export
    def tf_variables(self):
        """Every variable of the checkpoint the model came from, the trainable ones replaced by their current values: {name: ndarray}."""
        out = {k: np.asarray(v) for k, v in self._source.items()}
        for n in self.names:
            a = self.param(n).detach().cpu().numpy()
            out[n] = a.reshape(np.shape(self._source[n])).astype(np.asarray(self._source[n]).dtype)
        return out

    def save_checkpoint(self, prefix):
        """Write tf_variables() as a TensorFlow V2 checkpoint (`prefix`.index / .data-00000-of-00001) that HMMREngine and Tester load."""
        from .tf_checkpoint import save_checkpoint
        save_checkpoint(prefix, self.tf_variables())
        return prefix
