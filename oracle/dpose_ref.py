"""ORACLE (test infrastructure, not product): the adversarial pose prior D_pose (reference src/discriminators.py) and its LSGAN losses
(src/ops.py compute_loss_e_fake / d_fake / d_real / shape), forward and hand-written backward in numpy, in the dtype of the input
(float64 for judging the GPU, float32 for comparing with the stand-in execution in tests/golden/dpose_v1.npz).

Parameters: params_from_tf(weights) -> dict W1 [9,32], b1, W2 [32,32], b2, wj [23,32], bj [23], Wf1 [736,1024], bf1, Wf2 [1024,1024],
bf2, wo [1024], bo [].  ReLU sites 'conv1', 'conv2' ([N,23,32]), 'fc1', 'fc2' ([N,1024]): `masks` overrides the mask of a site (near-tie
handling, as in nets_grad_ref), `record` receives every site's pre-activation.  DPoseRef wraps forward / backward as a torch autograd
Function (CPU float64), for gradcheck and for chaining with nets_grad_ref / smpl_grad_ref.
"""
from __future__ import annotations

import numpy as np

J = 23
KEYS = ['W1', 'b1', 'W2', 'b2', 'wj', 'bj', 'Wf1', 'bf1', 'Wf2', 'bf2', 'wo', 'bo']


def params_from_tf(w, dtype=np.float64):
    a = lambda n: np.asarray(w['D_pose/' + n], dtype)       # noqa: E731
    return {'W1': a('D_conv1/weights').reshape(9, 32), 'b1': a('D_conv1/biases'),
            'W2': a('D_conv2/weights').reshape(32, 32), 'b2': a('D_conv2/biases'),
            'wj': np.stack([a('pose_out_j%d/weights' % j).reshape(32) for j in range(J)]),
            'bj': np.concatenate([a('pose_out_j%d/biases' % j).reshape(1) for j in range(J)]),
            'Wf1': a('D_alljoints_fc1/weights'), 'bf1': a('D_alljoints_fc1/biases'),
            'Wf2': a('D_alljoints_fc2/weights'), 'bf2': a('D_alljoints_fc2/biases'),
            'wo': a('D_alljoints_out/weights').reshape(1024), 'bo': a('D_alljoints_out/biases').reshape(())}


def _mask(a, name, masks, record):
    if record is not None:
        record[name] = a
    if masks is not None and name in masks:
        return np.asarray(masks[name]).reshape(a.shape).astype(a.dtype)
    return (a > 0).astype(a.dtype)


def forward(x, p, masks=None, record=None):
    """x (N, 23, 9) -> (logits (N, 24), cache for backward)."""
    x = np.asarray(x)
    N = x.shape[0]
    m1 = _mask(x @ p['W1'] + p['b1'], 'conv1', masks, record)
    h1 = (x @ p['W1'] + p['b1']) * m1
    m2 = _mask(h1 @ p['W2'] + p['b2'], 'conv2', masks, record)
    h2 = (h1 @ p['W2'] + p['b2']) * m2
    heads = np.einsum('njc,jc->nj', h2, p['wj']) + p['bj']
    flat = h2.reshape(N, J * 32)
    a3 = flat @ p['Wf1'] + p['bf1']
    m3 = _mask(a3, 'fc1', masks, record)
    f1 = a3 * m3
    a4 = f1 @ p['Wf2'] + p['bf2']
    m4 = _mask(a4, 'fc2', masks, record)
    f2 = a4 * m4
    out = f2 @ p['wo'] + p['bo']
    return np.concatenate([heads, out[:, None]], 1), (x, h1, h2, f1, f2, m1, m2, m3, m4)


def backward(p, cache, g):
    """Gradients of sum(g * logits): (dx (N, 23, 9), {key: gradient})."""
    x, h1, h2, f1, f2, m1, m2, m3, m4 = cache
    N = x.shape[0]
    g = np.asarray(g, x.dtype)
    gh, go = g[:, :J], g[:, J]
    gr = {'wo': f2.T @ go, 'bo': go.sum()}
    df2 = go[:, None] * p['wo'][None, :] * m4
    gr['Wf2'], gr['bf2'] = f1.T @ df2, df2.sum(0)
    df1 = (df2 @ p['Wf2'].T) * m3
    flat = h2.reshape(N, J * 32)
    gr['Wf1'], gr['bf1'] = flat.T @ df1, df1.sum(0)
    dh2 = (df1 @ p['Wf1'].T).reshape(N, J, 32) + gh[:, :, None] * p['wj'][None]
    gr['wj'], gr['bj'] = np.einsum('nj,njc->jc', gh, h2), gh.sum(0)
    da2 = dh2 * m2
    gr['W2'], gr['b2'] = np.einsum('njk,njc->kc', h1, da2), da2.sum((0, 1))
    da1 = (da2 @ p['W2'].T) * m1
    gr['W1'], gr['b1'] = np.einsum('nji,njc->ic', x, da1), da1.sum((0, 1))
    return da1 @ p['W1'].T, gr


def loss_e_fake(out):
    return np.mean(np.sum((out - 1) ** 2, axis=1))


def loss_d_fake(out):
    return np.mean(np.sum(out ** 2, axis=1))


def loss_d_real(out):
    return np.mean(np.sum((out - 1) ** 2, axis=1))


def loss_shape(beta):
    return np.mean(np.square(beta))


def _torch_function():
    import torch

    class DPoseRef(torch.autograd.Function):
        """(x (N,23,9), *params in KEYS order) -> logits; CPU tensors, numpy forward / backward in their dtype."""

        @staticmethod
        def forward(ctx, masks, x, *params):
            p = {k: t.detach().cpu().numpy() for k, t in zip(KEYS, params)}
            out, cache = forward(x.detach().cpu().numpy(), p, masks)
            ctx.p, ctx.cache, ctx.shapes = p, cache, [t.shape for t in params]
            return torch.from_numpy(out)

        @staticmethod
        def backward(ctx, g):
            dx, gr = backward(ctx.p, ctx.cache, g.detach().cpu().numpy())
            return (None, torch.from_numpy(np.ascontiguousarray(dx))) + tuple(torch.from_numpy(np.asarray(gr[k])).reshape(s)
                                                                           for k, s in zip(KEYS, ctx.shapes))
    return DPoseRef


def torch_apply(x, params, masks=None):
    """D_pose on CPU torch tensors, differentiable (first order) w.r.t. x and params (a dict over KEYS)."""
    return _torch_function().apply(masks, x, *[params[k] for k in KEYS])
