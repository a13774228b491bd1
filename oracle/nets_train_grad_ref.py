"""ORACLE (test infrastructure, not product): float64 autograd gradients of the training-mode ResNet trunk (slim resnet_v2_50 with
is_training=True, what the reference trains with freeze_phi=False) over torch-leaf variables.

The forward restates oracle/nets_train_ref.encoder_resnet_train (A1-A4 of nets_ref, A5t) with tensor weights, so torch autograd gives
the gradient of every conv weight and bias and every batch-norm gamma / beta, the gradient flowing through the batch mean and variance.
tests/test_resnet_grad_cpu.py pins its forward to nets_train_ref (1e-12 in float64; that module is pinned to the reference's own
encoder_resnet run over the TF stand-in, tests/golden/resnet_train_bn_v1.npz) and its gradients to central finite differences.  The TF
stand-in has no tf.gradients, so the backward is pinned through this module and finite differences only.

Conventions of the backward [TF-ext]: ReluGrad is 0 at 0 (torch.relu's gradient); MaxPoolGrad of the 3x3 stride-2 SAME pool sends each
window's gradient to its FIRST maximum in scan order (ky, then kx), as TF's CPU kernel does (torch.argmax returns the first maximum).

Near ties.  The GPU forward (fp16-split operands) and this float64 forward can disagree on the sign of a pre-activation within ~1e-6 of
zero, or on a pool window's maximum when two inputs nearly tie.  `masks` = {site: tensor} overrides the choice at a site: a bool mask of
the pre-activation at a ReLU site (the value is x * mask), the window index (0..8, ky * 3 + kx, int64 [N, C, Ho, Wo]) at 'pool1'.
`record` (a dict) receives each ReLU site's pre-activation and pool1's window index.  ReLU site names are the batch-norm scopes
(nets.resnet_bn_scopes): '<unit>/preact', '<unit>/conv1/BatchNorm', '<unit>/conv2/BatchNorm', 'resnet_v2_50/postnorm'.

Only tests/ and tools/ may import this module.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from .nets_ref import RESNET_BLOCKS, conv2d_nhwc, conv2d_same, same_pad

BN_EPS = 1e-5


def trunk_names(blocks=RESNET_BLOCKS):
    """Every trainable variable of the trunk: conv weights / biases in forward order, then gamma / beta per batch-norm scope."""
    p = 'resnet_v2_50'
    convs, scopes, d_in = [p + '/conv1/weights', p + '/conv1/biases'], [], 64
    for b, (base, units, _) in enumerate(blocks, start=1):
        for u in range(1, units + 1):
            q = '%s/block%d/unit_%d/bottleneck_v2' % (p, b, u)
            if d_in != 4 * base:
                convs += [q + '/shortcut/weights', q + '/shortcut/biases']
            convs += [q + '/conv1/weights', q + '/conv2/weights', q + '/conv3/weights', q + '/conv3/biases']
            scopes += [q + '/preact', q + '/conv1/BatchNorm', q + '/conv2/BatchNorm']
            d_in = 4 * base
    scopes.append(p + '/postnorm')
    return convs + [s + '/' + k for s in scopes for k in ('gamma', 'beta')]


def leaves(weights, blocks=RESNET_BLOCKS, dtype=torch.float64, device=None):
    """{name: leaf tensor requiring grad} for trunk_names(blocks) from a numpy weight dict."""
    return {n: torch.tensor(np.asarray(weights[n], np.float64), dtype=dtype, device=device, requires_grad=True) for n in trunk_names(blocks)}


def _relu(x, name, masks, record):
    if record is not None:
        record[name] = x.detach()
    if masks is not None and name in masks:
        return x * masks[name].to(device=x.device, dtype=x.dtype)
    return torch.relu(x)


def batch_norm_relu(x, L, scope, masks=None, record=None):
    """A5t + ReLU: batch moments over N, H, W (biased variance), gradient through both."""
    mean = x.mean(dim=(0, 1, 2))
    var = ((x - mean) ** 2).mean(dim=(0, 1, 2))
    y = L[scope + '/gamma'] * (x - mean) / torch.sqrt(var + BN_EPS) + L[scope + '/beta']
    return _relu(y, scope, masks, record)


def max_pool_3x3_s2(x, masks=None, record=None):
    """pool1 (3x3 stride 2 SAME, padding ignored) as a gather of one input per window: the first maximum, or masks['pool1']."""
    N, H, W, Cc = x.shape
    pt, pb, _ = same_pad(H, 3, 2)
    pl, pr, _ = same_pad(W, 3, 2)
    xp = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb), value=float('-inf'))
    win = xp.unfold(2, 3, 2).unfold(3, 3, 2)                      # N, C, Ho, Wo, 3, 3
    win = win.reshape(win.shape[:4] + (9,))
    idx = masks['pool1'].to(x.device) if masks is not None and 'pool1' in masks else win.detach().argmax(-1)
    if record is not None:
        record['pool1'] = idx
    return win.gather(-1, idx[..., None])[..., 0].permute(0, 2, 3, 1)


def encoder_resnet_train(x, L, blocks=RESNET_BLOCKS, masks=None, record=None):
    """x NHWC (N,S,S,3) tensor (no gradient) -> phi (N, 2048) on the autograd graph of the leaves L (name -> tensor)."""
    p = 'resnet_v2_50'
    net = conv2d_same(x, L[p + '/conv1/weights'], 2, L[p + '/conv1/biases'])
    net = max_pool_3x3_s2(net, masks, record)
    for b, (base, units, bstride) in enumerate(blocks, start=1):
        for u in range(1, units + 1):
            s = bstride if u == units else 1
            q = '%s/block%d/unit_%d/bottleneck_v2' % (p, b, u)
            depth = 4 * base
            preact = batch_norm_relu(net, L, q + '/preact', masks, record)
            if depth == net.shape[-1]:
                shortcut = net if s == 1 else net[:, ::s, ::s, :]
            else:
                shortcut = conv2d_nhwc(preact, L[q + '/shortcut/weights'], L[q + '/shortcut/biases'], s, 'VALID')
            r = conv2d_nhwc(preact, L[q + '/conv1/weights'], None, 1, 'SAME')
            r = batch_norm_relu(r, L, q + '/conv1/BatchNorm', masks, record)
            r = conv2d_same(r, L[q + '/conv2/weights'], s)
            r = batch_norm_relu(r, L, q + '/conv2/BatchNorm', masks, record)
            r = conv2d_nhwc(r, L[q + '/conv3/weights'], L[q + '/conv3/biases'], 1, 'SAME')
            net = shortcut + r
    net = batch_norm_relu(net, L, p + '/postnorm', masks, record)
    return net.mean(dim=(1, 2))


def trunk_gradients(x, weights, dphi, blocks=RESNET_BLOCKS, masks=None, record=None, device=None):
    """{name: float64 gradient of sum(phi * dphi)} for every trainable variable, and phi."""
    L = leaves(weights, blocks, device=device)
    xt = torch.as_tensor(np.asarray(x)).to(device=device, dtype=torch.float64)
    phi = encoder_resnet_train(xt, L, blocks, masks, record)
    names = list(L)
    g = torch.autograd.grad(phi, [L[n] for n in names], torch.as_tensor(np.asarray(dphi)).to(device=device, dtype=torch.float64))
    return dict(zip(names, g)), phi.detach()
