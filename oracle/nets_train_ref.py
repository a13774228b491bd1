"""ORACLE (test infrastructure, not product): float64 restatement of slim's resnet_v2_50 in TRAINING mode (is_training=True), the call
src/models.py:50-77 makes under trainer_sequence_fc.py:562-575.  Same topology and conventions as nets_ref (A1-A4); batch norm differs:

  A5t  BatchNorm training [TF-ext]: y = gamma * (x - mean_b) / sqrt(var_b + 1e-5) + beta with the moments of the batch over N, H, W
       (var_b biased); the layer's UPDATE_OPS step the moving statistics once, m -= (m - v) * (1 - decay), decay 0.997
       (resnet_arg_scope), v = mean_b for the mean and the Bessel-corrected var_b * rows / (rows - 1) for the variance (TF 1.8's fused
       kernel).  Pinned against the reference's own encoder_resnet run over the TF stand-in (tests/golden/make_resnet_train_golden.py).

Only tests/ and tools/ may import this module.
"""
from __future__ import annotations

import numpy as np
import torch

from .nets_ref import RESNET_BLOCKS, conv2d_nhwc, conv2d_same, max_pool_same_3x3_s2

BN_EPS = 1e-5
BN_DECAY = 0.997


class _Weights(object):
    def __init__(self, w, dtype, device):
        self.w, self.dtype, self.device = w, dtype, device

    def __call__(self, name):
        return torch.as_tensor(np.asarray(self.w[name])).to(device=self.device, dtype=self.dtype)


def batch_norm_train(x, W, prefix, moments, relu=True):
    """A5t on an NHWC map: normalised output (+ReLU); records (mean_b, var_b) under `prefix` in `moments`."""
    mean = x.mean(dim=(0, 1, 2))
    var = ((x - mean) ** 2).mean(dim=(0, 1, 2))
    moments[prefix] = (mean, var, x.shape[0] * x.shape[1] * x.shape[2])
    y = W(prefix + '/gamma') * (x - mean) / torch.sqrt(var + BN_EPS) + W(prefix + '/beta')
    return torch.relu(y) if relu else y


def encoder_resnet_train(x, weights, dtype=torch.float64, blocks=RESNET_BLOCKS, device='cpu', decay=BN_DECAY):
    """x NHWC (N,S,S,3) -> (phi (N,2048), moments {scope: (mean_b, var_b)}, moving {'<scope>/moving_mean' | '_variance': after one
    step of the update ops}), float64 numpy arrays."""
    W = _Weights(weights, dtype, device)
    x = torch.as_tensor(np.asarray(x)).to(device=device, dtype=dtype)
    p = 'resnet_v2_50'
    mom = {}
    net = conv2d_same(x, W(p + '/conv1/weights'), 2, W(p + '/conv1/biases'))
    net = max_pool_same_3x3_s2(net)
    for b, (base, units, bstride) in enumerate(blocks, start=1):
        for u in range(1, units + 1):
            s = bstride if u == units else 1
            q = '%s/block%d/unit_%d/bottleneck_v2' % (p, b, u)
            depth = 4 * base
            preact = batch_norm_train(net, W, q + '/preact', mom)
            if depth == net.shape[-1]:
                shortcut = net if s == 1 else net[:, ::s, ::s, :]
            else:
                shortcut = conv2d_nhwc(preact, W(q + '/shortcut/weights'), W(q + '/shortcut/biases'), s, 'VALID')
            r = conv2d_nhwc(preact, W(q + '/conv1/weights'), None, 1, 'SAME')
            r = batch_norm_train(r, W, q + '/conv1/BatchNorm', mom)
            r = conv2d_same(r, W(q + '/conv2/weights'), s)
            r = batch_norm_train(r, W, q + '/conv2/BatchNorm', mom)
            r = conv2d_nhwc(r, W(q + '/conv3/weights'), W(q + '/conv3/biases'), 1, 'SAME')
            net = shortcut + r
    net = batch_norm_train(net, W, p + '/postnorm', mom)
    phi = net.mean(dim=(1, 2))
    moments, moving = {}, {}
    for scope, (mean, var, rows) in mom.items():
        mean, var = mean.cpu().numpy().astype(np.float64), var.cpu().numpy().astype(np.float64)
        moments[scope] = (mean, var)
        mm = np.asarray(weights[scope + '/moving_mean'], np.float64)
        mv = np.asarray(weights[scope + '/moving_variance'], np.float64)
        moving[scope + '/moving_mean'] = mm - (mm - mean) * (1.0 - decay)
        moving[scope + '/moving_variance'] = mv - (mv - var * rows / (rows - 1)) * (1.0 - decay)
    return phi.cpu().numpy().astype(np.float64), moments, moving
