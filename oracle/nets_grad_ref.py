"""ORACLE (test infrastructure, not product): float64 autograd gradients of the trainable HMMR layers -- f_movie, the IEF heads
(call_hmr_ief as Tester wires it) and fc2_res -- on top of oracle/nets_ref.py's restatement (same assumptions A7 / A8).

Weights are torch leaves here (nets_ref's functions convert their numpy weights with `_t`, which would cut the graph), so this module
restates the three networks with tensor weights and reuses nets_ref's conv2d_nhwc / group_norm_tf.  tests/test_temporal_grad_cpu.py
pins it to nets_ref (1e-12 in float64) and to finite differences.

ReLU masks at near-tie sites.  The GPU forward (fp16-split operands, ~2^-22 relative) and this float64 forward disagree on the sign of a
few pre-activations within ~1e-6 of zero.  `masks` = {site name: bool tensor} overrides torch.relu's mask at a site (the value is
x * mask there); `record` (a dict) receives every site's pre-activation so a test can pick the near-tie positions and take the GPU's
sign only there.  Site names: 'fm<i>.gn1' / 'fm<i>.gn2' (block i of f_movie), '<scope>.s<stage>.fc1' / '.fc2', 'hal.fc1' / 'hal.fc2'.
"""
from __future__ import annotations

import torch

from .nets_ref import GN_EPS, GN_GROUPS, conv2d_nhwc, group_norm_tf


def _relu(x, name, masks, record):
    if record is not None:
        record[name] = x.detach()
    if masks is not None and name in masks:
        return x * masks[name].to(x.dtype)
    return torch.relu(x)


def fmovie(x, blocks, masks=None, record=None):
    """az_fc2_groupnorm.  x (B,T,C); blocks = [dict(gn1=(gamma, beta), conv1=(W, b), gn2=..., conv2=...)] with W HWIO (3,1,C,C)."""
    for i, p in enumerate(blocks):
        y = x[:, :, None, :]
        y = _relu(group_norm_tf(y, p['gn1'][0], p['gn1'][1], GN_GROUPS, GN_EPS), 'fm%d.gn1' % i, masks, record)
        y = conv2d_nhwc(y, p['conv1'][0], p['conv1'][1], 1, 'SAME')
        y = _relu(group_norm_tf(y, p['gn2'][0], p['gn2'][1], GN_GROUPS, GN_EPS), 'fm%d.gn2' % i, masks, record)
        y = conv2d_nhwc(y, p['conv2'][0], p['conv2'][1], 1, 'SAME')
        x = y[:, :, 0, :] + x
    return x


def hmr_ief(phi, start, p, name, num_stage=3, masks=None, record=None):
    """hmr_ief with encoder_fc3_dropout at inference; p = (W1, b1, W2, b2, W3, b3)."""
    W1, b1, W2, b2, W3, b3 = p
    theta = start
    for s in range(num_stage):
        state = torch.cat([phi, theta], dim=1)
        h = _relu(state @ W1 + b1, '%s.s%d.fc1' % (name, s), masks, record)
        h = _relu(h @ W2 + b2, '%s.s%d.fc2' % (name, s), masks, record)
        theta = theta + (h @ W3 + b3)
    return theta


def call_hmr_ief(phi, start, heads, delta_keys=(), masks=None, record=None):
    """Main head from `start` (N,85), then the delta heads from its pose with its beta carried (use_delta_from_pred=True,
    use_optcam=True).  heads = {0: p_main, dt: p_delta}.  Returns (theta (N,85), {dt: (N,85)})."""
    theta = hmr_ief(phi, start, heads[0], 'main', masks=masks, record=record)
    n = phi.shape[0]
    out = {}
    for dt in delta_keys:
        pred = hmr_ief(phi, theta[:, 3:75], heads[dt], 'd%d' % dt, masks=masks, record=record)
        one = dict(dtype=phi.dtype, device=phi.device)
        out[dt] = torch.cat([torch.ones(n, 1, **one), torch.zeros(n, 2, **one), pred, theta[:, 75:85]], dim=1)
    return theta, out


def fc2_res(x, p, masks=None, record=None):
    W1, b1, W2, b2, W3, b3 = p
    h = _relu(x @ W1 + b1, 'hal.fc1', masks, record)
    h = _relu(h @ W2 + b2, 'hal.fc2', masks, record)
    return h @ W3 + b3 + x


def leaves(weights, names, dtype=torch.float64, device=None):
    """{name: leaf tensor requiring grad} from a numpy weight dict."""
    import numpy as np
    return {n: torch.tensor(np.asarray(weights[n], np.float64), dtype=dtype, device=device, requires_grad=True) for n in names}


def fmovie_blocks(L, num_conv_layers=3):
    out = []
    for i in range(num_conv_layers):
        name = 'block_%d' % i
        out.append({'gn%d' % k: (L['AZ_FC_block_preact_gn%d%s/gamma' % (k, name)], L['AZ_FC_block_preact_gn%d%s/beta' % (k, name)])
                    for k in (1, 2)})
        out[-1].update({'conv%d' % k: (L['AZ_FC_block2_conv%d%s/weights' % (k, name)], L['AZ_FC_block2_conv%d%s/biases' % (k, name)])
                        for k in (1, 2)})
    return out


def ief_params(L, dt, scope='single_view_ief'):
    sc = scope if dt == 0 else scope + ('_future%d' % dt if dt > 0 else '_past%d' % abs(dt))
    q = sc + '/3D_module'
    return tuple(L[q + '/fc%d/%s' % (i, k)] for i in (1, 2, 3) for k in ('weights', 'biases'))
