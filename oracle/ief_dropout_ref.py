"""ORACLE (test infrastructure, not product): the IEF heads in training mode (is_training=True, src/models.py:101-105) with explicit
dropout masks, in float64 -- the forward of oracle/nets_ref.py's call_hmr_ief and the differentiable one of oracle/nets_grad_ref.py,
with nn.dropout after the ReLU of fc1 and fc2: (relu(x) / keep_prob) * keep.

Masks come from oracle/dropout_ref.py (`dropout_ref.ief_masks`: {(head, stage, layer): [N, 1024] uint8}, head 0 = main, then the delta
heads in ascending dt; layer 0 = dropout1); keep_prob is nn.dropout's float32 value (`dropout_ref.nn_keep_prob`).
"""
from __future__ import annotations

import torch

from .nets_grad_ref import _relu
from .nets_ref import _t


def _scope_delta(scope, dt):
    return scope + ('_future%d' % dt if dt > 0 else '_past%d' % abs(dt))


# ------------------------------------------------------------------------------------------------------------------------------------
# forward (nets_ref's, numpy weights keyed by TF names)
# ------------------------------------------------------------------------------------------------------------------------------------
def encoder_fc3_dropout(x, weights, scope, dtype, masks, keep_prob):
    """src/models.py:80-116 with is_training=True; masks = (dropout1, dropout2) keep masks [N, 1024]."""
    net = torch.relu(x @ _t(weights[scope + '/fc1/weights'], dtype) + _t(weights[scope + '/fc1/biases'], dtype))
    net = net / keep_prob * _t(masks[0], dtype)
    net = torch.relu(net @ _t(weights[scope + '/fc2/weights'], dtype) + _t(weights[scope + '/fc2/biases'], dtype))
    net = net / keep_prob * _t(masks[1], dtype)
    return net @ _t(weights[scope + '/fc3/weights'], dtype) + _t(weights[scope + '/fc3/biases'], dtype)


def hmr_ief(phi, omega_start, weights, scope, masks, keep_prob, num_stage=3, dtype=torch.float64):
    """src/models.py:380-415; masks = per stage the (dropout1, dropout2) keep masks."""
    theta = omega_start
    for stage in range(num_stage):
        theta = theta + encoder_fc3_dropout(torch.cat([phi, theta], dim=1), weights, scope + '/3D_module', dtype, masks[stage], keep_prob)
    return theta


def batch_pred_omega(input_features, batch_size, weights, omega_mean, sequence_length, delta_keys, masks, keep_prob,
                     scope='single_view_ief', dtype=torch.float64):
    """src/models.py:233-267 -> call_hmr_ief (:299-377) as the trainer wires it (num_output 85, use_delta_from_pred=True,
    use_optcam=True), in training mode.  masks = {dt: hmr_ief's per-stage masks}, dt 0 = the main head.  Returns (omega [B, T, 85],
    {dt: [B, T, 85]})."""
    phi = _t(input_features, dtype).reshape(batch_size * sequence_length, -1)
    theta = hmr_ief(phi, _t(omega_mean, dtype), weights, scope, masks[0], keep_prob, dtype=dtype)
    n = phi.shape[0]
    deltas = {}
    for dt in delta_keys:
        if dt == 0:
            continue
        pred = hmr_ief(phi, theta[:, 3:75], weights, _scope_delta(scope, dt), masks[dt], keep_prob, dtype=dtype)
        out = torch.cat([torch.ones(n, 1, dtype=dtype), torch.zeros(n, 2, dtype=dtype), pred, theta[:, -10:]], dim=1)
        deltas[dt] = out.reshape(batch_size, sequence_length, 85)
    return theta.reshape(batch_size, sequence_length, 85), deltas


# ------------------------------------------------------------------------------------------------------------------------------------
# differentiable (nets_grad_ref's: torch leaves, ReLU-sign overrides at near ties)
# ------------------------------------------------------------------------------------------------------------------------------------
def _relu_dropout(x, name, masks, record, drop):
    y = _relu(x, name, masks, record)
    return y / drop[1] * drop[0][name].to(x.dtype)


def grad_hmr_ief(phi, start, p, name, drop, num_stage=3, masks=None, record=None):
    """nets_grad_ref.hmr_ief with dropout: drop = ({site name: keep mask [N, H]}, keep_prob), site names '<name>.s<stage>.fc1' /
    '.fc2'; p = (W1, b1, W2, b2, W3, b3) (any widths)."""
    W1, b1, W2, b2, W3, b3 = p
    theta = start
    for s in range(num_stage):
        state = torch.cat([phi, theta], dim=1)
        h = _relu_dropout(state @ W1 + b1, '%s.s%d.fc1' % (name, s), masks, record, drop)
        h = _relu_dropout(h @ W2 + b2, '%s.s%d.fc2' % (name, s), masks, record, drop)
        theta = theta + (h @ W3 + b3)
    return theta


def grad_call_hmr_ief(phi, start, heads, delta_keys, drop, masks=None, record=None):
    """nets_grad_ref.call_hmr_ief with dropout (grad_hmr_ief's `drop`; heads 'main' and 'd<dt>')."""
    theta = grad_hmr_ief(phi, start, heads[0], 'main', drop, masks=masks, record=record)
    n = phi.shape[0]
    one = dict(dtype=phi.dtype, device=phi.device)
    out = {}
    for dt in delta_keys:
        pred = grad_hmr_ief(phi, theta[:, 3:75], heads[dt], 'd%d' % dt, drop, masks=masks, record=record)
        out[dt] = torch.cat([torch.ones(n, 1, **one), torch.zeros(n, 2, **one), pred, theta[:, 75:85]], dim=1)
    return theta, out


def drop_sites(masks, delta_keys):
    """dropout_ref.ief_masks' {(head, stage, layer): mask} -> grad_call_hmr_ief's {site name: bool tensor}."""
    names = ['main'] + ['d%d' % dt for dt in sorted(delta_keys)]
    return {'%s.s%d.fc%d' % (names[h], s, l + 1): torch.as_tensor(m.astype(bool)) for (h, s, l), m in masks.items() if h < len(names)}
