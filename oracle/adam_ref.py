"""TF 1.8's Adam (tf.train.AdamOptimizer, ApplyAdam with use_nesterov=False, training_ops.cc / training_ops_gpu.cu.cc) restated in
numpy, and the names its state takes in a checkpoint.  Restated from TF's source, not executed against TF.

    apply_adam_f64   the update in float64: the reference arithmetic
    apply_adam_f32   the same in float32, operation by operation in the kernel's order, each rounded once (csrc/adam.cu matches it
                     bit for bit)
    finish           _finish: beta1_power *= beta1, beta2_power *= beta2, once per step after every variable
    state_names      the optimizer entries of the reference trainer's checkpoint (trainer_sequence_fc.py:752-768 + tf.train.Saver)
"""
import numpy as np


def _update(p, g, m, v, lr, beta1, beta2, epsilon, b1p, b2p, dt):
    one = dt(1)
    lr, beta1, beta2, epsilon, b1p, b2p = (dt(x) for x in (lr, beta1, beta2, epsilon, b1p, b2p))
    p, g, m, v = (np.asarray(x, dt) for x in (p, g, m, v))
    alpha = (lr * np.sqrt(one - b2p)) / (one - b1p)
    m = m + (one - beta1) * (g - m)
    v = v + (one - beta2) * (g * g - v)
    p = p - (alpha * m) / (epsilon + np.sqrt(v))
    return p, m, v


def apply_adam_f64(p, g, m, v, lr, beta1, beta2, epsilon, b1p, b2p):
    """One ApplyAdam on one variable in float64: -> (p, m, v).  b1p, b2p are the powers before this step's finish."""
    return _update(p, g, m, v, lr, beta1, beta2, epsilon, b1p, b2p, np.float64)


def apply_adam_f32(p, g, m, v, lr, beta1, beta2, epsilon, b1p, b2p):
    """The same in float32: alpha = (lr * sqrt(1 - b2p)) / (1 - b1p); m + (1 - beta1) * (g - m); v + (1 - beta2) * (g*g - v);
    p - (alpha * m) / (epsilon + sqrt(v)), each operation rounded to float32 once (numpy does not contract)."""
    with np.errstate(under='ignore'):
        return _update(p, g, m, v, lr, beta1, beta2, epsilon, b1p, b2p, np.float32)


def finish(b1p, b2p, beta1, beta2, dtype=np.float32):
    """TF's _finish: (beta1_power * beta1, beta2_power * beta2) in `dtype`."""
    with np.errstate(under='ignore'):
        return dtype(b1p) * dtype(beta1), dtype(b2p) * dtype(beta2)


def state_names(e_names, d_names, d_trained):
    """The optimizer entries of the checkpoint, as TF names them: each trained variable's slots `<var>/Adam` (m) and `<var>/Adam_1`
    (v); E's optimizer is built first (setup_optimizers), so its powers are beta1_power / beta2_power and D's, made in the same graph,
    are uniquified to beta1_power_1 / beta2_power_1; D has an optimizer only when it trains (use_disc_pose = d_lw_pose > 0); and
    global_step, which both minimize calls advance."""
    out = [n + s for n in e_names for s in ('/Adam', '/Adam_1')] + ['beta1_power', 'beta2_power']
    if d_trained:
        out += [n + s for n in d_names for s in ('/Adam', '/Adam_1')] + ['beta1_power_1', 'beta2_power_1']
    return out + ['global_step']
