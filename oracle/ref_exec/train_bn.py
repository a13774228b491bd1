"""Training-mode batch_norm for the numpy TF stand-in [TF-ext] -- TEST INFRASTRUCTURE, not product code.

The stand-in's tf.contrib.layers.batch_norm is inference-only.  `install()` replaces it with one that also builds is_training=True as
TF 1.8's contrib batch_norm does for 4-D NHWC input (the fused kernel), restated from the TF API documentation:

  outputs   y = (x - mean_b) * rsqrt(var_b + epsilon) * gamma + beta, then activation_fn; mean_b / var_b are the moments over N, H, W
            (biased variance), in float32
  updates   two ops added to tf.GraphKeys.UPDATE_OPS: moving_mean -= (moving_mean - mean_b) * (1 - decay) and
            moving_variance -= (moving_variance - var_b * rows / (rows - 1)) * (1 - decay)  (assign_moving_average, zero_debias=False;
            the fused kernel's variance output is Bessel-corrected)

and gives the stand-in the graph-collection API the reference uses around it (tf.GraphKeys, tf.get_collection, tf.add_to_collection,
tf.group; the batch moments are also collected under MOMENTS as (scope, mean, variance)).  It also passes resnet_arg_scope's batch_norm_decay (0.997) to the resnet_v2 stand-in's batch norms, which the inference-only
stand-in never needed.  Nothing here is imported unless install() is called.
"""
import types

import numpy as np

MOMENTS = 'batch_norm_moments'


def install():
    import tensorflow as tf
    from tensorflow.contrib import layers
    from tensorflow.contrib.slim.python.slim.nets import resnet_v2
    if getattr(layers, '_train_bn_installed', False):
        return
    inference_bn = layers.batch_norm
    collections = {}

    tf.GraphKeys = types.SimpleNamespace(UPDATE_OPS='update_ops', GLOBAL_VARIABLES='variables', TRAINABLE_VARIABLES='trainable_variables')

    def add_to_collection(name, value):
        collections.setdefault(name, []).append(value)

    def get_collection(name, scope=None):
        return list(collections.get(name, []))

    def group(*inputs, **kw):
        flat = [t for x in inputs for t in (x if isinstance(x, (list, tuple)) else [x])]
        return tf._op(lambda *a: np.zeros((), np.float32), flat, 'group')

    def reset():
        collections.clear()

    tf.add_to_collection, tf.get_collection, tf.group = add_to_collection, get_collection, group
    tf.reset_collections = reset

    def assign_moving_average(var, value, decay):
        """An op that, when run, steps `var` in place and returns its new value (float32, like the TF kernel)."""
        one_minus = np.float32(1.0 - decay)

        def fn(v):
            if not var.initialized:            # graph construction evaluates every op on probe values: never step then
                return var.value
            var.value = (var.value - (var.value - v) * one_minus).astype(np.float32)
            return var.value
        return tf._op(fn, [value], 'AssignMovingAvg')

    def batch_norm(inputs, decay=0.999, center=True, scale=False, epsilon=0.001, activation_fn=None, is_training=True, reuse=None,
                   scope=None, updates_collections='update_ops', **kw):
        if not is_training:
            return inference_bn(inputs, decay=decay, center=center, scale=scale, epsilon=epsilon, activation_fn=activation_fn,
                                is_training=False, reuse=reuse, scope=scope, **kw)
        if len(inputs.shape) != 4:
            raise NotImplementedError('training-mode stand-in: 4-D NHWC input only')
        with tf.variable_scope(scope, 'BatchNorm', [inputs], reuse=reuse) as vs:
            C = inputs.shape[-1].value
            beta = tf.get_variable('beta', [C]) if center else None
            gamma = tf.get_variable('gamma', [C]) if scale else None
            moving_mean = tf.get_variable('moving_mean', [C], trainable=False)
            moving_var = tf.get_variable('moving_variance', [C], trainable=False)
        shp = inputs.shape.as_list()
        rows = shp[0] * shp[1] * shp[2]
        mean = tf._op(lambda a: a.mean(axis=(0, 1, 2), dtype=np.float32), [inputs], 'batch_mean')
        var = tf._op(lambda a, m: ((a - m) ** 2).mean(axis=(0, 1, 2), dtype=np.float32), [inputs, mean], 'batch_variance')
        inv = tf.rsqrt(var + np.float32(epsilon))
        if gamma is not None:
            inv = inv * gamma
        out = inputs * inv + ((beta - mean * inv) if beta is not None else (-mean * inv))
        var_u = var * np.float32(rows / (rows - 1.0))
        for u in (assign_moving_average(moving_mean, mean, decay), assign_moving_average(moving_var, var_u, decay)):
            add_to_collection(updates_collections, u)
        add_to_collection(MOMENTS, (vs.name, mean, var))          # for the fixture generator: the batch moments by scope
        return activation_fn(out) if activation_fn is not None else out

    layers.batch_norm = batch_norm
    resnet_v2._BN = dict(resnet_v2._BN, decay=0.997)          # resnet_arg_scope(batch_norm_decay=0.997)
    layers._train_bn_installed = True
