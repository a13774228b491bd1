"""Training-mode dropout for the TensorFlow stand-in (oracle/ref_exec/stubs), with its uniforms from an injected provider.

The stand-in's own `tf.nn.dropout` and `tf.contrib.layers.dropout(is_training=True)` raise: it is an inference stand-in.  `install`
replaces them (and `tf.contrib.slim.dropout`, which the reference calls: src/models.py:103,105) with TF 1.8's definitions, drawing
the uniforms of random_uniform from `provider`; `uninstall` puts the raising originals back.  Import this module after the stubs
are first on sys.path, so that `tensorflow` is the stand-in.

    provider(path) -> (shape -> float32 uniforms in [0, 1))
is called once per dropout op as the graph is built, with the op's path '<variable scope>/<name>' (e.g.
'single_view_ief_past5/3D_module/dropout2'); the function it returns is called with the op's shape when the op runs.
"""
import numpy as np

_saved = None


def _nn_dropout(provider):
    import tensorflow as tf

    def dropout(x, keep_prob, noise_shape=None, seed=None, name=None):
        """TF 1.8 nn_ops.dropout: keep_prob a float32 tensor, binary = floor(keep_prob + random_uniform), ret = div(x, keep_prob) *
        binary, all in float32."""
        x = tf.convert_to_tensor(x)
        p = np.float32(keep_prob)
        scope = tf.get_variable_scope().name
        uniform = provider('/'.join([n for n in (scope, name or 'dropout') if n]))

        def fn(a):
            binary = np.floor(p + np.asarray(uniform(a.shape), np.float32))
            return (a / p) * binary
        return tf._op(fn, [x], 'dropout')
    return dropout


def _layers_dropout(nn_dropout, inference):
    def dropout(inputs, keep_prob=0.5, is_training=True, scope=None, **kw):
        """TF 1.8 contrib.layers.dropout -> core_layers.Dropout(rate=1 - keep_prob) -> nn.dropout(x, 1 - rate): the keep_prob
        nn.dropout sees is worked out in Python float64 and becomes a float32 tensor there."""
        if not is_training:
            return inference(inputs, keep_prob, is_training=False, scope=scope, **kw)
        return nn_dropout(inputs, 1 - (1 - keep_prob), name=scope or 'Dropout')
    return dropout


def install(provider):
    """Training-mode dropout from `provider` in tf.nn, tf.contrib.layers and tf.contrib.slim until `uninstall`."""
    global _saved
    import tensorflow as tf
    from tensorflow.contrib import layers, slim
    if _saved is None:
        _saved = (tf.nn.dropout, layers.dropout, slim.dropout)
    nn_dropout = _nn_dropout(provider)
    tf.nn.dropout = nn_dropout
    layers.dropout = slim.dropout = _layers_dropout(nn_dropout, _saved[1])


def uninstall():
    """The stand-in's own dropout again: training mode raises."""
    global _saved
    if _saved is None:
        return
    import tensorflow as tf
    from tensorflow.contrib import layers, slim
    tf.nn.dropout, layers.dropout, slim.dropout = _saved
    _saved = None
