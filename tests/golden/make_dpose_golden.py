"""Generates tests/golden/dpose_v1.npz by EXECUTING THE REFERENCE'S OWN src/discriminators.py (PoseDiscriminator.get_output) and the
prior losses of its src/ops.py (compute_loss_e_fake, compute_loss_d_fake, compute_loss_d_real, compute_loss_shape) over the numpy
TensorFlow stand-in in oracle/ref_exec (set up exactly as make_ref_exec_golden.py does; extend_standin() below adds, in this process
only, the two features those files need that the stand-in does not have, so the stand-in and the fixtures made with it stay as they are).

As in the reference's trainer (trainer_sequence_fc.py:989-1018) the discriminator sees the reals and then the fakes concatenated.  The
variables the first get_output creates are read back through get_vars() (their names and shapes are stored) and loaded with seeded
values (human_dynamics_b200.synthetic.make_dpose_weights(3, bias_scale=0.1)); the inputs are regenerated from seeds by inputs() below.

Stored: x_real / x_fake (N, 23, 1, 9), beta, var_names and var_shapes (zero-padded to 4 dims) in creation order, logits
(N_REAL + N_FAKE, 24), e_pose, d_fake, d_real, e_shape.  The variable values are not stored: inputs() regenerates them.

Needs a checkout of the reference project, named by HD_REFERENCE_ROOT.  Run from the repo root:
    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_dpose_golden.py            (writes tests/golden/dpose_v1.npz)
    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_dpose_golden.py --check    (exit 0 when it reproduces the file)
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'dpose_v1.npz')
N_REAL, N_FAKE = 5, 7


def _by_path(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def rotations(rng, n):
    """(n, 23, 1, 9) float32 rotation matrices (Rodrigues of axis-angles with |angle| up to pi)."""
    aa = rng.normal(0, 1, size=(n * 23, 3))
    aa *= (rng.uniform(0, np.pi, size=(n * 23, 1)) / np.linalg.norm(aa, axis=1, keepdims=True))
    th = np.linalg.norm(aa, axis=1)[:, None, None]
    k = aa / th[:, :, 0]
    K = np.zeros((n * 23, 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    K = K - K.transpose(0, 2, 1)
    R = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
    return R.reshape(n, 23, 1, 9).astype(np.float32)


def inputs():
    """(weights, x_real, x_fake, beta) from seeds."""
    syn = _by_path('_hd_synthetic', os.path.join(ROOT, 'human_dynamics_b200', 'synthetic.py'))
    rng = np.random.RandomState(8)
    return (syn.make_dpose_weights(3, bias_scale=0.1), rotations(rng, N_REAL), rotations(rng, N_FAKE),
            rng.normal(0, 1, size=(N_FAKE, 10)).astype(np.float32))


def extend_standin(tf):
    """The two TF 1.x features discriminators.py / ops.py use that the stand-in lacks, added to this process's copy of it:
    slim.flatten ([N, ...] -> [N, prod(...)], row-major, tf.contrib.layers.flatten) and Tensor ** (tf.pow, element-wise)."""
    import tensorflow.contrib.slim as slim
    if not hasattr(slim, 'flatten'):
        def flatten(inputs, outputs_collections=None, scope=None):
            shp = inputs.shape.as_list()
            return tf.reshape(inputs, [shp[0], int(np.prod(shp[1:]))])
        slim.flatten = flatten
    if not hasattr(tf.Tensor, '__pow__'):
        tf.Tensor.__pow__ = lambda self, o: tf._binary(lambda a, b: a ** b, 'pow')(self, o)


def run_reference():
    gen = _by_path('_make_ref_exec_golden', os.path.join(HERE, 'make_ref_exec_golden.py'))
    w, xr, xf, beta = inputs()
    gen.setup_paths()
    import tensorflow as tf
    extend_standin(tf)
    from src.discriminators import PoseDiscriminator
    import src.ops as ops
    pr = tf.placeholder(tf.float32, xr.shape)
    pf = tf.placeholder(tf.float32, xf.shape)
    pb = tf.placeholder(tf.float32, beta.shape)
    D = PoseDiscriminator(1e-4)
    out = D.get_output(tf.concat([pr, pf], 0))
    out_real, out_fake = out[:N_REAL], out[N_REAL:]
    fetch = {'logits': out, 'e_pose': ops.compute_loss_e_fake(out_fake), 'd_fake': ops.compute_loss_d_fake(out_fake),
             'd_real': ops.compute_loss_d_real(out_real), 'e_shape': ops.compute_loss_shape(pb)}
    res = {'x_real': xr, 'x_fake': xf, 'beta': beta}
    names, shapes = [], []
    for v in D.get_vars():
        v.load(w[v.op_name])
        names.append(v.op_name)
        shapes.append(list(v.shape.as_list()) + [0] * (4 - len(v.shape)))
    res['var_names'], res['var_shapes'] = np.array(names), np.array(shapes, np.int64)
    with tf.Session() as sess:
        got = sess.run(fetch, feed_dict={pr: xr, pf: xf, pb: beta})
    res.update({k: np.asarray(v) for k, v in got.items()})
    return res


def main():
    res = run_reference()
    if '--check' in sys.argv:
        with np.load(OUT) as z:
            same = sorted(z.files) == sorted(res) and all(np.array_equal(z[k], res[k]) for k in z.files)
        print('reproduces %s: %s' % (OUT, same))
        raise SystemExit(0 if same else 1)
    np.savez_compressed(OUT, **res)
    print('wrote %s: %s' % (OUT, ', '.join('%s %s' % (k, np.shape(v)) for k, v in res.items())))


if __name__ == '__main__':
    main()
