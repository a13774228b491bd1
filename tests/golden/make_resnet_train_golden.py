"""Generates tests/golden/resnet_train_bn_v1.npz by EXECUTING THE REFERENCE'S OWN src/models.py: encoder_resnet(x, is_training=True), the
call trainer_sequence_fc.py:562-575 makes on every iteration with precomputed_phi=False, then one sess.run of the UPDATE_OPS the
trainer groups with e_loss (trainer_sequence_fc.py:745-750).  It runs over the numpy TensorFlow stand-in, set up as
make_ref_exec_golden.py does, with oracle/ref_exec/train_bn.py installed: the training-mode batch_norm [TF-ext] the inference-only
stand-in lacks.

Inputs (regenerated from seeds, not stored): the golden weights (synthetic.make_synthetic_weights(seed=1)) and FRAMES frames of
synthetic.make_images(FRAMES, seed=SEED, size=SIZE).  Stored: phi [FRAMES, 2048]; for each of the 49 batch-norm scopes (index i in
`scopes` order) mean_<i> / var_<i>, the batch moments (biased variance), and moving_mean_<i> / moving_variance_<i> after the one run of
the update ops.  The stand-in computes in float32.

Needs a checkout of the reference project, named by HD_REFERENCE_ROOT.  Run from the repo root:
    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_resnet_train_golden.py            (about a minute)
"""
import importlib.util
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'resnet_train_bn_v1.npz')
FRAMES, SEED, SIZE = 3, 71, 224


def _by_path(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    rx = _by_path('_make_ref_exec_golden', os.path.join(HERE, 'make_ref_exec_golden.py'))
    syn, _ = rx.setup_paths()
    train_bn = _by_path('_train_bn', os.path.join(ROOT, 'oracle', 'ref_exec', 'train_bn.py'))
    train_bn.install()
    import tensorflow as tf
    from src import models
    weights = syn.make_synthetic_weights(seed=1)
    images = syn.make_images(FRAMES, seed=SEED, size=SIZE)
    tf.reset_default_graph()
    phi, scope = models.encoder_resnet(tf.constant(images), is_training=True, reuse=False)
    assert scope == 'resnet_v2_50'
    for v in tf.global_variables():
        v.load(weights[v.op_name])
    sess = tf.Session()
    moments = tf.get_collection(train_bn.MOMENTS)
    updates = tf.get_collection(tf.GraphKeys.UPDATE_OPS)
    assert len(moments) == 49 and len(updates) == 98, (len(moments), len(updates))
    out = {'frames': np.array(FRAMES), 'seed': np.array(SEED), 'size': np.array(SIZE)}
    r = sess.run({'phi': phi, 'moments': [(m, v) for _, m, v in moments]})
    out['phi'] = r['phi']
    out['scopes'] = np.array([s for s, _, _ in moments])
    for i, (m, v) in enumerate(r['moments']):
        out['mean_%d' % i], out['var_%d' % i] = m, v
    sess.run(tf.group(*updates))
    by_name = {v.op_name: v for v in tf.global_variables()}
    for i, s in enumerate(out['scopes']):
        out['moving_mean_%d' % i] = np.array(by_name[s + '/moving_mean'].value)
        out['moving_variance_%d' % i] = np.array(by_name[s + '/moving_variance'].value)
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
