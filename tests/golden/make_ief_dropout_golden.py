"""Generates tests/golden/ief_dropout_v1.npz by EXECUTING THE REFERENCE'S OWN src/models.py in training mode:

    batch_pred_omega(is_training=True, predict_delta_keys=[-5, 5], use_delta_from_pred=True, use_optcam=True)
        -> call_hmr_ief -> hmr_ief -> encoder_fc3_dropout -> slim.dropout(0.5) after fc1 and fc2 (models.py:101-105)

over the numpy TensorFlow stand-in (oracle/ref_exec/stubs), with training-mode dropout installed over it by
oracle/ref_exec/training_dropout.py and its uniforms from a provider set here: the
uniforms of oracle/dropout_ref.py, keyed by the dropout op's variable scope (-> head: single_view_ief = 0, then _past5, _future5),
its occurrence within that scope (-> stage) and its name (dropout1 / dropout2 -> layer).  The vectors pin where the reference
applies dropout (after the ReLU, both layers, every stage, every head) and nn.dropout's arithmetic; TF's own random stream is not
reproduced (its op seeds come from graph construction).

Cases: call 0 (the pred strips) and call 1 (the hal strips), B=2, T=5, weights = synthetic.make_synthetic_weights(seed=1), features
stored.  Needs a checkout of the reference project, named by HD_REFERENCE_ROOT.  Run from the repo root:
    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_ief_dropout_golden.py
"""
import collections
import importlib.util
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
KEYS = (-5, 5)
SEED = 1
CASES = (('pred', 0, 7, 51), ('hal', 1, 2 ** 32 + 3, 52))        # (name, call, step, feature seed)
B, T = 2, 5
KEEP = 0.5


def _by_path(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def head_of(scope):
    m = re.fullmatch(r'single_view_ief(?:_(past|future)(\d+))?/3D_module', scope)
    assert m, scope
    if m.group(1) is None:
        return 0
    dt = int(m.group(2)) * (1 if m.group(1) == 'future' else -1)
    return 1 + sorted(KEYS).index(dt)


def main():
    gen = _by_path('_make_ref_exec_golden', os.path.join(ROOT, 'tests', 'golden', 'make_ref_exec_golden.py'))
    syn, _ = gen.setup_paths()
    dref = _by_path('_dropout_ref', os.path.join(ROOT, 'oracle', 'dropout_ref.py'))
    training_dropout = _by_path('_training_dropout', os.path.join(ROOT, 'oracle', 'ref_exec', 'training_dropout.py'))
    import tensorflow as tf
    from src import models
    weights = syn.make_synthetic_weights(seed=1)
    out = {'keys': np.array(KEYS), 'seed': np.uint64(SEED), 'keep_prob': np.float64(KEEP), 'B': B, 'T': T}
    for name, call, step, fseed in CASES:
        seen = []
        count = collections.Counter()

        def provider(path):
            scope, op = path.rsplit('/', 1)
            layer = {'dropout1': 0, 'dropout2': 1}[op]
            head = head_of(scope)
            stage = count[(head, layer)]
            count[(head, layer)] += 1
            site = dref.site(call, head, stage, layer)
            seen.append(path)

            def uniform(shape):
                n, c = shape
                return dref.uniform(dref.words(SEED, step, site, n, c))
            return uniform
        tf.reset_default_graph()
        training_dropout.install(provider)
        feats = np.random.RandomState(fseed).normal(0, 1, size=(B, T, 2048)).astype(np.float32)
        omega_mean = np.tile(np.asarray(weights['mean_param'], np.float32).reshape(1, 85), (B * T, 1))
        om, deltas = models.batch_pred_omega(input_features=tf.constant(feats), batch_size=B, is_training=True, num_output=85,
                                             omega_mean=tf.constant(omega_mean), sequence_length=T, scope='single_view_ief',
                                             predict_delta_keys=list(KEYS), use_delta_from_pred=True, use_optcam=True)
        for v in tf.global_variables():
            if not v.initialized:
                v.load(weights[v.op_name])
        r = tf.Session().run({'omega': om, 'deltas': deltas})
        training_dropout.uninstall()
        out['%s_call' % name] = np.int64(call)
        out['%s_step' % name] = np.uint64(step)
        out['%s_feats' % name] = feats
        out['%s_omega' % name] = r['omega']
        for dt, v in r['deltas'].items():
            out['%s_delta_%d' % (name, dt)] = v
        out['%s_dropout_ops' % name] = np.array(seen)
    path = os.path.join(ROOT, 'tests', 'golden', 'ief_dropout_v1.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes,', len(out), 'arrays')


if __name__ == '__main__':
    main()
