"""Generates tests/golden/losses_v1.npz by EXECUTING THE REFERENCE'S OWN SOURCE: src/ops.py, src/tf_smpl/projection.py, src/omega.py
(OmegasGt, and OmegasPred.compute_smpl with the predicted joints and rotations fed in through its `smpl` callable) and, unbound over a
namespace `self`, trainer_sequence_fc.HMRSequenceTrainer.compute_losses_deltas / compute_losses_batched / compute_losses_prior /
gather_losses, in build_model's order (the hallucinated sets, the prediction, the delta heads, the prior).  It runs over the numpy
TensorFlow stand-in in oracle/ref_exec, set up as make_ref_exec_golden.py does; extend_standin() adds, in this process only, what these
files need that the stand-in does not have:
  - tf.losses.absolute_difference / mean_squared_error with SUM_BY_NONZERO_WEIGHTS: the weights are broadcast to the loss's shape and
    the weighted sum is divided by the number of non-zero weights (0 when there are none);
  - tf.split into equal parts along axis 0; tf.summary.scalar / histogram / merge, tf.get_collection and tf.GraphKeys (summaries
    are not computed);
  - slim.flatten and Tensor ** (as make_dpose_golden.py), and the trainer's imports (tensorflow.python.ops.control_flow_ops) as stubs.
The stand-in's own stop_gradient, matrix_inverse and trace are used.  The namespace `self` holds what HMRSequenceTrainer.__init__ would
hold: its self.losses initial dict (trainer_sequence_fc.py:235-274) and self.loss_weights (:280-310) at the default flags, restated.

Configuration: B = 3, T = 10, K = 25, delta_t = -5, 5, predict_delta, do_hallucinate, do_hallucinate_preds, use_3d_label.  Inputs
from seeds (inputs() below): has_3d = joints only / SMPL only / none per clip, visibility mixing 0, 0.5 and 1 (one keypoint always
visible, so that no optimal-camera frame is empty: the reference's value is NaN there), one frame of the first hallucinated past set
mirrored against its label so that its optimal scale hits the 0.7 clip.  The reference computes in float64 here (float32-valued inputs
fed as float64).

Stored: the inputs (omega [S,B,T,85], joints [S,B,T,K,3], rots [S,B,T,216] per prediction set in pred_poses_all order; labels, poses,
shape, gt3ds, has_3d, strips, pred_strips, mocap), gt_rots (OmegasGt's rotations), every named loss under its key, e_loss, d_loss, and
each delta set's best cameras (cam_<group>_<dt> [B, T-|dt|, 3]).  D_pose's variables are synthetic.make_dpose_weights(3, 0.1).

Needs a checkout of the reference project, named by HD_REFERENCE_ROOT.  Run from the repo root:
    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_losses_golden.py            (writes tests/golden/losses_v1.npz)
    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_losses_golden.py --check    (exit 0 when it reproduces the file)
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'losses_v1.npz')
B, T, K, DTS = 3, 10, 25, (-5, 5)
SETS = [('hal', 0), ('hal', -5), ('hal', 5), ('pred', 0), ('dt', -5), ('dt', 5)]     # pred_poses_all order


def _by_path(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def inputs():
    """The seeded inputs, float32."""
    rng = np.random.RandomState(20)
    S = len(SETS)
    lab = rng.normal(0, 0.5, size=(B, 1, K, 3)) + rng.normal(0, 0.05, size=(B, T, K, 3))
    lab[..., 2] = rng.choice([0., 1., 1., 0.5], size=(B, T, K))
    lab[:, :, 0, 2] = 1.
    js = rng.normal(0, 0.5, size=(S, B, T, K, 3))
    js[..., :2] = lab[None, ..., :2] / rng.uniform(0.8, 1.6, size=(S, B, T, 1, 1)) + rng.normal(0, 0.1, size=(S, B, T, K, 2))
    s = SETS.index(('hal', -5))        # its window: prediction frames 5.., label frames ..4
    lab[0, 0, :, 2] = 1.
    js[s, 0, 5, :, 0] = -lab[0, 0, :, 0]
    js[s, 0, 5, :, 1] = lab[0, 0, :, 1]
    om = rng.normal(0, 0.3, size=(S, B, T, 85))
    om[..., 0] = rng.uniform(0.6, 1.4, size=(S, B, T))
    strips = rng.normal(0, 1, size=(B, T, 2048))
    n_fake = S * B * T
    aa = rng.normal(0, 0.5, size=(n_fake * 24, 3))
    th = np.linalg.norm(aa, axis=1)[:, None, None]
    k = aa / th[:, :, 0]
    Km = np.zeros((n_fake * 24, 3, 3))
    Km[:, 0, 1], Km[:, 0, 2], Km[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    Km = Km - Km.transpose(0, 2, 1)
    mocap = (np.eye(3) + np.sin(th) * Km + (1 - np.cos(th)) * Km @ Km).reshape(n_fake, 216)
    x = {'omega': om, 'joints': js, 'rots': rng.normal(0, 0.5, size=(S, B, T, 216)), 'labels': lab,
         'poses': rng.normal(0, 0.4, size=(B, T, 72)), 'shape': rng.normal(0, 0.5, size=(B, 10)),
         'gt3ds': rng.normal(0, 0.5, size=(B, T, 14, 3)), 'has_3d': np.array([[1, 0], [0, 1], [0, 0]], np.float64),
         'strips': strips, 'pred_strips': strips + rng.normal(0, 0.3, size=(B, T, 2048)), 'mocap': mocap}
    return {k: np.ascontiguousarray(v, np.float32) for k, v in x.items()}


def extend_standin(tf):
    dp = _by_path('_make_dpose_golden', os.path.join(HERE, 'make_dpose_golden.py'))
    dp.extend_standin(tf)

    def _sum_by_nonzero(loss, weights):
        w = tf.convert_to_tensor(weights)
        return tf._binary(lambda l, ww: np.sum(np.broadcast_to(ww, l.shape) * l) / max(np.count_nonzero(np.broadcast_to(ww, l.shape)), 1),
                          'sum_by_nonzero')(loss, w)
    losses = types.SimpleNamespace(
        absolute_difference=lambda labels, predictions, weights=1.0, **kw: _sum_by_nonzero(tf.abs(labels - predictions), weights),
        mean_squared_error=lambda labels, predictions, weights=1.0, **kw: _sum_by_nonzero(tf.square(labels - predictions), weights))
    tf.losses = losses
    tf.summary = types.SimpleNamespace(scalar=lambda *a, **k: None, histogram=lambda *a, **k: None, merge=lambda *a, **k: None)
    tf.GraphKeys = types.SimpleNamespace(UPDATE_OPS='update_ops')
    tf.get_collection = lambda *a, **k: []

    def split(value, num, axis=0, name=None):          # tf.split into `num` equal parts along axis 0 (the only use here)
        assert axis == 0
        n = int(value.shape[0]) // num
        return [value[i * n:(i + 1) * n] for i in range(num)]
    tf.split = split
    for name in ('tensorflow.python', 'tensorflow.python.ops', 'tensorflow.python.ops.control_flow_ops'):
        sys.modules.setdefault(name, types.ModuleType(name))


def run_reference():
    gen = _by_path('_make_ref_exec_golden', os.path.join(HERE, 'make_ref_exec_golden.py'))
    syn, _ = gen.setup_paths()
    import tensorflow as tf
    extend_standin(tf)
    import src.util
    render = sys.modules.setdefault('src.util.render', types.ModuleType('src.util.render'))
    render.nmr_renderer = sys.modules['src.util.render.nmr_renderer']        # `import a.b.c as m` reads the attributes
    src.util.render = render
    from src.omega import OmegasGt, OmegasPred
    from src.discriminators import PoseDiscriminator
    import src.trainer_sequence_fc as TR
    x = inputs()
    f64 = {k: v.astype(np.float64) for k, v in x.items()}
    ph = {k: tf.placeholder(tf.float64, v.shape) for k, v in f64.items()}
    config = types.SimpleNamespace(batch_size=B, num_kps=K, T=T)
    omegas_gt = OmegasGt(config=config, poses_aa=tf.reshape(ph['poses'], (B, T, 24, 3)), shapes=ph['shape'], joints=ph['gt3ds'],
                         kps=ph['labels'])

    def make_pred(s, use_optcam):
        def smpl(beta, theta, get_skin=False):
            return (tf.zeros((B * T, 6890, 3), tf.float64), tf.reshape(ph['joints'][s], (B * T, K, 3)),
                    tf.reshape(ph['rots'][s], (B * T, 24, 3, 3)))
        o = OmegasPred(config=config, smpl=smpl, use_optcam=use_optcam, vis_max_batch=2, batch_size=B, is_training=True)
        o.append_batched(ph['omega'][s])
        o.compute_smpl()
        return o
    preds = {key: make_pred(s, key[1] != 0) for s, key in enumerate(SETS)}
    self = types.SimpleNamespace(
        batch_size=B, sequence_length=T, omegas_gt=omegas_gt, omegas_pred=preds[('pred', 0)], use_3d_label=True,
        has_gt3d_joints=ph['has_3d'][:, 0], has_gt3d_smpl=ph['has_3d'][:, 1], do_hallucinate=True, use_hmr_only=False,
        movie_strip=ph['strips'], pred_movie_strip=ph['pred_strips'], poses_real_loader=ph['mocap'], pred_poses_all=[],
        pred_shapes_all=[], disc_pose=PoseDiscriminator(1e-4), summaries_list=[], loss_proportions={},
        omegas_pred_hal={dt: preds[('hal', dt)] for dt in (0,) + DTS}, omegas_delta={dt: preds[('dt', dt)] for dt in DTS})
    self.add_scalar_summary = lambda name, value: None
    self.setup_disc_summary = lambda poses_out: None
    z = tf.constant(0.)
    # trainer_sequence_fc.py:235-274 (predict_delta, do_hallucinate, do_hallucinate_preds) and :280-310 at the default flags
    self.losses = {k: z for k in ('d_pose', 'e_const', 'e_joints', 'e_kp', 'e_pose', 'e_shape', 'e_smpl', 'e_joints_dt_future',
                                  'e_kp_dt_future', 'e_smpl_dt_future', 'e_joints_dt_past', 'e_kp_dt_past', 'e_smpl_dt_past',
                                  'e_hallucinate', 'e_joints_hal', 'e_kp_hal', 'e_smpl_hal', 'e_joints_hal_future', 'e_kp_hal_future',
                                  'e_smpl_hal_future', 'e_joints_hal_past', 'e_kp_hal_past', 'e_smpl_hal_past')}
    lw = {'d_pose': 1., 'e_const': 1., 'e_pose': 1., 'e_shape': 1., 'e_hallucinate': 1.}
    for k in self.losses:
        if k not in lw:
            lw[k] = 60.
    self.loss_weights = lw
    C = TR.HMRSequenceTrainer
    C.compute_losses_deltas(self, omegas_dict=self.omegas_pred_hal, suffix_future='_hal_future', suffix_past='_hal_past',
                            suffix_present='_hal')
    C.compute_losses_batched(self)
    C.compute_losses_deltas(self, omegas_dict=self.omegas_delta, suffix_future='_dt_future', suffix_past='_dt_past', suffix_present='_dt')
    C.compute_losses_prior(self)
    dw = syn.make_dpose_weights(3, bias_scale=0.1)
    for v in self.disc_pose.get_vars():
        v.load(dw[v.op_name].astype(np.float64))
    C.gather_losses(self)
    fetch = dict(self.losses)
    fetch.update(e_loss=self.e_loss, d_loss=self.d_loss, gt_rots=tf.reshape(omegas_gt.get_poses_rot(), (B, T, 216)))
    for key in SETS:
        if key[1] != 0:
            dt = key[1]
            cams = preds[key].get_cams()
            fetch['cam_%s_%d' % key] = cams[:, abs(dt):] if dt < 0 else cams[:, :T - dt]
    with tf.Session() as sess:
        got = sess.run(fetch, feed_dict={ph[k]: f64[k] for k in ph})
    res = dict(x)
    res.update({k: np.asarray(v, np.float64) for k, v in got.items()})
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
