"""compute_errors_batched (src/evaluation/eval.py:114-193) restated in float64 on this repository's eval_util and the numpy SMPL of
oracle/smpl_ref.py -- the checker for human_dynamics_b200.evaluate / csrc/eval.cu.

Everything is float64 except the one step the reference does in float32 on purpose: the prediction's keypoints are brought to pixels
as ((k + 1) * 0.5) * img_size in float32 (eval.py:131), which can move a PCK decision.
"""
import numpy as np

from src.evaluation import eval_util
from oracle.smpl_ref import SMPLRef
from oracle.eval_cases import make_eval_tubes  # noqa: F401  (the seeded test inputs)


def kps_to_pixels(kps_pred, img_size):
    """eval.py:131 in float32, one rounding per operation (numpy never contracts to FMA)."""
    k = np.asarray(kps_pred, np.float32)
    return ((k + np.float32(1)) * np.float32(0.5)) * np.float32(img_size)


def smpl_verts(smpl, poses, shapes):
    """compute_gpu_smpl (eval.py:68-90) in float64: the skinned vertices of axis-angle poses [N,72] and shapes [N,10]."""
    verts, _, _ = smpl(np.asarray(shapes, np.float64), np.asarray(poses, np.float64).reshape(len(shapes), 72), get_skin=True)
    return verts


def compute_errors_batched(kps_gt, kps_pred, joints_gt=None, joints_pred=None, poses_gt=None, poses_pred=None, shape_gt=None,
                           shapes_pred=None, img_size=224, has_3d=False, min_visible=6, compute_mesh=False, smpl_model=None):
    """The reference's error dict of one tube: same keys, same lengths; values in float64.  `smpl_model` (the un-pickled SMPL dict) is
    needed only with compute_mesh."""
    kps_gt = np.asarray(kps_gt, np.float64)
    errors_kp, errors_kp_pa, errors_kp_pck = eval_util.compute_error_kp(
        kps_gt=kps_gt, kps_pred=kps_to_pixels(kps_pred, img_size).astype(np.float64), alpha=0.05 * img_size,
        min_visible=min_visible)
    joints_pred = np.asarray(joints_pred, np.float64)
    errors = {'accel': eval_util.compute_accel(joints_pred), 'kp': errors_kp, 'kp_pa': errors_kp_pa, 'kp_pck': errors_kp_pck}
    if not has_3d:
        return errors
    joints_gt = np.asarray(joints_gt, np.float64)
    vis = np.sum(kps_gt[:, :14, 2], axis=1) > min_visible
    errors_accel = eval_util.compute_error_accel(joints_gt=joints_gt, joints_pred=joints_pred, vis=vis)
    if compute_mesh:
        smpl = SMPLRef(smpl_model, dtype=np.float64)
        shapes_gt = np.tile(np.asarray(shape_gt, np.float64), (len(poses_gt), 1))
        poses_pred_aa = np.array([eval_util.rot_mat_to_axis_angle(p) for p in np.asarray(poses_pred, np.float64)])
        zeros = np.zeros((len(poses_gt), 72))
        mesh_tpose = eval_util.compute_error_verts(smpl_verts(smpl, zeros, shapes_gt)[vis], smpl_verts(smpl, zeros, shapes_pred)[vis])
        mesh_posed = eval_util.compute_error_verts(smpl_verts(smpl, poses_gt, shapes_gt)[vis],
                                                   smpl_verts(smpl, poses_pred_aa, shapes_pred)[vis])
    else:
        mesh_posed, mesh_tpose = -1, -1
    errors_joints, errors_joints_pa = eval_util.compute_error_3d(gt3ds=joints_gt, preds=joints_pred, vis=vis)
    errors.update({'accel_error': errors_accel, 'mesh_posed': mesh_posed, 'mesh_tpose': mesh_tpose, 'pose': -1,
                   'joints': errors_joints, 'joints_pa': errors_joints_pa, 'shape': -1})
    return errors
