"""src/ops.py of the reference: the training losses (ops.py:14-182) and a duplicate of the IEF wrappers (ops.py:184,270).  BASELINE.json
names `src/ops.batch_orth_proj_idrot`; export it here as an alias.

The encoder losses (keypoints, 3-D, smoothness) run on the GPU loss kernels (csrc/losses.cu) as single-term objectives, so they share
one path with human_dynamics_b200.objective; tensors are float32 CUDA.  The adversarial prior's losses (ops.py:127-137, 160) are torch
expressions over the discriminator's outputs (src/discriminators.py) and the predicted shapes."""
import torch

from src.tf_smpl.projection import batch_orth_proj_idrot  # noqa: F401
from src.models import call_hmr_ief, hmr_ief              # noqa: F401


def compute_loss_e_kp_optcam(kp_gt, kp_pred, name=None):
    """kp_gt (B,T,K,3), kp_pred (B,T,K,2) -> (L1 loss after the optimal camera of procrustes2d_vis, best_cam (B,T,3))."""
    from human_dynamics_b200.objective import kp_loss
    B, T = kp_gt.shape[0], kp_gt.shape[1]
    loss, cam = kp_loss(kp_gt.reshape(B * T, -1, 3), kp_pred.reshape(B * T, -1, 2), optcam=True)
    return loss, cam.reshape(B, T, 3)


def compute_loss_e_kp(kp_gt, kp_pred, name=None):
    """sum v * |x - x_hat| / (2 * #{v != 0}) over kp_gt (..., 3) and kp_pred (..., 2)."""
    from human_dynamics_b200.objective import kp_loss
    K = kp_gt.shape[-2] if kp_gt.dim() >= 3 else 1
    return kp_loss(kp_gt.reshape(-1, K, 3).contiguous(), kp_pred.reshape(-1, K, 2).contiguous())[0]


def compute_loss_e_3d(poses_gt, poses_pred, shapes_gt, shapes_pred, joints_gt, joints_pred, batch_size, has_gt3d_smpl,
                      has_gt3d_joints):
    """(pose, shape, joints) losses of ops.py:59-84; joints (B,T,14,3) are aligned by the pelvis."""
    from human_dynamics_b200.objective import mse_loss
    assert joints_gt.dim() == 4
    jg = joints_gt.reshape(-1, joints_gt.shape[2] * 3)
    jp = joints_pred.reshape(-1, joints_pred.shape[2] * 3)
    return (compute_loss_mse(poses_gt.reshape(batch_size, -1), poses_pred.reshape(batch_size, -1), has_gt3d_smpl),
            compute_loss_mse(shapes_gt.reshape(batch_size, -1), shapes_pred.reshape(batch_size, -1), has_gt3d_smpl),
            mse_loss(jp.contiguous(), jg.contiguous(), has_gt3d_joints.reshape(-1), scale=0.5, align=True))


def compute_loss_mse(params_gt, params_pred, has_gt3d):
    """0.5 * mean squared error over the rows with has_gt3d != 0 (N x D)."""
    from human_dynamics_b200.objective import mse_loss
    N = params_pred.shape[0]
    return mse_loss(params_pred.reshape(N, -1).contiguous(), params_gt.reshape(N, -1).contiguous(), has_gt3d.reshape(N), scale=0.5)


def compute_loss_e_smooth(joints_prev, joints_curr):
    from human_dynamics_b200.objective import mse_loss
    D = joints_prev.shape[-1]
    return mse_loss(joints_prev.reshape(-1, D).contiguous(), joints_curr.reshape(-1, D).contiguous(), None, scale=0.5)


def compute_loss_e_fake(out_fake):
    return ((out_fake - 1) ** 2).sum(dim=1).mean()


def compute_loss_d_fake(out_fake):
    return (out_fake ** 2).sum(dim=1).mean()


def compute_loss_d_real(out_real):
    return ((out_real - 1) ** 2).sum(dim=1).mean()


def compute_deltas_batched(poses_prev, poses_curr):
    """R_prev R_curr^T for (B,T,24,3,3) rotations."""
    assert poses_prev.shape == poses_curr.shape and poses_prev.dim() == 5 and tuple(poses_prev.shape[2:]) == (24, 3, 3)
    return torch.matmul(poses_prev, poses_curr.transpose(-1, -2))


def compute_loss_shape(shapes):
    """L2 loss on shapes."""
    return shapes.square().mean()


def align_by_pelvis(joints):
    """joints N x 14 x 3 in LSP order, minus the midpoint of the hips (joints 2 and 3)."""
    pelvis = (joints[:, 3, :] + joints[:, 2, :]) / 2.
    return joints - pelvis.unsqueeze(1)
