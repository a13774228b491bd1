"""Util functions implementing the camera -- drop-in for src/tf_smpl/projection.py:16-29.

@@batch_orth_proj_idrot
"""
from human_dynamics_b200.smpl import batch_orth_proj_idrot as _proj
from human_dynamics_b200.smpl import OrthProjFunction, _needs_grad, _cuda_f32


def batch_orth_proj_idrot(X, camera, name=None):
    """X is N x num_points x 3, camera is N x 3 -> N x num_points x 2: [s(x+tx), s(y+ty)].
    Differentiable w.r.t. X and camera (GPU backward kernel) when grad mode is on and either requires grad."""
    if _needs_grad(X, camera):
        _cuda_f32('batch_orth_proj_idrot', X, camera)
        return OrthProjFunction.apply(X, camera)
    return _proj(X, camera)


def batch_orth_proj_optcam(X, X_gt, name=None):
    """X N x K x 2 (or 3), X_gt N x K x 3 (x, y, visibility) -> (s(X + t) N x K x 2, best_cam N x 3) with the optimal camera of
    procrustes2d_vis, gradient stopped on the camera."""
    cam = procrustes2d_vis(X, X_gt)
    return cam[:, None, 0:1] * (X[:, :, :2] + cam[:, None, 1:]), cam


def procrustes2d_vis(X, X_target):
    """Optimal scale and translation in 2-D on the visible (vis > 0) points, the scale clipped to [0.7, 10], solved on the GPU by the
    loss kernels (csrc/losses.cu).  A frame without a visible point gets (0.7, 0, 0) (the reference divides 0 / 0 there)."""
    from human_dynamics_b200.objective import kp_loss
    assert X_target.dim() == 3
    return kp_loss(X_target.contiguous(), X.contiguous(), optcam=True)[1].detach()
