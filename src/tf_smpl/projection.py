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
