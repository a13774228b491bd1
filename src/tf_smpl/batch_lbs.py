""" Util functions for SMPL -- drop-in for the reference's src/tf_smpl/batch_lbs.py on CUDA tensors.

@@batch_skew
@@batch_rodrigues
@@batch_global_rigid_transformation

Same names / argument meaning as the reference (batch_lbs.py:15,42,133); eager on float32 CUDA
torch.Tensors, executed by libhd_b200.so.  A CPU tensor is an error (no fallback).  batch_rodrigues and
batch_global_rigid_transformation are differentiable (GPU backward kernels) when grad mode is on and an input requires grad.
"""
from human_dynamics_b200.smpl import batch_rodrigues as _rodrigues
from human_dynamics_b200.smpl import batch_global_rigid_transformation as _global_rigid
from human_dynamics_b200.smpl import RodriguesFunction, GlobalRigidFunction, _needs_grad, _cuda_f32


def batch_rodrigues(theta, name=None):
    """Theta is N x 3 -> N x 3 x 3   (batch_lbs.py:42-60)."""
    if _needs_grad(theta):
        _cuda_f32('batch_rodrigues', theta)
        return RodriguesFunction.apply(theta)
    return _rodrigues(theta)


def batch_global_rigid_transformation(Rs, Js, parent, rotate_base=False):
    """Rs N x 24 x 3 x 3, Js N x 24 x 3, parent 24 -> (new_J N x 24 x 3, A N x 24 x 4 x 4)   (batch_lbs.py:133-194)."""
    if _needs_grad(Rs, Js):
        _cuda_f32('batch_global_rigid_transformation', Rs, Js)
        return GlobalRigidFunction.apply(Rs, Js, parent, rotate_base)
    return _global_rigid(Rs, Js, parent, rotate_base)


def batch_rot2aa(Rs):
    """Rs is B x 3 x 3 -> B x 3 axis-angle   (batch_lbs.py:63-105)."""
    from human_dynamics_b200.smpl import batch_rot2aa as _rot2aa
    return _rot2aa(Rs)
