"""SMPL implementation as batch -- drop-in for the reference's src/tf_smpl/batch_smpl.py:26-162.

Specify joint types: 'cocoplus' (all regressor columns: 19 or 25) or 'lsp' (first 14).
To get original smpl joints, use self.J_transformed.
"""
import torch

from human_dynamics_b200.smpl import SMPLConstants, SMPLFunction, _needs_grad, _cuda_f32


class SMPL(object):
    def __init__(self, pkl_path, joint_type='cocoplus', dtype=torch.float32):
        """pkl_path is the path to a SMPL model pickle (or the already-loaded dict)."""
        if dtype not in (torch.float32, 'float32', None):
            raise ValueError('only float32 is supported on the CUDA path')
        self.consts = SMPLConstants(pkl_path, joint_type=joint_type)
        self.parents = self.consts.parents
        self.size = self.consts.size
        self.num_betas = self.consts.num_betas
        self.J_transformed = None

    def __call__(self, beta, theta, get_skin=False, name=None):
        """beta: N x 10, theta: N x 72 (or N x 24 x 3).

        Updates self.J_transformed (N x 24 x 3).  Returns joints (N x K x 3), or
        (verts N x 6890 x 3, joints, Rs N x 24 x 3 x 3) if get_skin.   (batch_smpl.py:89-162)

        When grad mode is on and beta or theta requires grad, all four outputs are on the autograd graph (backward on the GPU,
        human_dynamics_b200/csrc/smpl_grad.cu); otherwise no graph is built.
        """
        N = beta.shape[0]
        beta = beta.reshape(N, 10)
        theta = theta.reshape(N, 72)
        if beta.stride(1) != 1:
            beta = beta.contiguous()
        if theta.stride(1) != 1:
            theta = theta.contiguous()
        if _needs_grad(beta, theta):
            _cuda_f32('SMPL', beta, theta)
            verts, joints, Rs, self.J_transformed = SMPLFunction.apply(self.consts, beta, theta)
            return (verts, joints, Rs) if get_skin else joints
        o = self.consts.forward(beta.float(), theta.float())
        self.J_transformed = o['Jtr']
        if get_skin:
            return o['verts'], o['joints'], o['Rs']
        return o['joints']
