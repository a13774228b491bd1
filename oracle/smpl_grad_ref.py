"""ORACLE (test infrastructure, not product): differentiable torch-CPU restatement of the reference SMPL path.

The same functions as oracle/smpl_ref.py -- SMPLRef, batch_rodrigues (with the +1e-8 shift inside the norm), the FK of
batch_global_rigid_transformation and batch_orth_proj_idrot -- written with torch ops in the same operation order, so torch
autograd differentiates them.  `dtype` is torch.float64 (the truth) or torch.float32.

PARITY STATUS: the forward is pinned to oracle/smpl_ref.py (tests/test_smpl_grad_cpu.py, 1e-12 in float64), and the gradients
are pinned to central finite differences by torch.autograd.gradcheck in float64, which does not rely on autograd being right.
TensorFlow's own gradient kernels for the reference graph stay unpinned: TF 1.8 cannot run here.

Only tests/ may import this module.
"""
from __future__ import annotations

import numpy as np
import torch


def batch_skew(vec):
    """src/tf_smpl/batch_lbs.py:15-39 -> [M,3,3] skew matrices."""
    z = torch.zeros_like(vec[:, 0])
    x, y, w = vec[:, 0], vec[:, 1], vec[:, 2]
    return torch.stack([z, -w, y, w, z, -x, -y, x, z], dim=1).reshape(-1, 3, 3)


def batch_rodrigues(theta):
    """src/tf_smpl/batch_lbs.py:42-60.  theta [M,3] -> R [M,3,3]."""
    shifted = theta + 1e-8
    angle = torch.sqrt(torch.sum(shifted * shifted, dim=1))[:, None]
    r = (theta / angle)[:, :, None]
    angle = angle[:, :, None]
    cos, sin = torch.cos(angle), torch.sin(angle)
    outer = torch.matmul(r, r.transpose(1, 2))
    eyes = torch.eye(3, dtype=theta.dtype).expand(theta.shape[0], 3, 3)
    return cos * eyes + (1 - cos) * outer + sin * batch_skew(r[:, :, 0])


def batch_global_rigid_transformation(Rs, Js, parent, rotate_base=False):
    """src/tf_smpl/batch_lbs.py:133-194.  Rs [N,24,3,3], Js [N,24,3] -> new_J [N,24,3], A [N,24,4,4]."""
    N, nj = Rs.shape[0], len(parent)
    dt = Rs.dtype
    if rotate_base:
        rot_x = torch.tensor([[1, 0, 0], [0, -1, 0], [0, 0, -1]], dtype=dt)
        root_rotation = torch.matmul(Rs[:, 0], rot_x)
    else:
        root_rotation = Rs[:, 0]
    Js_e = Js[..., None]

    def make_A(R, t):
        R_homo = torch.cat([R, torch.zeros((N, 1, 3), dtype=dt)], dim=1)
        t_homo = torch.cat([t, torch.ones((N, 1, 1), dtype=dt)], dim=1)
        return torch.cat([R_homo, t_homo], dim=2)

    results = [make_A(root_rotation, Js_e[:, 0])]
    for i in range(1, nj):
        j_here = Js_e[:, i] - Js_e[:, int(parent[i])]
        results.append(torch.matmul(results[int(parent[i])], make_A(Rs[:, i], j_here)))
    results = torch.stack(results, dim=1)
    new_J = results[:, :, :3, 3]
    Js_w0 = torch.cat([Js_e, torch.zeros((N, nj, 1, 1), dtype=dt)], dim=2)
    init_bone = torch.matmul(results, Js_w0)
    init_bone = torch.cat([torch.zeros((N, nj, 4, 3), dtype=dt), init_bone], dim=3)
    return new_J, results - init_bone


def batch_orth_proj_idrot(X, camera):
    """src/tf_smpl/projection.py:16-29."""
    camera = camera.reshape(-1, 1, 3)
    X_trans = X[:, :, :2] + camera[:, :, 1:]
    shape = X_trans.shape
    return (camera[:, :, 0] * X_trans.reshape(shape[0], -1)).reshape(shape)


class SMPLGradRef(object):
    """src/tf_smpl/batch_smpl.py:26-162 in torch (the model constants are plain tensors, not leaves of the graph)."""

    def __init__(self, model: dict, joint_type='cocoplus', dtype=torch.float64):
        def t(a):
            a = np.asarray(a.todense()) if hasattr(a, 'todense') else np.asarray(a)
            return torch.from_numpy(a.astype(np.float64)).to(dtype)
        self.dtype = dtype
        self.v_template = t(model['v_template'])
        V = self.v_template.shape[0]
        self.size = [V, 3]
        nb = model['shapedirs'].shape[-1]
        self.shapedirs = t(np.reshape(np.asarray(model['shapedirs']), [-1, nb]).T)
        self.J_regressor = t(model['J_regressor']).T
        self.posedirs = t(np.reshape(np.asarray(model['posedirs']), [-1, model['posedirs'].shape[-1]]).T)
        self.parents = np.asarray(model['kintree_table'])[0].astype(np.int64)
        self.parents = np.where(self.parents >= 2 ** 31, -1, self.parents)
        self.weights = t(model['weights'])
        self.joint_regressor = t(model['cocoplus_regressor']).T
        if joint_type == 'lsp':
            self.joint_regressor = self.joint_regressor[:, :14]
        self.J_transformed = None

    def __call__(self, beta, theta, get_skin=False):
        N, V = beta.shape[0], self.size[0]
        v_shaped = torch.matmul(beta, self.shapedirs).reshape(-1, V, 3) + self.v_template
        J = torch.stack([torch.matmul(v_shaped[:, :, c], self.J_regressor) for c in range(3)], dim=2)
        Rs = batch_rodrigues(theta.reshape(-1, 3)).reshape(-1, 24, 3, 3)
        pose_feature = (Rs[:, 1:] - torch.eye(3, dtype=self.dtype)).reshape(-1, 207)
        v_posed = torch.matmul(pose_feature, self.posedirs).reshape(-1, V, 3) + v_shaped
        self.J_transformed, A = batch_global_rigid_transformation(Rs, J, self.parents)
        W = self.weights.expand(N, V, 24)
        T = torch.matmul(W, A.reshape(N, 24, 16)).reshape(N, -1, 4, 4)
        v_posed_homo = torch.cat([v_posed, torch.ones((N, V, 1), dtype=self.dtype)], dim=2)
        verts = torch.matmul(T, v_posed_homo[..., None])[:, :, :3, 0]
        joints = torch.stack([torch.matmul(verts[:, :, c], self.joint_regressor) for c in range(3)], dim=2)
        if get_skin:
            return verts, joints, Rs
        return joints
