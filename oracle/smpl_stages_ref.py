"""ORACLE (test infrastructure, not product): the SMPL forward restated stage by stage in torch float64.

oracle/smpl_ref.py restates the reference's whole call (src/tf_smpl/batch_smpl.py:89-162) on numpy; this module splits the
same arithmetic at the boundaries of the device kernels (smpl_pose_kernel, the blend GEMM, smpl_skin / smpl_lbs / smpl_lbs_tc,
smpl_joints_kernel, orth_proj_kernel), so a test can feed each stage the kernel's own upstream outputs and judge that stage
alone.  Every function takes torch tensors and computes in float64 on their device: the GPU tests run it on the H100 at
batches of thousands of poses, the CPU tests (tests/test_oracle_smpl.py) pin it to smpl_ref.SMPLRef(dtype=float64) and
smpl_ref.batch_global_rigid_transformation.

Stages, in the reference's operation order:
  rodrigues       batch_lbs.py:42-60: angle = ||theta + 1e-8||, r = theta / angle, R = cos I + (1 - cos) r r^T + sin [r]x
  rest_joints     J = J_template + beta . J_shapedirs (J_regressor . v_shaped, batch_smpl.py:115-118, precomposed)
  forward_kinematics  batch_lbs.py:133-194, one depth level of the tree at a time; A = [R | t - R J]
  blend_coef / blend  v_posed = v_template + [beta | (R_j - I), j = 1..23] . dirs (batch_smpl.py:110-112,127-133)
  skin            T = sum_k w_k A_k applied to [v_posed; 1] (batch_smpl.py:141-151)
  regress         joints = regressor . verts (batch_smpl.py:154-157; the kernel walks the CSC form of the same matrix)
  orth_proj       s * (xy + t) (projection.py:16-29)

Only tests/ may import this module.
"""
from __future__ import annotations

import numpy as np
import torch

F64 = torch.float64


def _t(x, device=None):
    """A float64 tensor of x (a tensor keeps its device unless one is given; an array goes to `device`, default CPU)."""
    if isinstance(x, torch.Tensor):
        return x.to(dtype=F64, device=device if device is not None else x.device)
    return torch.as_tensor(np.asarray(x), dtype=F64, device=device)


def tree_depths(parents):
    """Depth of every joint of a kinematic tree with parent[i] < i (the root, whose parent entry is ignored, has depth 0)."""
    p = [int(x) for x in np.asarray(parents).astype(np.int64).tolist()]
    depth = [0] * len(p)
    for i in range(1, len(p)):
        if not 0 <= p[i] < i:
            raise ValueError('parents must satisfy 0 <= parent[i] < i, got parent[%d] = %d' % (i, p[i]))
        depth[i] = depth[p[i]] + 1
    return depth


def test_trees():
    """Kinematic trees (24 joints, parent[i] < i) that bound what the level-by-level FK has to handle: SMPL's own (depth 9), a chain
    0 -> 1 -> ... -> 23 (depth 23, one joint per level), a star (depth 1, 23 joints on one level) and two seeded random trees."""
    from human_dynamics_b200.synthetic import SMPL_PARENTS
    trees = {'smpl': np.asarray(SMPL_PARENTS, np.int64),
             'chain': np.arange(-1, 23, dtype=np.int64),
             'star': np.array([-1] + [0] * 23, np.int64)}
    for seed in (1, 2):
        rng = np.random.RandomState(seed)
        trees['random%d' % seed] = np.array([-1] + [rng.randint(0, i) for i in range(1, 24)], np.int64)
    return trees


def with_tree(model, parents):
    """A copy of a model dict whose kintree_table has the given parents (stored as the pickles do: uint32, root = 2^32 - 1)."""
    m = dict(model)
    m['kintree_table'] = np.stack([np.asarray(parents, np.int64).astype(np.uint32), np.arange(24, dtype=np.uint32)])
    return m


def rodrigues(theta):
    """theta [..., 3] -> R [..., 3, 3] (batch_lbs.py:42-60): the 1e-8 shift goes into the angle only."""
    th = _t(theta)
    shifted = th + 1e-8
    angle = torch.sqrt((shifted * shifted).sum(-1, keepdim=True))
    r = th / angle
    c, s = torch.cos(angle)[..., None], torch.sin(angle)[..., None]
    rx, ry, rz = r.unbind(-1)
    z = torch.zeros_like(rx)
    skew = torch.stack([z, -rz, ry, rz, z, -rx, -ry, rx, z], -1).reshape(r.shape[:-1] + (3, 3))
    eye = torch.eye(3, dtype=F64, device=th.device)
    return c * eye + (1.0 - c) * (r[..., :, None] * r[..., None, :]) + s * skew


def rest_joints(beta, J_template, J_shapedirs):
    """beta [N,10], J_template [24,3] (or [72]), J_shapedirs [10,72] -> J [N,24,3]."""
    b = _t(beta)
    return (_t(J_template, b.device).reshape(1, 72) + b @ _t(J_shapedirs, b.device)).reshape(-1, 24, 3)


def forward_kinematics(Rs, J, parents, rotate_base=False):
    """Rs [N,24,3,3] local rotations, J [N,24,3] rest joints -> (Jtr [N,24,3] world joints, A [N,24,3,4] = [Rw | tw - Rw J]).

    Level by level: every joint of depth d composes its parent's world transform (depth d - 1, final by then) with its own."""
    Rl, J = _t(Rs), _t(J)
    if rotate_base:                                                     # Rs[:, 0] . diag(1, -1, -1), batch_lbs.py:151-156
        Rl = Rl.clone()
        Rl[:, 0] = Rl[:, 0] * torch.tensor([1.0, -1.0, -1.0], dtype=F64, device=Rl.device)
    par = np.asarray(parents).astype(np.int64)
    depth = tree_depths(par)
    par[0] = 0
    tl = J - J[:, par]
    tl[:, 0] = J[:, 0]
    Rw, tw = Rl.clone(), tl.clone()
    for level in range(1, max(depth) + 1):
        idx = [i for i in range(len(depth)) if depth[i] == level]
        pi = par[idx].tolist()
        pR, pt = Rw[:, pi], tw[:, pi]
        Rw[:, idx] = pR @ Rl[:, idx]
        tw[:, idx] = (pR @ tl[:, idx, :, None])[..., 0] + pt
    A = torch.cat([Rw, (tw - (Rw @ J[..., None])[..., 0])[..., None]], -1)
    return tw, A


def blend_coef(beta, Rs):
    """The blend GEMM's operand row [beta (10) | R_j - I, j = 1..23 (207)] -> [N, 217]."""
    b, R = _t(beta), _t(Rs)
    eye = torch.eye(3, dtype=F64, device=R.device)
    return torch.cat([b, (R[:, 1:] - eye).reshape(-1, 207)], 1)


def blend(beta, Rs, v_template, dirs):
    """v_posed [N, 3V] = v_template + coef . dirs; v_template [3V] (or [V,3]), dirs [217, 3V] (10 shape rows, then 207 pose rows)."""
    c = blend_coef(beta, Rs)
    return _t(v_template, c.device).reshape(1, -1) + c @ _t(dirs, c.device)


def skin(v_posed, A, weights, chunk=256):
    """v_posed [N,V,3], A [N,24,3,4], weights [V,24] (dense) -> verts [N,V,3]: (sum_k w_k A_k) [v; 1], `chunk` poses at a time."""
    vp, A = _t(v_posed), _t(A)
    W = _t(weights, vp.device)
    N, V = vp.shape[0], vp.shape[1]
    out = torch.empty((N, V, 3), dtype=F64, device=vp.device)
    for n0 in range(0, N, chunk):
        T = (W @ A[n0:n0 + chunk].reshape(-1, 24, 12)).reshape(-1, V, 3, 4)
        out[n0:n0 + chunk] = (T[..., :3] @ vp[n0:n0 + chunk, :, :, None])[..., 0] + T[..., 3]
    return out


def regress(verts, regressor):
    """verts [N,V,3], regressor [K,V] -> joints [N,K,3]."""
    v = _t(verts)
    return torch.einsum('kv,nvc->nkc', _t(regressor, v.device), v)


def orth_proj(X, cam):
    """X [N,P,3], cam [N,3] -> [N,P,2] = s * (xy + t)."""
    X, c = _t(X), _t(cam)
    c = c.to(X.device)
    return c[:, None, 0:1] * (X[..., :2] + c[:, None, 1:3])


def model_constants(model, joint_type='cocoplus'):
    """The float64 constants of a model dict (synthetic.make_synthetic_smpl's keys, dense arrays): what SMPLConstants packs, before
    its float32 rounding."""
    def dense(m):
        return np.asarray(m.todense()) if hasattr(m, 'todense') else np.asarray(m)
    v_template = dense(model['v_template']).astype(np.float64)
    V = v_template.shape[0]
    shapedirs = dense(model['shapedirs']).astype(np.float64)
    posedirs = dense(model['posedirs']).astype(np.float64)
    Jreg = dense(model['J_regressor']).astype(np.float64)
    kreg = dense(model['cocoplus_regressor']).astype(np.float64)
    if joint_type == 'lsp':
        kreg = kreg[:14]
    return {
        'v_template': v_template.reshape(-1),
        'dirs': np.concatenate([shapedirs.reshape(-1, 10).T, posedirs.reshape(-1, 207).T], 0),
        'J_template': (Jreg @ v_template).reshape(-1),
        'J_shapedirs': np.einsum('jv,vcb->bjc', Jreg, shapedirs).reshape(10, 72),
        'weights': dense(model['weights']).astype(np.float64),
        'regressor': kreg,
        'parents': np.asarray(model['kintree_table'])[0].astype(np.int64),
        'num_verts': V,
    }


def smpl_forward(consts, beta, theta, cam=None):
    """All stages chained: beta [N,10], theta [N,72] (cam [N,3]) -> dict(verts, joints, Rs, Jtr, A, v_posed[, kps]), float64.

    `consts` is model_constants(...) or the same keys as tensors (e.g. the float32 arrays a kernel read, so the comparison sees
    the kernel's arithmetic and not the rounding of its inputs)."""
    b = _t(beta)
    dev = b.device
    V = int(consts['num_verts'])
    Rs = rodrigues(_t(theta, dev).reshape(-1, 24, 3))
    J = rest_joints(b, consts['J_template'], consts['J_shapedirs'])
    Jtr, A = forward_kinematics(Rs, J, consts['parents'])
    v_posed = blend(b, Rs, consts['v_template'], consts['dirs']).reshape(-1, V, 3)
    verts = skin(v_posed, A, consts['weights'])
    joints = regress(verts, consts['regressor'])
    out = {'verts': verts, 'joints': joints, 'Rs': Rs, 'Jtr': Jtr, 'A': A, 'v_posed': v_posed}
    if cam is not None:
        out['kps'] = orth_proj(joints, _t(cam, dev))
    return out
