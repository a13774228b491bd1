"""CPU: the differentiable torch oracle of the SMPL path (oracle/smpl_grad_ref.py), known-answer gradients, the host packing of the
backward's extra arrays and the layout of hd_smpl_grad_consts.  No GPU needed."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64


def _inputs(n, seed, zero_pose=False, scale=0.4):
    rng = np.random.RandomState(seed)
    beta = rng.normal(0, 1.0, size=(n, 10))
    theta = np.zeros((n, 72)) if zero_pose else rng.normal(0, scale, size=(n, 72))
    return beta, theta


def test_torch_oracle_equals_numpy_oracle(smpl_model, smpl_model_dense):
    from oracle.smpl_ref import SMPLRef
    from oracle.smpl_grad_ref import SMPLGradRef
    for model, jt in ((smpl_model, 'cocoplus'), (smpl_model_dense, 'lsp')):
        beta, theta = _inputs(3, 1)
        ref = SMPLRef(model, joint_type=jt, dtype=np.float64)
        v, j, R = ref(beta, theta, get_skin=True)
        tr = SMPLGradRef(model, joint_type=jt)
        tv, tj, tR = tr(torch.from_numpy(beta), torch.from_numpy(theta), get_skin=True)
        for a, b in ((tv, v), (tj, j), (tR, R), (tr.J_transformed, ref.J_transformed)):
            assert np.abs(a.numpy() - b).max() <= 1e-12 * max(1.0, np.abs(b).max())


def test_torch_oracle_helpers_equal_numpy_oracle():
    from oracle import smpl_ref
    from oracle import smpl_grad_ref as g
    from human_dynamics_b200.synthetic import SMPL_PARENTS
    rng = np.random.RandomState(3)
    th = rng.normal(0, 0.7, size=(50, 3))
    assert np.abs(g.batch_rodrigues(torch.from_numpy(th)).numpy() - smpl_ref.batch_rodrigues(th, np.float64)).max() < 1e-14
    Rs = smpl_ref.batch_rodrigues(rng.normal(0, 0.5, size=(48, 3)), np.float64).reshape(2, 24, 3, 3)
    Js = rng.normal(0, 0.3, size=(2, 24, 3))
    par = SMPL_PARENTS.astype(np.int64)
    for rb in (False, True):
        nj, A = g.batch_global_rigid_transformation(torch.from_numpy(Rs), torch.from_numpy(Js), par, rotate_base=rb)
        nj_r, A_r = smpl_ref.batch_global_rigid_transformation(Rs, Js, par, rotate_base=rb, dtype=np.float64)
        assert np.abs(nj.numpy() - nj_r).max() < 1e-13 and np.abs(A.numpy() - A_r).max() < 1e-13
    X, cam = rng.normal(size=(2, 7, 3)), rng.uniform(0.5, 1.5, size=(2, 3))
    assert np.abs(g.batch_orth_proj_idrot(torch.from_numpy(X), torch.from_numpy(cam)).numpy() -
                  smpl_ref.batch_orth_proj_idrot(X, cam, np.float64)).max() < 1e-14


@pytest.mark.parametrize('zero_pose', [False, True])
def test_gradcheck_smpl_oracle(smpl_model, zero_pose):
    """Finite differences pin the float64 oracle's gradients (all four outputs, contracted with fixed random weights so that the
    analytic Jacobian needs one backward per contraction)."""
    from oracle.smpl_grad_ref import SMPLGradRef
    tr = SMPLGradRef(smpl_model)
    beta, theta = _inputs(2, 5, zero_pose=zero_pose)
    rng = np.random.RandomState(9)
    V, K = tr.size[0], tr.joint_regressor.shape[1]
    U = [torch.from_numpy(rng.normal(size=s)) for s in ((2, V, 3), (2, K, 3), (2, 24, 3, 3), (2, 24, 3))]

    def f(b, t):
        v, j, R = tr(b, t, get_skin=True)
        return torch.stack([(v * U[0]).sum(), (j * U[1]).sum(), (R * U[2]).sum(), (tr.J_transformed * U[3]).sum()])
    b = torch.from_numpy(beta).requires_grad_()
    t = torch.from_numpy(theta).requires_grad_()
    assert torch.autograd.gradcheck(f, (b, t), eps=1e-6, atol=1e-6, rtol=1e-5)


def test_gradcheck_helpers():
    from oracle import smpl_grad_ref as g
    from human_dynamics_b200.synthetic import SMPL_PARENTS
    rng = np.random.RandomState(4)
    th = torch.from_numpy(rng.normal(0, 0.8, size=(6, 3))).requires_grad_()
    assert torch.autograd.gradcheck(g.batch_rodrigues, (th,))
    Rs = torch.from_numpy(rng.normal(size=(2, 24, 3, 3))).requires_grad_()
    Js = torch.from_numpy(rng.normal(size=(2, 24, 3))).requires_grad_()
    par = SMPL_PARENTS.astype(np.int64)
    for rb in (False, True):
        assert torch.autograd.gradcheck(lambda r, j: g.batch_global_rigid_transformation(r, j, par, rotate_base=rb), (Rs, Js))
    X = torch.from_numpy(rng.normal(size=(2, 5, 3))).requires_grad_()
    cam = torch.from_numpy(rng.uniform(0.5, 1.5, size=(2, 3))).requires_grad_()
    assert torch.autograd.gradcheck(g.batch_orth_proj_idrot, (X, cam))


def test_known_answer_dverts_dbeta_at_zero_pose(smpl_model):
    """theta = 0 => every A_k = [I | 0] and the skinning weights are row-stochastic, so verts = v_shaped and d verts / d beta is
    exactly the shapedirs column."""
    from oracle.smpl_grad_ref import SMPLGradRef
    tr = SMPLGradRef(smpl_model)
    beta, _ = _inputs(1, 2)
    V = tr.size[0]
    Jac = torch.autograd.functional.jacobian(lambda b: tr(b, torch.zeros(1, 72, dtype=F64), get_skin=True)[0],
                                             torch.from_numpy(beta))        # [1,V,3,1,10]
    sd = np.asarray(smpl_model['shapedirs'])                                 # (V,3,10)
    assert np.abs(Jac[0, :, :, 0, :].numpy() - sd).max() < 1e-12


def test_known_answer_rodrigues_at_zero():
    """d R / d theta_i at theta = 0 is the skew generator [e_i]x (up to the O(1e-8) shift of the reference's expression)."""
    from oracle.smpl_grad_ref import batch_rodrigues, batch_skew
    Jac = torch.autograd.functional.jacobian(lambda t: batch_rodrigues(t), torch.zeros(1, 3, dtype=F64))   # [1,3,3,1,3]
    for i in range(3):
        e = torch.zeros(1, 3, dtype=F64)
        e[0, i] = 1
        assert (Jac[0, :, :, 0, i] - batch_skew(e)[0]).abs().max() < 1e-7
    assert torch.isfinite(Jac).all()


def test_known_answer_projection():
    from oracle.smpl_grad_ref import batch_orth_proj_idrot
    rng = np.random.RandomState(1)
    X = torch.from_numpy(rng.normal(size=(3, 4, 3))).requires_grad_()
    cam = torch.from_numpy(rng.uniform(0.5, 1.5, size=(3, 3))).requires_grad_()
    gk = torch.from_numpy(rng.normal(size=(3, 4, 2)))
    gX, gc = torch.autograd.grad(batch_orth_proj_idrot(X, cam), (X, cam), gk)
    s, t = cam[:, 0].detach(), cam[:, 1:].detach()
    assert torch.allclose(gX[:, :, :2], s[:, None, None] * gk, atol=1e-14) and torch.all(gX[:, :, 2] == 0)
    assert torch.allclose(gc[:, 0], ((X.detach()[:, :, :2] + t[:, None]) * gk).sum((1, 2)), atol=1e-13)
    assert torch.allclose(gc[:, 1:], s[:, None] * gk.sum(1), atol=1e-13)


def test_vertex_major_regressor_is_transpose_of_csc(smpl_model_dense):
    from human_dynamics_b200.smpl import pack_grad_arrays
    from human_dynamics_b200.synthetic import make_synthetic_smpl
    for model in (make_synthetic_smpl(seed=2), smpl_model_dense):
        W = np.asarray(model['weights'], np.float64)
        kreg = np.asarray(model['cocoplus_regressor'], np.float64)
        V, K = W.shape[0], kreg.shape[0]
        p = pack_grad_arrays(W, kreg)
        # CSC over keypoints as hd_smpl_consts holds it (smpl.py / hd_smpl_pack)
        csc = np.zeros((K, V))
        for k in range(K):
            nz = np.nonzero(kreg[k])[0]
            csc[k, nz] = kreg[k, nz].astype(np.float32)
        vm = np.zeros((V, K))
        assert p['kpv_ptr'][0] == 0 and p['kpv_ptr'][-1] == len(p['kpv_kidx']) == np.count_nonzero(kreg)
        for v in range(V):
            b, e = p['kpv_ptr'][v], p['kpv_ptr'][v + 1]
            ks = p['kpv_kidx'][b:e]
            assert np.all(np.diff(ks) > 0)
            vm[v, ks] = p['kpv_w'][b:e]
        assert np.array_equal(vm, csc.T)
        # joint-major skinning tiles reproduce the dense weights
        T = (V + 255) // 256
        dense = np.zeros((V, 24), np.float32)
        assert len(p['lbt_ptr']) == T * 24 + 1
        for t in range(T):
            for k in range(24):
                b, e = p['lbt_ptr'][t * 24 + k], p['lbt_ptr'][t * 24 + k + 1]
                vs = p['lbt_v'][b:e]
                assert np.all((vs >= t * 256) & (vs < (t + 1) * 256)) and np.all(np.diff(vs) > 0)
                dense[vs, k] = p['lbt_w'][b:e]
        assert np.array_equal(dense, W.astype(np.float32))


def test_grad_consts_layout_matches_gcc():
    from human_dynamics_b200 import _lib
    if shutil.which('gcc') is None:
        pytest.skip('gcc not available')
    fields = [f for f, _ in _lib.SmplGradConsts._fields_]
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "hd_b200.h"\nint main(){printf("%zu %d %d", sizeof(hd_smpl_grad_consts), ' \
          'HD_SMPL_GRAD_TILE, HD_SMPL_GRAD_CLD);\n'
    src += ''.join('printf(" %%zu", offsetof(hd_smpl_grad_consts, %s));\n' % f for f in fields) + 'return 0;}\n'
    with tempfile.TemporaryDirectory() as td:
        c, exe = os.path.join(td, 't.c'), os.path.join(td, 't')
        open(c, 'w').write(src)
        subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe])
        out = [int(x) for x in subprocess.check_output([exe]).split()]
    assert out[0] == ctypes.sizeof(_lib.SmplGradConsts)
    assert (out[1], out[2]) == (_lib.SMPL_GRAD_TILE, _lib.SMPL_GRAD_CLD)
    for f, off in zip(fields, out[3:]):
        assert getattr(_lib.SmplGradConsts, f).offset == off, f


def test_backward_entries_reject_bad_arguments_without_launch():
    from human_dynamics_b200 import _lib
    lib = _lib.lib
    lib.hd_launch_count_reset()
    c, g = _lib.SmplConsts(), _lib.SmplGradConsts()
    assert lib.hd_smpl_lbs_backward(ctypes.byref(c), ctypes.byref(g), None, 0, None, None, None, None, None, 4, None) == 1
    assert lib.hd_smpl_pose_backward(ctypes.byref(c), None, 10, None, 72, 4, None, None, 0, None, None, None, 10, None, 72, None) == 1
    assert lib.hd_rodrigues_backward(None, None, None, 4, None) == 1
    assert lib.hd_global_rigid_backward(None, None, None, None, None, None, None, 2, 0, None) == 1
    assert lib.hd_orth_proj_backward(None, None, None, None, None, 2, 3, None) == 1
    assert b'hd_orth_proj_backward' in lib.hd_last_error()
    assert lib.hd_launch_count() == 0
    assert lib.hd_smpl_backward_workspace_bytes(0, 6890) == 0
    assert lib.hd_smpl_backward_workspace_bytes(3, 6890) >= 3 * (2 * 6892 * 4 + (288 * 2 + 224 + 216) * 4 + 512 * 2)
    assert lib.hd_version() >= 102
