"""GPU: the SMPL backward (csrc/smpl_grad.cu through the C-ABI and torch autograd) against the float64 torch oracle
(oracle/smpl_grad_ref.py, itself pinned to finite differences in test_smpl_grad_cpu.py)."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

REL = 1e-4
GUARD = 2.5e-5      # the float32 oracle must agree with the float64 one this well, else the case is too ill-conditioned to judge
HERE = os.path.dirname(os.path.abspath(__file__))
_SMPL = {}


def rel_err(a, b):
    a = a.detach().cpu().double().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, np.float64)
    b = b.detach().cpu().double().numpy() if isinstance(b, torch.Tensor) else np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _smpl(model, jt='cocoplus'):
    from src.tf_smpl.batch_smpl import SMPL
    key = (id(model), jt)
    if key not in _SMPL:
        _SMPL[key] = SMPL(model, joint_type=jt)
    return _SMPL[key]


def _upstream(n, V, K, seed, scale=1.0):
    rng = np.random.RandomState(seed)
    return [torch.from_numpy(rng.normal(0, 1, size=s) * scale) for s in ((n, V, 3), (n, K, 3), (n, 24, 3, 3), (n, 24, 3))]


def _gpu_grads(smpl, beta, theta, ups):
    b = torch.from_numpy(beta).cuda().requires_grad_()
    t = torch.from_numpy(theta).cuda().requires_grad_()
    v, j, R = smpl(b, t, get_skin=True)
    torch.autograd.backward([v, j, R, smpl.J_transformed], [u.float().cuda() for u in ups])
    return b.grad, t.grad


def _oracle_grads(model, jt, beta, theta, ups, dtype=torch.float64):
    from oracle.smpl_grad_ref import SMPLGradRef
    tr = SMPLGradRef(model, joint_type=jt, dtype=dtype)
    b = torch.tensor(np.asarray(beta, np.float64), dtype=dtype, requires_grad=True)
    t = torch.tensor(np.asarray(theta, np.float64), dtype=dtype, requires_grad=True)
    v, j, R = tr(b, t, get_skin=True)
    return torch.autograd.grad([v, j, R, tr.J_transformed], [b, t], [u.to(dtype) for u in ups])


def _check(model, jt, beta, theta, seed, rows=None, scale=1.0):
    smpl = _smpl(model, jt)
    n = beta.shape[0]
    V, K = smpl.consts.num_verts, smpl.consts.num_kps
    ups = _upstream(n, V, K, seed, scale)
    gb, gt = _gpu_grads(smpl, beta, theta, ups)
    idx = np.arange(n) if rows is None else rows       # pose n's gradient depends on pose n only: the oracle checks a sample
    sub = [u[idx] for u in ups]
    r64 = _oracle_grads(model, jt, beta[idx], theta[idx], sub)
    r32 = _oracle_grads(model, jt, beta[idx], theta[idx], sub, torch.float32)
    for got, ref, ref32, name in ((gb, r64[0], r32[0], 'beta'), (gt, r64[1], r32[1], 'theta')):
        assert rel_err(ref32, ref) < GUARD, 'oracle f32 vs f64 ill-conditioned on d' + name
        err = rel_err(got[idx], ref)
        assert np.isfinite(got.detach().cpu().numpy()).all()
        assert err < REL, (name, err)
    return gb, gt


@pytest.mark.parametrize('n', [1, 37, 255, 256, 777, 2112])
def test_smpl_grad_matches_oracle(smpl_model, n):
    from human_dynamics_b200 import synthetic
    beta, theta = synthetic.make_smpl_inputs(n, seed=n)
    rows = None if n <= 37 else np.unique(np.r_[0, n - 1, np.random.RandomState(n).choice(n, 6, replace=False)])
    _check(smpl_model, 'cocoplus', beta, theta, seed=n, rows=rows)


def test_smpl_grad_zero_pose_and_large_rotations(smpl_model, smpl_model_dense):
    from human_dynamics_b200 import synthetic
    beta, theta = synthetic.make_smpl_inputs(5, seed=1, zero_pose=True)
    _check(smpl_model, 'cocoplus', beta, theta, seed=2)
    spec = importlib.util.spec_from_file_location('_ref_sweeps', os.path.join(HERE, 'golden', 'make_ref_sweeps_golden.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    beta, theta, _ = mod.smpl_inputs()                 # beta ~ N(0, 2), theta ~ N(0, 1), one root rotation of pi
    _check(smpl_model, 'cocoplus', beta[:12], theta[:12], seed=3)
    _check(smpl_model_dense, 'lsp', beta[:12], theta[:12], seed=4)


def test_smpl_grad_dense_weights_lsp(smpl_model_dense):
    from human_dynamics_b200 import synthetic
    beta, theta = synthetic.make_smpl_inputs(300, seed=6)
    _check(smpl_model_dense, 'lsp', beta, theta, seed=6, rows=np.array([0, 150, 299]))


@pytest.mark.parametrize('scale', [1e8, 1e-8])
def test_smpl_grad_upstream_scale(smpl_model, scale):
    """Gradients carry the loss's arbitrary scale: the relative error must not depend on it (no fp16 range anywhere)."""
    from human_dynamics_b200 import synthetic
    beta, theta = synthetic.make_smpl_inputs(300, seed=8)
    rows = np.array([0, 7, 299])
    gb1, gt1 = _check(smpl_model, 'cocoplus', beta, theta, seed=8, rows=rows)
    gb, gt = _check(smpl_model, 'cocoplus', beta, theta, seed=8, rows=rows, scale=scale)
    assert rel_err(gb / scale, gb1) < 1e-6 and rel_err(gt / scale, gt1) < 1e-6


def test_helper_grads_match_oracle():
    from src.tf_smpl.batch_lbs import batch_rodrigues, batch_global_rigid_transformation
    from src.tf_smpl.projection import batch_orth_proj_idrot
    from oracle import smpl_grad_ref as g
    from human_dynamics_b200.synthetic import SMPL_PARENTS
    rng = np.random.RandomState(0)
    th = rng.normal(0, 1.0, size=(600, 3))
    th[::7] = 0.0
    gR = rng.normal(size=(600, 3, 3))
    t = torch.from_numpy(th).float().cuda().requires_grad_()
    batch_rodrigues(t).backward(torch.from_numpy(gR).float().cuda())
    t64 = torch.from_numpy(th).requires_grad_()
    ref, = torch.autograd.grad(g.batch_rodrigues(t64), t64, torch.from_numpy(gR))
    assert rel_err(t.grad, ref) < REL
    # zero rotation: dR/dtheta = skew generators, so dtheta = (G21 - G12, G02 - G20, G10 - G01)
    G = gR[::7]
    skew = np.stack([G[:, 2, 1] - G[:, 1, 2], G[:, 0, 2] - G[:, 2, 0], G[:, 1, 0] - G[:, 0, 1]], 1)
    assert np.abs(t.grad[::7].cpu().numpy() - skew).max() < 1e-5 * np.abs(skew).max()

    par = SMPL_PARENTS.astype(np.int64)
    Rs = g.batch_rodrigues(torch.from_numpy(rng.normal(0, 0.6, size=(40 * 24, 3)))).reshape(40, 24, 3, 3).numpy()
    Js = rng.normal(0, 0.3, size=(40, 24, 3))
    gJ, gA = rng.normal(size=(40, 24, 3)), rng.normal(size=(40, 24, 4, 4))
    for rb in (False, True):
        R = torch.from_numpy(Rs).float().cuda().requires_grad_()
        J = torch.from_numpy(Js).float().cuda().requires_grad_()
        nj, A = batch_global_rigid_transformation(R, J, par, rotate_base=rb)
        torch.autograd.backward([nj, A], [torch.from_numpy(gJ).float().cuda(), torch.from_numpy(gA).float().cuda()])
        R64, J64 = torch.from_numpy(Rs).requires_grad_(), torch.from_numpy(Js).requires_grad_()
        rr = torch.autograd.grad(g.batch_global_rigid_transformation(R64, J64, par, rotate_base=rb), (R64, J64),
                                 (torch.from_numpy(gJ), torch.from_numpy(gA)))
        assert rel_err(R.grad, rr[0]) < REL and rel_err(J.grad, rr[1]) < REL, rb

    X, cam, gk = rng.normal(size=(50, 19, 3)), rng.uniform(0.5, 1.5, size=(50, 3)), rng.normal(size=(50, 19, 2))
    Xg = torch.from_numpy(X).float().cuda().requires_grad_()
    cg = torch.from_numpy(cam).float().cuda().requires_grad_()
    batch_orth_proj_idrot(Xg, cg).backward(torch.from_numpy(gk).float().cuda())
    X64, c64 = torch.from_numpy(X).requires_grad_(), torch.from_numpy(cam).requires_grad_()
    rX, rc = torch.autograd.grad(g.batch_orth_proj_idrot(X64, c64), (X64, c64), torch.from_numpy(gk))
    assert rel_err(Xg.grad, rX) < REL and rel_err(cg.grad, rc) < REL


def test_bit_identity_split_permute_repeat(smpl_model):
    from human_dynamics_b200 import synthetic
    smpl = _smpl(smpl_model)
    n = 300
    beta, theta = synthetic.make_smpl_inputs(n, seed=21)
    ups = _upstream(n, smpl.consts.num_verts, smpl.consts.num_kps, 21)
    gb, gt = _gpu_grads(smpl, beta, theta, ups)
    gb2, gt2 = _gpu_grads(smpl, beta, theta, ups)
    assert torch.equal(gb, gb2) and torch.equal(gt, gt2)
    for part in (slice(0, 100), slice(100, n)):         # both halves stay on the tensor-core blend path like the full batch
        pb, pt = _gpu_grads(smpl, beta[part], theta[part], [u[part] for u in ups])
        assert torch.equal(pb, gb[part]) and torch.equal(pt, gt[part])
    perm = np.random.RandomState(0).permutation(n)
    pb, pt = _gpu_grads(smpl, beta[perm], theta[perm], [u[perm] for u in ups])
    assert torch.equal(pb, gb[perm]) and torch.equal(pt, gt[perm])


def test_forward_unchanged_and_no_grad_launches(smpl_model):
    from human_dynamics_b200 import synthetic, _lib
    smpl = _smpl(smpl_model)
    for n in (7, 300):
        beta, theta = synthetic.make_smpl_inputs(n, seed=n)
        b, t = torch.from_numpy(beta).cuda(), torch.from_numpy(theta).cuda()
        _lib.lib.hd_launch_count_reset()
        plain = [x.clone() for x in smpl(b, t, get_skin=True)] + [smpl.J_transformed.clone()]
        torch.cuda.synchronize()
        n_plain = _lib.lib.hd_launch_count()
        _lib.lib.hd_launch_count_reset()
        smpl.consts.forward(b, t)
        torch.cuda.synchronize()
        assert _lib.lib.hd_launch_count() == n_plain
        with torch.no_grad():
            _lib.lib.hd_launch_count_reset()
            out = smpl(b.clone().requires_grad_(), t.clone().requires_grad_(), get_skin=True)
            torch.cuda.synchronize()
            assert _lib.lib.hd_launch_count() == n_plain and all(x.grad_fn is None for x in out)
        bg, tg = b.clone().requires_grad_(), t.clone().requires_grad_()
        graded = list(smpl(bg, tg, get_skin=True)) + [smpl.J_transformed]
        for x, y in zip(graded, plain):
            assert x.grad_fn is not None and torch.equal(x.detach(), y)


def test_strided_omega_views_get_their_columns(smpl_model):
    smpl = _smpl(smpl_model)
    n = 21
    omega_np = np.random.RandomState(3).normal(0, 0.3, size=(n, 85)).astype(np.float32)
    omega = torch.from_numpy(omega_np).cuda().requires_grad_()
    ups = _upstream(n, smpl.consts.num_verts, smpl.consts.num_kps, 5)
    v, j, R = smpl(omega[:, 75:85], omega[:, 3:75].reshape(n, 24, 3), get_skin=True)
    torch.autograd.backward([v, j, R, smpl.J_transformed], [u.float().cuda() for u in ups])
    gb, gt = _gpu_grads(smpl, omega_np[:, 75:85].copy(), omega_np[:, 3:75].copy(), ups)
    assert torch.all(omega.grad[:, :3] == 0)
    assert torch.equal(omega.grad[:, 3:75], gt) and torch.equal(omega.grad[:, 75:85], gb)


def test_errors(smpl_model):
    from human_dynamics_b200 import _lib
    from src.tf_smpl.batch_lbs import batch_rodrigues
    smpl = _smpl(smpl_model)
    with pytest.raises(RuntimeError):
        smpl(torch.zeros(2, 10, requires_grad=True), torch.zeros(2, 72, requires_grad=True))
    with pytest.raises(RuntimeError):
        batch_rodrigues(torch.zeros(4, 3, requires_grad=True))
    b = torch.zeros(2, 10, device='cuda', requires_grad=True)
    t = torch.full((2, 72), 0.1, device='cuda', requires_grad=True)
    j = smpl(b, t)
    gb, = torch.autograd.grad((j ** 2).sum(), b, create_graph=True)     # upstream 2j is on the graph
    with pytest.raises(RuntimeError, match='twice'):
        gb.sum().backward()
    # a grad-consts block that does not match the model: HD_ERR_INVALID, nothing launched
    g, keep, _ = smpl.consts.grad_state()
    bad = _lib.SmplGradConsts.from_buffer_copy(g)
    bad.num_tiles += 1
    ws, views, _, _ = smpl.consts.backward_workspace(2)
    x = views['vpos']
    _lib.lib.hd_launch_count_reset()
    rc = _lib.lib.hd_smpl_lbs_backward(ctypes.byref(smpl.consts.c), ctypes.byref(bad), x.data_ptr(), smpl.consts.vp_ld,
                                       views['A12'].data_ptr(), x.data_ptr(), None, views['dvpos'].data_ptr(), views['dA12'].data_ptr(),
                                       2, None)
    assert rc == 1 and _lib.lib.hd_launch_count() == 0
    rc = _lib.lib.hd_smpl_pose_backward(ctypes.byref(smpl.consts.c), b.data_ptr(), 10, t.data_ptr(), 72, 2, None, views['dc'].data_ptr(), 100,
                                        None, None,
                                        b.data_ptr(), 10, t.data_ptr(), 72, None)
    assert rc == 1 and _lib.lib.hd_launch_count() == 0      # dc_ld < 217


def test_neutral_shape_fit_tracks_oracle(smpl_model):
    """The loop of compute_neutral_shape.py:100-135: theta = 0, plain gradient descent with lr = 1 on the mean vertex distance,
    fitting beta to the vertices of a synthetic target shape; GPU and float64 oracle step for step."""
    from oracle.smpl_grad_ref import SMPLGradRef
    smpl = _smpl(smpl_model)
    tr = SMPLGradRef(smpl_model)
    n = 4
    beta_star = np.random.RandomState(11).normal(0, 1.5, size=(n, 10))
    theta0 = np.zeros((n, 72))
    target64 = tr(torch.from_numpy(beta_star), torch.from_numpy(theta0), get_skin=True)[0].detach()
    target = target64.float().cuda()
    b_gpu = torch.zeros(n, 10, device='cuda', requires_grad=True)
    t_gpu = torch.zeros(n, 72, device='cuda')
    b_ref = torch.zeros(n, 10, dtype=torch.float64, requires_grad=True)
    losses = []
    for step in range(20):
        v = smpl(b_gpu, t_gpu, get_skin=True)[0]
        loss = torch.sqrt(((target - v) ** 2).sum(2)).mean()
        g, = torch.autograd.grad(loss, b_gpu)
        vr = tr(b_ref, torch.from_numpy(theta0), get_skin=True)[0]
        gr, = torch.autograd.grad(torch.sqrt(((target64 - vr) ** 2).sum(2)).mean(), b_ref)
        with torch.no_grad():
            b_gpu -= 1.0 * g
            b_ref -= 1.0 * gr
        losses.append(float(loss.detach()))
        assert rel_err(b_gpu, b_ref) < REL, step
    assert losses[-1] < losses[0]


def test_keypoint_fit_tracks_oracle(smpl_model):
    """theta / beta / cam fitted to the 2D keypoints of a known pose through batch_orth_proj_idrot, 20 SGD steps, GPU vs oracle."""
    from oracle.smpl_grad_ref import SMPLGradRef, batch_orth_proj_idrot as proj_ref
    from src.tf_smpl.projection import batch_orth_proj_idrot
    smpl = _smpl(smpl_model)
    tr = SMPLGradRef(smpl_model)
    n = 3
    rng = np.random.RandomState(12)
    beta_star, theta_star = rng.normal(0, 1, size=(n, 10)), rng.normal(0, 0.3, size=(n, 72))
    cam_star = np.c_[rng.uniform(0.8, 1.2, size=(n, 1)), rng.normal(0, 0.1, size=(n, 2))]
    kp64 = proj_ref(tr(torch.from_numpy(beta_star), torch.from_numpy(theta_star)), torch.from_numpy(cam_star)).detach()
    kp = kp64.float().cuda()
    x0 = [np.zeros((n, 10)), theta_star * 0.5, np.c_[np.ones((n, 1)), np.zeros((n, 2))]]
    gpu = [torch.tensor(a, dtype=torch.float32, device='cuda', requires_grad=True) for a in x0]
    ref = [torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in x0]
    lr = 0.5
    losses = []
    for step in range(20):
        loss = ((batch_orth_proj_idrot(smpl(gpu[0], gpu[1]), gpu[2]) - kp) ** 2).sum(2).mean()
        gg = torch.autograd.grad(loss, gpu)
        lr_ = ((proj_ref(tr(ref[0], ref[1]), ref[2]) - kp64) ** 2).sum(2).mean()
        gr = torch.autograd.grad(lr_, ref)
        with torch.no_grad():
            for a, b, ga, gb in zip(gpu, ref, gg, gr):
                a -= lr * ga
                b -= lr * gb
        losses.append(float(loss.detach()))
        for a, b in zip(gpu, ref):
            assert rel_err(a, b) < REL, step
    assert losses[-1] < losses[0]
