"""GPU: the trainer's objective (csrc/losses.cu through objective.LossFunction) against the float64 oracle (oracle/losses_ref.py):
values, input gradients, the edge cases, determinism and the launch count; HMMRTrainer against the float64 oracle chain, its
convergence and its checkpoint; the src/ shims."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F64 = torch.float64
DIFF = ('omega', 'joints', 'rots', 'strips', 'pred_strips')


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def cfg(**kw):
    from human_dynamics_b200.objective import TrainConfig
    return TrainConfig(**kw)


ALL = dict(do_hallucinate=True, do_hallucinate_preds=True)


def gpu_inputs(x, grad=True):
    return {k: torch.from_numpy(v).cuda().requires_grad_(grad and k in DIFF) for k, v in x.items()}


def ref_inputs(x):
    return {k: torch.from_numpy(v).to(F64).requires_grad_(k in DIFF) for k, v in x.items()}


def kp_ties(obj, x, tol=1e-6):
    """Boolean masks of the joints / omega elements an L1 residual within tol of 0 feeds (their gradient is excluded)."""
    from oracle import losses_ref as R
    S, B, T, K = len(obj.sets), obj.B, obj.T, obj.K
    tj = np.zeros((S, B, T, K, 3), bool)
    tc = np.zeros((S, B, T, 85), bool)
    lab = torch.from_numpy(x['labels']).to(F64)
    for s, (g, dt) in enumerate(obj.sets):
        if abs(dt) >= T:
            continue
        Tw = T - abs(dt)
        p0, q0 = (abs(dt), 0) if dt < 0 else (0, dt)
        j = torch.from_numpy(x['joints'][s, :, p0:p0 + Tw]).to(F64)
        lb = lab[:, q0:q0 + Tw]
        if dt == 0:
            cam = torch.from_numpy(x['omega'][s, :, :, :3]).to(F64)
            xh = cam[..., None, 0:1] * (j[..., :2] + cam[..., None, 1:])
        else:
            cam, _ = R.procrustes2d_vis(j.reshape(-1, K, 3), lb.reshape(-1, K, 3))
            cam = cam.reshape(B, Tw, 1, 3)
            xh = cam[..., 0:1] * (j[..., :2] + cam[..., 1:])
        tie = ((xh - lb[..., :2]).abs() < tol) & (lb[..., 2:3] != 0)
        tj[s, :, p0:p0 + Tw, :, :2] |= tie.numpy()
        if dt == 0:
            tc[s, :, :, :3] |= tie.reshape(B, Tw, -1).any(-1).numpy()[..., None]
    return {'joints': tj, 'omega': tc}


def run_gpu(obj, x, coef):
    from human_dynamics_b200.objective import evaluate
    t = gpu_inputs(x)
    named, cams = evaluate(obj, t)
    L = sum(named[k] * c for k, c in zip(obj.names, coef))
    L.backward()
    return named, cams, {k: t[k].grad for k in DIFF if k in t}


def run_ref(config, obj, x, coef, nan_frames=False):
    from oracle import losses_ref as R
    t = ref_inputs(x)
    named, cams = R.objective(config, t, nan_frames=nan_frames)
    L = sum(named[k] * c for k, c in zip(obj.names, coef))
    L.backward()
    return named, cams, {k: t[k].grad for k in DIFF if k in t}


SHAPES = [(1, 1, dict(predict_delta=False)), (3, 10, ALL), (8, 20, ALL), (32, 20, ALL)]


@pytest.mark.parametrize('B,T,flags', SHAPES)
@pytest.mark.parametrize('scale', [1.0, 1e8, 1e-8])
def test_values_and_grads_match_oracle(B, T, flags, scale):
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import build_objective
    c = cfg(**flags)
    obj = build_objective(c, B, T, 25)
    x = synthetic.make_loss_inputs(obj, seed=B * 100 + T)
    coef = list(np.random.RandomState(B).uniform(0.5, 2.0, size=len(obj.names)) * scale)
    named, cams, grads = run_gpu(obj, x, coef)
    rn, rc, rg = run_ref(c, obj, x, coef)
    for k in obj.names:
        a, b = named[k].item(), rn[k].item()
        assert abs(a - b) <= 1e-5 * abs(b) + 1e-12, (k, a, b)
    for key, cam in cams.items():
        assert rel_err(cam.cpu().numpy(), rc[key].numpy()) < 1e-5, key
    ties = kp_ties(obj, x)
    excluded = 0
    for k, g in grads.items():
        a, b = g.cpu().numpy(), rg[k].numpy()
        keep = ~ties[k] if k in ties else np.ones(a.shape, bool)
        excluded += int((~keep).sum())
        assert np.abs(a - b)[keep].max() <= 1e-5 * np.abs(b).max(), (k, rel_err(a[keep], b[keep]))
    print('B=%d T=%d scale=%g: %d gradient elements excluded as L1 ties (%.2e of the joints)'
          % (B, T, scale, excluded, excluded / x['joints'].size))


def test_golden_sized_case_against_oracle_and_terms():
    """The 3 x 10 case: the scale clip is engaged on the flipped frame, and each named loss is the sum of its terms."""
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import build_objective, LossFunction
    c = cfg(**ALL)
    obj = build_objective(c, 3, 10, 25)
    x = synthetic.make_loss_inputs(obj, seed=1)
    t = gpu_inputs(x, grad=False)
    values, cams = LossFunction.apply(obj, *[t[n] for n in obj.inputs])
    first = obj.cameras(cams)[obj.cam_terms[0][1]]
    assert first[0, 0, 0].item() == pytest.approx(0.7)
    named = obj.named(values)
    v = values.cpu().numpy()
    for i, n in enumerate(obj.names):
        assert named[i].item() == pytest.approx(sum(v[j] for j, m in enumerate(obj.term_names) if m == n), rel=1e-6)


def test_no_3d_labels_gives_zero_terms():
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import build_objective
    c = cfg(**ALL)
    obj = build_objective(c, 3, 10, 25)
    x = synthetic.make_loss_inputs(obj, seed=2)
    x['w_joints'][:] = 0
    x['w_smpl'][:] = 0
    named, _, grads = run_gpu(obj, x, [1.0] * len(obj.names))
    for k in obj.names:
        assert np.isfinite(named[k].item())
        if k.startswith('e_joints') or k.startswith('e_smpl'):
            assert named[k].item() == 0.0, k
    assert float(grads['rots'].abs().max()) == 0.0
    for g in grads.values():
        assert torch.isfinite(g).all()


def test_all_invisible_frame_contributes_zero():
    """The deliberate deviation: an optimal-camera frame without a visible keypoint (the reference's value is NaN) contributes 0 and gets
    the camera (0.7, 0, 0)."""
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import build_objective
    c = cfg(**ALL)
    obj = build_objective(c, 3, 10, 25)
    x = synthetic.make_loss_inputs(obj, seed=3, flip_frame=False)
    i, key = obj.cam_terms[-1]
    q0 = obj.terms[i]['q'][4]
    x['labels'][1, q0 + 2, :, 2] = 0.
    coef = [1.0] * len(obj.names)
    named, cams, grads = run_gpu(obj, x, coef)
    rn, rc, rg = run_ref(c, obj, x, coef)
    nn_, _, _ = run_ref(c, obj, x, coef, nan_frames=True)
    name = obj.term_names[i]
    assert np.isnan(nn_[name].item())
    assert np.isfinite(named[name].item()) and named[name].item() == pytest.approx(rn[name].item(), rel=1e-5)
    assert cams[key][1, 2].tolist() == pytest.approx([0.7, 0.0, 0.0])
    s = obj.sets.index(key)
    p0 = obj.terms[i]['p'][4]
    assert float(grads['joints'][s, 1, p0 + 2].abs().max()) == 0.0


def test_determinism_and_clip_permutation():
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import build_objective
    c = cfg(**ALL)
    obj = build_objective(c, 8, 20, 25)
    x = synthetic.make_loss_inputs(obj, seed=4, flip_frame=False)
    coef = [1.0] * len(obj.names)
    n1, c1, g1 = run_gpu(obj, x, coef)
    n2, c2, g2 = run_gpu(obj, x, coef)
    for k in obj.names:
        assert n1[k].item() == n2[k].item()
    for k in g1:
        assert torch.equal(g1[k], g2[k])
    perm = np.random.RandomState(0).permutation(8)
    xp = {}
    for k, v in x.items():
        xp[k] = np.ascontiguousarray(v[:, perm] if k in ('omega', 'joints', 'rots') else v[perm])
    _, _, gp = run_gpu(obj, xp, coef)
    for k in g1:
        a = g1[k][:, perm] if k in ('omega', 'joints', 'rots') else g1[k][perm]
        assert torch.equal(a, gp[k]), k


@pytest.mark.parametrize('B,T,flags', SHAPES)
def test_launch_count(B, T, flags):
    from human_dynamics_b200 import synthetic, _lib
    from human_dynamics_b200.objective import build_objective, LossFunction
    obj = build_objective(cfg(**flags), B, T, 25)
    t = gpu_inputs(synthetic.make_loss_inputs(obj, seed=5))
    dv = torch.ones(len(obj.terms), device='cuda')
    _lib.lib.hd_launch_count_reset()
    values, _ = LossFunction.apply(obj, *[t[n] for n in obj.inputs])
    values.backward(dv)
    assert _lib.lib.hd_launch_count() == 3


def _target_batch(smpl, B, T, K, seed):
    """A batch whose labels are SMPL of one fixed target omega per clip (vis 1, all 3-D labels)."""
    from human_dynamics_b200.smpl import batch_orth_proj_idrot
    rng = np.random.RandomState(seed)
    om = np.zeros((B, T, 85), np.float32)
    om[..., 0] = 0.9
    om[..., 3:75] = rng.normal(0, 0.2, size=(B, 1, 72)) + rng.normal(0, 0.02, size=(B, T, 72))
    om[..., 75:] = rng.normal(0, 0.5, size=(B, 1, 10))
    o = torch.from_numpy(om).cuda().reshape(-1, 85)
    with torch.no_grad():
        _, joints, _ = smpl(o[:, 75:], o[:, 3:75], get_skin=True)
        kp = batch_orth_proj_idrot(joints, o[:, :3])
    labels = torch.cat([kp, torch.ones_like(kp[..., :1])], -1).reshape(B, T, K, 3)
    return {'phis': torch.from_numpy(rng.normal(0, 1, size=(B, T, 2048)).astype(np.float32)).cuda(), 'labels': labels.contiguous(),
            'poses': o[:, 3:75].reshape(B, T, 72).contiguous(), 'shape': o.reshape(B, T, 85)[:, 0, 75:].contiguous(),
            'gt3ds': joints[:, :14].reshape(B, T, 14, 3).contiguous(), 'has_3d': torch.ones((B, 2), device='cuda')}


def _mocap(n, seed):
    from human_dynamics_b200.smpl import batch_rodrigues
    aa = torch.from_numpy(np.random.RandomState(seed).normal(0, 0.3, size=(n * 24, 3)).astype(np.float32)).cuda()
    return batch_rodrigues(aa).reshape(n, 216)


def test_training_converges(weights, smpl_model):
    from human_dynamics_b200.objective import HMMRTrainer
    from src.tf_smpl.batch_smpl import SMPL
    c = cfg(**ALL)
    smpl = SMPL(smpl_model)
    tr = HMMRTrainer(c, weights, smpl)
    B, T = 2, 10
    batch = _target_batch(smpl, B, T, smpl.consts.num_kps, 11)
    mocap = _mocap(tr.n_fake(B, T), 12)
    hist = []
    for _ in range(20):
        out = tr.step(batch, mocap)
        hist.append(out['e_loss'])
    h = torch.stack(hist).cpu().numpy()
    print('e_loss over 20 Adam steps:', h[0], '->', h[-1])
    assert np.isfinite(h).all() and h[-1] < h[0]
    with pytest.raises(Exception):
        tr.step(batch, mocap[:-1])


def test_d_frozen_when_weight_is_zero(weights, smpl_model):
    from human_dynamics_b200.objective import HMMRTrainer
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    tr = HMMRTrainer(cfg(d_lw_pose=0.0), weights, smpl)
    before = [p.detach().clone() for p in tr.disc.parameters()]
    e0 = [p.detach().clone() for p in tr.model.parameters()]
    batch = _target_batch(smpl, 2, 10, smpl.consts.num_kps, 5)
    tr.step(batch, _mocap(tr.n_fake(2, 10), 6))
    assert all(torch.equal(a, b) for a, b in zip(before, tr.disc.parameters()))
    assert any(not torch.equal(a, b) for a, b in zip(e0, tr.model.parameters()))


def test_trainer_tracks_oracle(weights, smpl_model):
    """Five SGD steps at B = 2, T = 10 with every flag on, against the float64 oracle chain (nets_grad_ref -> smpl_grad_ref ->
    losses_ref + dpose_ref).  Asserted: every named loss, e_loss and d_loss to 1e-3 and the D parameters to 1e-4 at every step.  The E
    parameters are reported, not asserted: they inherit the open finding of test_gpu_temporal_grad.py::test_finetune_tracks_oracle."""
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.adversarial import PARAM_NAMES
    from human_dynamics_b200.objective import HMMRTrainer, loss_keys
    from human_dynamics_b200.trainable import trainable_names
    from oracle import dpose_ref as R, losses_ref as LR, nets_grad_ref as G
    from oracle.smpl_grad_ref import SMPLGradRef, batch_rodrigues as rod_ref
    from src import ops
    from src.tf_smpl.batch_smpl import SMPL
    c = cfg(**ALL)
    smpl = SMPL(smpl_model)
    sgd = (lambda params, lr: torch.optim.SGD(params, lr))
    # D starts from the weights test_gpu_dpose.py uses (non-zero biases): with slim's zero biases, a bias's error relative to its own
    # magnitude is the relative error of five small updates, which no D test bounds
    tr = HMMRTrainer(c, weights, smpl, disc_weights=synthetic.make_dpose_weights(3, bias_scale=0.1), optimizer=sgd)
    B, T, K = 2, 10, smpl.consts.num_kps
    N = B * T
    batch = _target_batch(smpl, B, T, K, 21)
    mocap = _mocap(tr.n_fake(B, T), 22)
    names = trainable_names(weights)
    L = G.leaves(weights, names)
    P = {k: torch.tensor(v, requires_grad=True) for k, v in R.params_from_tf(tr.disc.tf_variables()).items()}
    opt_e = torch.optim.SGD([L[n] for n in names], c.e_lr)
    opt_d = torch.optim.SGD(list(P.values()), c.d_lr)
    ref_smpl = SMPLGradRef(smpl_model)
    obj = tr.objective(B, T, K)
    b64 = {k: v.detach().cpu().to(F64) for k, v in batch.items()}
    keys = tuple(sorted(int(d) for d in c.delta_t_values))

    def oracle_forward():
        phi = b64['phis']
        strips = G.fmovie(phi, G.fmovie_blocks(L))
        heads = {dt: G.ief_params(L, dt) for dt in (0,) + keys}
        mean = L['mean_param'].reshape(1, 85).expand(N, 85)
        th, dl = G.call_hmr_ief(strips.reshape(N, 2048), mean, heads, keys)
        om = {('pred', 0): th}
        om.update({('dt', k): v for k, v in dl.items()})
        ps = G.fc2_res(phi.reshape(N, 2048), tuple(L['fc2_res/fc%d/%s' % (i, k)] for i in (1, 2, 3) for k in ('weights', 'biases')))
        th, dl = G.call_hmr_ief(ps, mean, heads, keys)
        om[('hal', 0)] = th
        om.update({('hal', k): v for k, v in dl.items()})
        omega = torch.cat([om[s] for s in obj.sets], 0)
        _, joints, Rs = ref_smpl(omega[:, 75:], omega[:, 3:75], get_skin=True)
        S = len(obj.sets)
        inp = {'omega': omega.reshape(S, B, T, 85), 'joints': joints.reshape(S, B, T, K, 3), 'rots': Rs.reshape(S, B, T, 216),
               'labels': b64['labels'], 'gt_rots': rod_ref(b64['poses'].reshape(-1, 3)).reshape(B, T, 216), 'gt_shape': b64['shape'],
               'gt3ds': b64['gt3ds'], 'w_joints': b64['has_3d'][:, 0], 'w_smpl': b64['has_3d'][:, 1],
               'strips': strips.reshape(B, T, 2048), 'pred_strips': ps.reshape(B, T, 2048)}
        named, _ = LR.objective(c, inp)
        fakes = Rs.reshape(S * N, 24, 9)[:, 1:]
        reals = mocap.detach().cpu().to(F64).reshape(-1, 24, 9)[:, 1:]
        logits = R.torch_apply(torch.cat([reals, fakes], 0), P)
        named['e_pose'] = ops.compute_loss_e_fake(logits[S * N:])
        named['d_pose'] = ops.compute_loss_d_fake(logits[S * N:]) + ops.compute_loss_d_real(logits[:S * N])
        w = obj.weights
        e_loss = sum(named[k] * w[k] for k in obj.names) + named['e_pose'] * w['e_pose']
        return named, e_loss, named['d_pose'] * w['d_pose']

    worst = {}
    for step in range(5):
        out = tr.step(batch, mocap)
        named, e_loss, d_loss = oracle_forward()
        ge = torch.autograd.grad(e_loss, [L[n] for n in names], retain_graph=True, allow_unused=True)
        gd = torch.autograd.grad(d_loss, list(P.values()), allow_unused=True)
        for p, g in zip([L[n] for n in names], ge):
            p.grad = g
        for p, g in zip(P.values(), gd):
            p.grad = g
        opt_e.step()
        opt_d.step()
        errs = {}
        for k in loss_keys(c) + ['e_loss', 'd_loss']:
            ref = {'e_loss': e_loss, 'd_loss': d_loss}.get(k, named.get(k))
            a, b = out[k].item(), float(ref)
            errs[k] = abs(a - b) / max(abs(b), 1e-12) if b != 0 else abs(a)
            assert errs[k] < 1e-3, (step, k, a, b)
        ref_d = {n: P[k].detach().numpy() for n, k in zip(PARAM_NAMES, R.KEYS)}
        for n in PARAM_NAMES:
            errs[n] = rel_err(tr.disc.param(n).detach().cpu().numpy().reshape(ref_d[n].shape), ref_d[n])
            assert errs[n] < 1e-4, (step, n, errs[n])
        for n in names:      # reported only (open finding)
            errs['E:' + n] = rel_err(tr.model.param(n).detach().cpu().numpy(), L[n].detach().numpy().reshape(tr.model.param(n).shape))
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
    print('worst relative error over 5 steps:', sorted(((v, k) for k, v in worst.items()), reverse=True)[:12])


def test_checkpoint_loads_in_tester_and_discriminator(weights, smpl_model, tmp_path):
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.adversarial import PoseDiscriminator
    from human_dynamics_b200.config import HMMRConfig
    from human_dynamics_b200.objective import HMMRTrainer
    from src.evaluation.tester import Tester
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    tr = HMMRTrainer(cfg(), weights, smpl)
    tr.step(_target_batch(smpl, 1, 20, smpl.consts.num_kps, 9), _mocap(tr.n_fake(1, 20), 8))
    prefix = tr.save_checkpoint(str(tmp_path / 'model.ckpt-1'))
    d = PoseDiscriminator(prefix)
    x = _mocap(7, 1).reshape(7, 24, 9)[:, 1:].contiguous()
    with torch.no_grad():
        assert torch.equal(d(x), tr.disc(x))
    hc = HMMRConfig(load_path=prefix, batch_size=1, sequence_length=20)
    hc.smpl_model = smpl_model
    res = Tester(hc).predict(synthetic.make_images(20, seed=4).reshape(1, 20, 224, 224, 3), copy=True)
    assert np.isfinite(np.asarray(res['omegas'])).all()


def test_src_shims_equal_library_path():
    from human_dynamics_b200.objective import kp_loss, mse_loss
    from src import ops
    from src.tf_smpl import projection
    rng = np.random.RandomState(9)
    B, T, K = 3, 10, 25
    gt = torch.from_numpy(rng.normal(0, 0.5, size=(B, T, K, 3)).astype(np.float32)).cuda()
    gt[..., 2] = torch.from_numpy(rng.choice([0., 1.], size=(B, T, K)).astype(np.float32)).cuda()
    pr = torch.from_numpy(rng.normal(0, 0.5, size=(B, T, K, 2)).astype(np.float32)).cuda()
    a, cam = ops.compute_loss_e_kp_optcam(gt, pr)
    b, cam2 = kp_loss(gt.reshape(B * T, K, 3), pr.reshape(B * T, K, 2), optcam=True)
    assert torch.equal(a, b) and torch.equal(cam.reshape(-1, 3), cam2.reshape(-1, 3))
    _, c3 = projection.batch_orth_proj_optcam(pr.reshape(B * T, K, 2), gt.reshape(B * T, K, 3))
    assert torch.equal(c3, cam2.reshape(-1, 3))
    assert torch.equal(projection.procrustes2d_vis(pr.reshape(B * T, K, 2), gt.reshape(B * T, K, 3)), cam2.reshape(-1, 3))
    assert torch.equal(ops.compute_loss_e_kp(gt, pr), kp_loss(gt.reshape(-1, K, 3), pr.reshape(-1, K, 2))[0])
    p = torch.from_numpy(rng.normal(size=(30, 216)).astype(np.float32)).cuda()
    q = torch.from_numpy(rng.normal(size=(30, 216)).astype(np.float32)).cuda()
    h = torch.from_numpy((rng.uniform(size=30) > 0.5).astype(np.float32)).cuda()
    assert torch.equal(ops.compute_loss_mse(q, p, h), mse_loss(p, q, h, scale=0.5))
    assert torch.equal(ops.compute_loss_e_smooth(p, q), mse_loss(p, q, None, scale=0.5))
    j = torch.from_numpy(rng.normal(size=(30, 14, 3)).astype(np.float32)).cuda()
    al = ops.align_by_pelvis(j)
    assert torch.allclose(al, j - (j[:, 2:3] + j[:, 3:4]) / 2, atol=1e-6)


def test_golden_fixture_values():
    """The fixture made by executing the reference's own losses (tests/golden/losses_v1.npz, B = 3, T = 10): every named loss and every
    optimal camera of the library path to 1e-4."""
    import os
    from human_dynamics_b200.objective import build_objective, evaluate
    with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'losses_v1.npz')) as z:
        gold = {k: z[k] for k in z.files}
    obj = build_objective(cfg(**ALL), 3, 10, 25)
    t = {k: torch.from_numpy(gold[k]).cuda() for k in ('omega', 'joints', 'rots', 'labels', 'gt_rots', 'gt3ds', 'strips', 'pred_strips')}
    t['gt_rots'] = t['gt_rots'].float()
    t['gt_shape'] = torch.from_numpy(gold['shape']).cuda()
    t['w_joints'] = torch.from_numpy(gold['has_3d'][:, 0].copy()).cuda()
    t['w_smpl'] = torch.from_numpy(gold['has_3d'][:, 1].copy()).cuda()
    named, cams = evaluate(obj, t)
    for k in obj.names:
        assert abs(named[k].item() - gold[k]) <= 1e-4 * abs(gold[k]), (k, named[k].item(), gold[k])
    for (g, dt), cam in cams.items():
        ref = gold['cam_%s_%d' % (g, dt)]
        assert np.abs(cam.cpu().numpy() - ref).max() <= 1e-4 * np.abs(ref).max(), (g, dt)


def test_step_issues_no_synchronisation(weights, smpl_model):
    """HMMRTrainer.step queues its work without a host-device synchronisation (after a first step, which builds the objective)."""
    from human_dynamics_b200.objective import HMMRTrainer
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    tr = HMMRTrainer(cfg(**ALL), weights, smpl)
    batch = _target_batch(smpl, 2, 10, smpl.consts.num_kps, 13)
    mocap = _mocap(tr.n_fake(2, 10), 14)
    tr.step(batch, mocap)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = tr.step(batch, mocap)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert np.isfinite(out['e_loss'].item())


def test_labels_take_no_gradient():
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.objective import kp_loss
    gt = torch.rand((4, 25, 3), device='cuda', requires_grad=True)
    pr = torch.rand((4, 25, 2), device='cuda', requires_grad=True)
    with pytest.raises(_lib.HDError):
        kp_loss(gt, pr)
    loss, _ = kp_loss(gt.detach(), pr)
    loss.backward()
    assert torch.isfinite(pr.grad).all()
