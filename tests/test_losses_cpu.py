"""CPU: the trainer objective's key set, weights and mocap count against the reference trainer's, the float64 oracle
(oracle/losses_ref.py) against closed forms and against the fixture made by executing the reference's own losses
(tests/golden/losses_v1.npz), and the C-ABI's argument checks of the loss entries (no device needed)."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

# trainer_sequence_fc.py:235-274, the keys of self.losses (the static use_hmr_only branch is not built)
BASE = {'d_pose', 'e_const', 'e_joints', 'e_kp', 'e_pose', 'e_shape', 'e_smpl'}
DELTA = {'e_joints_dt_future', 'e_kp_dt_future', 'e_smpl_dt_future', 'e_joints_dt_past', 'e_kp_dt_past', 'e_smpl_dt_past'}
HAL = {'e_hallucinate', 'e_joints_hal', 'e_kp_hal', 'e_smpl_hal'}
HAL_PREDS = {'e_joints_hal_future', 'e_kp_hal_future', 'e_smpl_hal_future', 'e_joints_hal_past', 'e_kp_hal_past', 'e_smpl_hal_past'}


def _cfg(**kw):
    from human_dynamics_b200.objective import TrainConfig
    return TrainConfig(**kw)


def test_version():
    from human_dynamics_b200 import _lib
    assert _lib.lib.hd_version() >= 104


def test_defaults_are_the_references():
    c = _cfg()
    assert (c.e_lw_kp, c.e_lw_joints, c.e_lw_smpl) == (60, 60, 60)
    assert (c.e_lw_const, c.e_lw_pose, c.e_lw_shape, c.e_lw_hallucinate, c.d_lw_pose) == (1, 1, 1, 1, 1)
    assert (c.e_lr, c.d_lr) == (1e-5, 1e-4)
    assert c.use_3d_label and c.predict_delta and not c.mosh_ignore and not c.do_hallucinate and not c.do_hallucinate_preds


@pytest.mark.parametrize('pd,hal,halp,u3d', list(itertools.product([False, True], repeat=4)))
def test_key_set_and_weights(pd, hal, halp, u3d):
    from human_dynamics_b200.objective import build_objective, loss_keys
    c = _cfg(predict_delta=pd, do_hallucinate=hal, do_hallucinate_preds=halp, use_3d_label=u3d, e_lw_kp=3., e_lw_joints=5., e_lw_smpl=7.,
             e_lw_const=11., e_lw_pose=13., e_lw_shape=17., e_lw_hallucinate=19., d_lw_pose=23.)
    want = set(BASE)
    if pd:
        want |= DELTA
    if hal:
        want |= HAL
        if halp:
            want |= HAL_PREDS
    assert set(loss_keys(c)) == want
    obj = build_objective(c, 2, 10, 25)
    assert set(obj.names) | {'d_pose', 'e_pose'} == want
    assert set(obj.weights) == want
    for k, w in obj.weights.items():
        exp = {'d_pose': 23., 'e_const': 11., 'e_pose': 13., 'e_shape': 17., 'e_hallucinate': 19.}.get(k)
        if exp is None:
            exp = {'e_kp': 3., 'e_joints': 5., 'e_smpl': 7.}['_'.join(k.split('_')[:2])]
        assert w == exp, k
    # every named loss has terms exactly when the reference computes something for it
    for n in obj.names:
        has = any(m == n for m in obj.term_names)
        if n.startswith('e_joints') or n.startswith('e_smpl'):
            assert has == u3d, n
        else:
            assert has, n


@pytest.mark.parametrize('pd,hal,halp', list(itertools.product([False, True], repeat=3)))
def test_n_fake(pd, hal, halp):
    """data_loader_sequence.py:185-196, restated."""
    from human_dynamics_b200.objective import n_fake, prediction_sets
    B, T = 8, 20
    c = _cfg(predict_delta=pd, do_hallucinate=hal, do_hallucinate_preds=halp)
    mosh = B * T
    delta = B * 2 * T if pd else 0
    if hal:
        mosh *= 2
        if halp:
            delta *= 2
    assert n_fake(c, B, T) == mosh + delta
    if pd or not (hal and halp):
        assert len(prediction_sets(c)) * B * T == n_fake(c, B, T)
    assert n_fake(_cfg(do_hallucinate=True, do_hallucinate_preds=True), 8, 20) == 960


def test_pred_poses_all_order():
    """trainer_sequence_fc.py:586-633: the hallucinated sets first (present, then the delta_t order), the prediction, the delta heads."""
    from human_dynamics_b200.objective import prediction_sets
    assert prediction_sets(_cfg(do_hallucinate=True, do_hallucinate_preds=True)) == \
        [('hal', 0), ('hal', -5), ('hal', 5), ('pred', 0), ('dt', -5), ('dt', 5)]
    assert prediction_sets(_cfg(predict_delta=False)) == [('pred', 0)]


def test_oracle_divisors_and_zero_counts():
    from oracle import losses_ref as R
    gt = torch.zeros(2, 3, 3, dtype=torch.float64)
    gt[0, 0, 2] = 1.
    gt[1, 2, 2] = 0.5
    gt[..., :2] = 1.
    pred = torch.zeros(2, 3, 2, dtype=torch.float64)
    # sum v |x - xhat| = 1 * 2 + 0.5 * 2 = 3; divisor 2 * (visible) = 4
    assert R.compute_loss_e_kp(gt, pred).item() == pytest.approx(0.75)
    assert R.compute_loss_e_kp(gt * torch.tensor([1., 1., 0.], dtype=torch.float64), pred).item() == 0.0
    p = torch.ones(4, 216, dtype=torch.float64)
    has = torch.tensor([1., 0., 0., 1.], dtype=torch.float64)
    assert R.compute_loss_mse(p * 0, p, has).item() == pytest.approx(0.5)
    assert R.compute_loss_mse(p * 0, p, has * 0).item() == 0.0


def test_oracle_procrustes_recovers_a_known_camera():
    from oracle import losses_ref as R
    rng = np.random.RandomState(0)
    x = torch.from_numpy(rng.normal(size=(5, 25, 2)))
    s, t = torch.tensor([[0.9], [1.3], [2.0], [5.0], [1.0]], dtype=torch.float64), torch.from_numpy(rng.normal(size=(5, 2)))
    y = s[:, :, None] * (x + t[:, None])
    tgt = torch.cat([y, torch.ones(5, 25, 1, dtype=torch.float64)], -1)
    cam, empty = R.procrustes2d_vis(x, tgt)
    assert not empty.any()
    assert torch.allclose(cam[:, 0:1], s, rtol=1e-5) and torch.allclose(cam[:, 1:], t, atol=1e-5)
    flipped = torch.cat([-y[..., :1], y[..., 1:], torch.ones(5, 25, 1, dtype=torch.float64)], -1)
    assert (R.procrustes2d_vis(x, flipped)[0][:, 0] >= 0.7).all()


def _term(**kw):
    from human_dynamics_b200 import _lib
    t = _lib.LossTerm()
    t.kind, t.proj, t.B, t.Tw, t.p_T, t.q_T, t.K, t.D, t.scale = _lib.HD_LOSS_MSE_ROWS, 0, 2, 4, 4, 4, 0, 10, 1.
    t.p, t.p_clip, t.p_frame = 4096, 40, 10
    for k, v in kw.items():
        setattr(t, k, v)
    return t


def test_abi_argument_checks_without_device():
    from human_dynamics_b200 import _lib
    L = _lib.lib
    p = ctypes.c_void_p(4096)          # never dereferenced: every call below fails its argument check first

    def arr(*ts):
        return (_lib.LossTerm * len(ts))(*ts)
    good = arr(_term())
    ws = L.hd_loss_workspace_bytes(good, 1)
    assert ws > 0
    assert L.hd_loss_workspace_bytes(None, 1) == 0 and L.hd_loss_workspace_bytes(good, 0) == 0
    assert L.hd_loss_forward(good, 1, None, p, ws, None) == 1                                          # null values
    assert L.hd_loss_forward(good, 1, p, p, ws - 4, None) == 1                                          # workspace too small
    assert L.hd_loss_forward(arr(_term(p=None)), 1, p, p, ws, None) == 1                                # null p
    assert L.hd_loss_forward(arr(_term(p_t0=1)), 1, p, p, ws, None) == 1                                # window overruns T
    assert L.hd_loss_forward(arr(_term(q=8192, q_clip=40, q_frame=10, q_t0=2, q_T=5)), 1, p, p, ws, None) == 1
    assert L.hd_loss_forward(arr(_term(proj=1, D=39)), 1, p, p, ws, None) == 1                          # pelvis on 13 joints
    assert L.hd_loss_forward(arr(_term(kind=_lib.HD_LOSS_KP_L1, K=25, D=3)), 1, p, p, ws, None) == 1   # KP without labels
    assert L.hd_loss_forward(arr(_term(kind=_lib.HD_LOSS_KP_L1, K=25, D=3, q=8192, q_clip=300, q_frame=75)), 1, p, p, ws,
                             None) == 1                                                                 # KP_CAMERA without cam
    assert L.hd_loss_forward(arr(_term(kind=7)), 1, p, p, ws, None) == 1
    assert L.hd_loss_forward(arr(*[_term()] * 65), 65, p, p, ws, None) == 1                             # too many terms
    g = (_lib.LossGrad * 1)()
    g[0].src, g[0].grad, g[0].numel = 4096, 65536, 80
    assert L.hd_loss_backward(good, 1, g, 1, None, p, ws, None) == 1                                    # null dvalues
    assert L.hd_loss_backward(good, 1, g, 0, p, p, ws, None) == 1                                       # no target
    assert L.hd_loss_backward(good, 1, g, 1, p, p, ws - 4, None) == 1
    assert L.hd_loss_backward(arr(_term(p_frame=0)), 1, g, 1, p, p, ws, None) == 1                      # gradient through stride 0
    assert b'hd_loss' in L.hd_last_error()


# ---- the fixture made by executing the reference's own losses (tests/golden/make_losses_golden.py) ----
import importlib.util  # noqa: E402
import os  # noqa: E402
import subprocess  # noqa: E402
import sys  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
GEN = os.path.join(HERE, 'golden', 'make_losses_golden.py')


def _gen():
    spec = importlib.util.spec_from_file_location('_make_losses_golden', GEN)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def gold():
    with np.load(os.path.join(HERE, 'golden', 'losses_v1.npz')) as z:
        return {k: z[k] for k in z.files}


def gold_inputs(gold, dtype=torch.float64):
    t = {k: torch.from_numpy(gold[k]).to(dtype) for k in ('omega', 'joints', 'rots', 'labels', 'gt_rots', 'gt3ds', 'strips', 'pred_strips')}
    t['gt_shape'] = torch.from_numpy(gold['shape']).to(dtype)
    t['w_joints'] = torch.from_numpy(gold['has_3d'][:, 0]).to(dtype).contiguous()
    t['w_smpl'] = torch.from_numpy(gold['has_3d'][:, 1]).to(dtype).contiguous()
    return t


GOLD_CFG = dict(do_hallucinate=True, do_hallucinate_preds=True)


def test_golden_inputs_regenerate(gold):
    x = _gen().inputs()
    for k, v in x.items():
        assert np.array_equal(v, gold[k]), k


@pytest.mark.skipif(not os.path.isdir(os.path.join(os.environ.get('HD_REFERENCE_ROOT', '/nonexistent'), 'src')),
                    reason='HD_REFERENCE_ROOT does not name a reference checkout')
def test_golden_generator_reproduces_the_fixture():
    r = subprocess.run([sys.executable, GEN, '--check'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout


def test_oracle_matches_golden(gold):
    """Every named loss and every optimal camera of oracle/losses_ref.py equals the reference's own, executed, to 1e-6 relative; and the
    fixture's key set, weights and e_loss are the objective's."""
    from human_dynamics_b200.objective import build_objective, loss_keys
    from oracle import losses_ref as R
    c = _cfg(**GOLD_CFG)
    named, cams = R.objective(c, gold_inputs(gold))
    keys = loss_keys(c)
    assert set(keys) <= set(gold) and set(named) == set(keys) - {'d_pose', 'e_pose'}
    for k, v in named.items():
        assert abs(v.item() - gold[k]) <= 1e-6 * abs(gold[k]), (k, v.item(), gold[k])
    assert len(cams) == 4
    for (g, dt), cam in cams.items():
        ref = gold['cam_%s_%d' % (g, dt)]
        assert np.abs(cam.numpy() - ref).max() <= 1e-6 * np.abs(ref).max(), (g, dt)
    assert gold['cam_hal_-5'][0, 0, 0] == pytest.approx(0.7)          # the mirrored frame hits the scale clip
    obj = build_objective(c, 3, 10, 25)
    e = sum(gold[k] * obj.weights[k] for k in obj.names) + gold['e_pose'] * obj.weights['e_pose']
    assert e == pytest.approx(float(gold['e_loss']), rel=1e-12)
    assert float(gold['d_loss']) == pytest.approx(float(gold['d_pose']) * obj.weights['d_pose'], rel=1e-12)
