"""GPU: the IEF heads' training-mode dropout (csrc/dropout.cuh, hd_ief_fc1_theta_dropout / hd_ief_fc3_dropout, the scaled ReLU
backwards, nets.IEFPlan(dropout=...), TemporalModel.regress(dropout=...), TrainConfig.ief_keep_prob).  The masks bit for bit against
oracle/dropout_ref.py; the forward against tests/golden/ief_dropout_v1.npz (the reference's own batch_pred_omega(is_training=True))
and the float64 oracle with the same masks; ief_keep_prob 1 bit-identical to a trainer without it; the gradients against the masked
float64 grad oracle in both gradient precisions; trainer reproducibility from the seed and across resume; mask statistics."""
import itertools
import os

import numpy as np
import pytest
import torch

from oracle import dropout_ref as D
from test_gpu_resnet_grad import _mocap
from test_gpu_tf_adam import _phi_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
KEYS = (-5, 5)
REL = 1e-4          # the FP32-class bar of the IEF tests (test_gpu_temporal_grad.py)
GUARD = 2.5e-5      # as there: where the float32 oracle is off by this much, the case is judged against 10x its error
MARGIN = 1e-5       # as there: |pre-activation| below this takes the GPU's ReLU sign
TF32_BAR = 6e-3     # 'tf32' gradients, relative L2 against the float64 oracle (test_gpu_tf32_grad.py's GRAD_BAR)


def rel_err(a, b):
    a, b = a.detach().double(), b.detach().double().to(a.device)
    return float((a - b).abs().max() / max(b.abs().max().item(), 1e-300))


def rel_l2(a, b):
    a, b = a.detach().double(), b.detach().double().to(a.device)
    return float((a - b).norm() / max(b.norm().item(), 1e-300))


@pytest.fixture(scope='module')
def gweights():
    from human_dynamics_b200 import synthetic
    return synthetic.make_synthetic_weights(seed=1, with_hal=True)


@pytest.fixture(scope='module')
def model(gweights):
    from human_dynamics_b200.trainable import TemporalModel
    return TemporalModel(gweights)


@pytest.fixture(scope='module')
def golden():
    with np.load(os.path.join(ROOT, 'tests', 'golden', 'ief_dropout_v1.npz')) as z:
        return {k: z[k] for k in z.files}


def _device_mask(seed, step, site, N, C, p):
    from human_dynamics_b200._lib import check, current_stream, lib
    out = torch.full((N * C + 16,), 7, dtype=torch.uint8, device='cuda')
    check(lib.hd_dropout_mask(seed, step, site, N, C, p, out.data_ptr(), current_stream()), 'hd_dropout_mask')
    o = out.cpu().numpy()
    assert (o[N * C:] == 7).all()                          # nothing written past N*C
    return o[:N * C].reshape(N, C)


# ------------------------------------------------------------------------------------------------------------------------------------
# masks
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('seed,step,site,N,C,p', [
    (1, 0, 0, 160, 1024, 0.5), (1, 7, 37, 3, 7, 0.5), (0xfedcba9876543210, 2 ** 32 + 5, 101, 5, 1023, 0.7),
    (42, 2 ** 40 + 3, 3, 17, 85, 0.9), (2 ** 64 - 1, 2 ** 64 - 1, 127, 1, 1, 0.5), (9, 12, 64, 160, 1024, 0.3)])
def test_device_mask_equals_host(seed, step, site, N, C, p):
    p32 = float(D.nn_keep_prob(p))
    got = _device_mask(seed, step, site, N, C, p32)
    assert np.array_equal(got, D.mask(seed, step, site, N, C, p32))
    # rows are chunks of the same stream: a call over the first n rows draws their masks
    for n in {1, N // 2, N - 1} - {0}:
        assert np.array_equal(_device_mask(seed, step, site, n, C, p32), got[:n])


def test_bad_arguments_are_refused():
    from human_dynamics_b200._lib import current_stream, lib
    out = torch.empty(64, dtype=torch.uint8, device='cuda')
    for p in (0.0, -0.5, 1.5, float('nan')):
        assert lib.hd_dropout_mask(1, 0, 0, 4, 4, p, out.data_ptr(), current_stream()) == 1
    assert lib.hd_dropout_mask(1, 0, -1, 4, 4, 0.5, out.data_ptr(), current_stream()) == 1
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200.objective import TrainConfig
    for p in (0.0, -1.0, 1.0001):
        with pytest.raises(HDError):
            TrainConfig(ief_keep_prob=p)


# ------------------------------------------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------------------------------------------
def _masks(golden, name, N):
    m = D.ief_masks(int(golden['seed']), int(golden['%s_step' % name]), int(golden['%s_call' % name]), N, 1 + len(KEYS),
                    D.nn_keep_prob(0.5))
    return m, {dt: [(m[(h, s, 0)], m[(h, s, 1)]) for s in range(3)] for h, dt in enumerate((0,) + KEYS)}


@pytest.mark.parametrize('name', ['pred', 'hal'])
def test_forward_matches_reference_and_oracle(model, gweights, golden, name):
    from oracle import ief_dropout_ref
    from human_dynamics_b200.trainable import regress_plan
    B, T = int(golden['B']), int(golden['T'])
    N = B * T
    feats = torch.from_numpy(golden['%s_feats' % name].reshape(N, 2048)).cuda()
    spec = (int(golden['seed']), int(golden['%s_step' % name]), int(golden['%s_call' % name]), float(golden['keep_prob']))
    with torch.no_grad():
        th, dl = model.regress(feats, dropout=spec)
    m, masks = _masks(golden, name, N)
    start = np.tile(np.asarray(gweights['mean_param'], np.float32).reshape(1, 85), (N, 1))
    om64, dl64 = ief_dropout_ref.batch_pred_omega(golden['%s_feats' % name], B, gweights, start, T, KEYS, masks, 0.5)
    for got, ref, o64 in [(th, golden['%s_omega' % name], om64)] + [(dl[k], golden['%s_delta_%d' % (name, k)], dl64[k]) for k in KEYS]:
        got = got.cpu().double().reshape(B, T, 85)
        assert rel_err(got, torch.from_numpy(ref)) < REL
        assert rel_err(got, o64) < REL
    # the activations the backward reads are the masked ones: nothing survives where the mask drops, 2 * relu where it keeps
    with torch.no_grad():
        plan = regress_plan(model, KEYS, True, feats, model.param('mean_param'), spec)[2]
    for h, (h1, h2, _, _) in enumerate(plan.saved):
        for s in range(3):
            for layer, act in ((0, h1[s]), (1, h2[s])):
                keep = torch.from_numpy(m[(h, s, layer)]).cuda().bool()
                assert not (act[~keep] != 0).any(), (h, s, layer)
                assert (act[keep] > 0).any()
    # a call over the first rows is the first rows of the call
    with torch.no_grad():
        th4, dl4 = model.regress(feats[:4].contiguous(), dropout=spec)
    assert torch.equal(th4, th[:4]) and all(torch.equal(dl4[k], dl[k][:4]) for k in KEYS)


def test_keep_prob_one_is_the_inference_graph(model):
    rng = np.random.RandomState(5)
    feats = torch.from_numpy(rng.normal(0, 1, (40, 2048)).astype(np.float32)).cuda()
    with torch.no_grad():
        a, da = model.regress(feats)
        b, db = model.regress(feats, dropout=(3, 11, 0, 1.0))
        c, _ = model.regress(feats, dropout=(3, 11, 0, 0.5))
    assert torch.equal(a, b) and all(torch.equal(da[k], db[k]) for k in KEYS)
    assert not torch.equal(a, c)


def test_trainer_keep_prob_one_is_bit_identical(gweights, smpl_model):
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    kw = dict(do_hallucinate=True, do_hallucinate_preds=True, e_lr=1e-4)
    plain = HMMRTrainer(TrainConfig(**kw), gweights, smpl)
    ones = HMMRTrainer(TrainConfig(ief_keep_prob=1.0, seed=99, **kw), gweights, smpl)
    for s in range(2):
        batch, mocap = _phi_batch(2, 6, 60 + s), _mocap(plain.n_fake(2, 6), 70 + s)
        la, lb = plain.step(batch, mocap), ones.step(batch, mocap)
        assert all(torch.equal(la[k], lb[k]) for k in la)
    assert all(torch.equal(p, q) for p, q in zip(plain.e_params + plain.d_params, ones.e_params + ones.d_params))


# ------------------------------------------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------------------------------------------
def _ief_names():
    from human_dynamics_b200.trainable import ief_names
    return [n for dt in (0,) + KEYS for n in ief_names(dt)]


@pytest.mark.parametrize('precision', ['fp32', 'tf32'])
@pytest.mark.parametrize('BT', [(2, 20), (3, 7)])
def test_grads_match_masked_oracle(gweights, BT, precision):
    """Both IEF calls of a step (call 0 over f_movie's strips, call 1 over fc2_res's), every head, with dropout at keep_prob 0.5:
    the gradients of phi, f_movie, every IEF head's six parameters, mean_param and fc2_res against the float64 oracle with the same
    masks and the GPU's ReLU signs at near-ties."""
    from oracle import ief_dropout_ref as R, nets_grad_ref as g
    from human_dynamics_b200.objective import TrainConfig
    from human_dynamics_b200.trainable import HAL_NAMES, TemporalModel, regress_plan, trainable_names
    model = TemporalModel(gweights, TrainConfig(grad_precision=precision))
    B, T = BT
    N = B * T
    names = trainable_names(gweights)
    seed, step = 1234, 2 ** 32 + 6
    rng = np.random.RandomState(B * 10 + T)
    ups = [torch.from_numpy(rng.normal(0, 1, size=(N, 85)).astype(np.float32)).cuda() for _ in range(6)]
    phi = torch.from_numpy(rng.normal(0, 1, size=(B, T, 2048)).astype(np.float32)).cuda().requires_grad_()
    f = model.temporal_encode(phi)
    hal = model.hallucinate(phi)
    outs = []
    for call, x in enumerate((f, hal)):
        th, dl = model.regress(x.reshape(N, 2048), dropout=(seed, step, call, 0.5))
        outs += [th] + [dl[k] for k in KEYS]
    loss = sum((o * u).sum() for o, u in zip(outs, ups))
    got = dict(zip(['phi'] + names, torch.autograd.grad(loss, [phi] + [model.param(n) for n in names])))
    # oracle masks: dropout from oracle/dropout_ref, ReLU signs from float64 except near ties (the GPU's, read from its saved activations)
    p = float(D.nn_keep_prob(0.5))
    heads = ['main'] + ['d%d' % k for k in KEYS]
    drops, relus = [], []
    gpu = model.relu_masks(phi=phi.detach(), hal=phi.detach().reshape(-1, 2048))
    L = g.leaves(gweights, names, F64, 'cuda')
    hal_p = tuple(L[n] for n in HAL_NAMES)
    with torch.no_grad():
        rec = {}
        x64 = phi.detach().double()
        f64 = g.fmovie(x64, g.fmovie_blocks(L), None, rec)
        h64 = g.fc2_res(x64.reshape(N, 2048), hal_p, None, rec)
        base = {n: torch.where(pre.abs() < MARGIN, gpu[n].to(pre.device).reshape(pre.shape), pre > 0) for n, pre in rec.items()}
        for call, (x, x64c) in enumerate(((f, f64), (hal, h64))):
            m = D.ief_masks(seed, step, call, N, 1 + len(KEYS), p)
            drop = ({k: v.cuda() for k, v in R.drop_sites(m, KEYS).items()}, p)
            crec = {}
            R.grad_call_hmr_ief(x64c.reshape(N, 2048), L['mean_param'].reshape(1, 85).expand(N, 85),
                                {dt: g.ief_params(L, dt) for dt in (0,) + KEYS}, KEYS, drop, None, crec)
            plan = regress_plan(model, KEYS, True, x.detach().reshape(N, 2048), model.param('mean_param'), (seed, step, call, 0.5))[2]
            rm = {}
            for hn, (h1, h2, _, _) in zip(heads, plan.saved):
                for s in range(3):
                    for layer, act in ((1, h1[s]), (2, h2[s])):
                        n = '%s.s%d.fc%d' % (hn, s, layer)
                        keep = drop[0][n]
                        near = (crec[n].abs() < MARGIN) & keep
                        rm[n] = torch.where(near, act > 0, crec[n] > 0)
            drops.append(drop)
            relus.append(rm)

    def oracle(dtype):
        Lx = g.leaves(gweights, names, dtype, 'cuda')
        x = phi.detach().to(dtype).requires_grad_()
        fx = g.fmovie(x, g.fmovie_blocks(Lx), base)
        hx = g.fc2_res(x.reshape(N, 2048), tuple(Lx[n] for n in HAL_NAMES), base)
        o = []
        for call, xs in enumerate((fx, hx)):
            th, dl = R.grad_call_hmr_ief(xs.reshape(N, 2048), Lx['mean_param'].reshape(1, 85).expand(N, 85),
                                         {dt: g.ief_params(Lx, dt) for dt in (0,) + KEYS}, KEYS, drops[call], relus[call])
            o += [th] + [dl[k] for k in KEYS]
        lo = sum((a * u.to(dtype)).sum() for a, u in zip(o, ups))
        return dict(zip(['phi'] + names, torch.autograd.grad(lo, [x] + [Lx[n] for n in names])))
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        r64, r32 = oracle(F64), oracle(torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    judged = ['phi'] + names
    assert set(_ief_names()) | {'mean_param'} | set(HAL_NAMES) <= set(judged)
    worst, relaxed = [], []
    for n in judged:
        assert got[n] is not None and torch.isfinite(got[n]).all(), n
        if precision == 'tf32':
            e = rel_l2(got[n], r64[n])
            worst.append((e, n))
            assert e < TF32_BAR, (n, e)
            continue
        e32, e = rel_err(r32[n], r64[n]), rel_err(got[n], r64[n])
        bar = REL
        if e32 >= GUARD:
            bar = max(REL, 10 * e32)
            relaxed.append((n, e32, e))
        worst.append((e, n))
        assert e < bar, (n, e, e32)
    print('%s BT=%s worst: %s; relaxed: %s' % (precision, BT, max(worst), relaxed))
    assert len(relaxed) <= len(judged) // 4, relaxed


# ------------------------------------------------------------------------------------------------------------------------------------
# the trainer
# ------------------------------------------------------------------------------------------------------------------------------------
def _cfg(seed):
    from human_dynamics_b200.objective import TrainConfig
    return TrainConfig(do_hallucinate=True, do_hallucinate_preds=True, e_lr=1e-4, ief_keep_prob=0.5, seed=seed)


def _data(n_fake, steps):
    return [(_phi_batch(2, 6, 80 + s), _mocap(n_fake, 90 + s)) for s in range(steps)]


def test_trainer_is_reproducible_from_its_seed(gweights, smpl_model):
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    trs = [HMMRTrainer(_cfg(s), gweights, smpl) for s in (1, 1, 2)]
    plain = HMMRTrainer(TrainConfig(do_hallucinate=True, do_hallucinate_preds=True, e_lr=1e-4), gweights, smpl)
    data = _data(trs[0].n_fake(2, 6), 3)
    for d in data:
        la, lb, lc, lp = (t.step(*d) for t in trs + [plain])
        assert all(torch.equal(la[k], lb[k]) for k in la)
        assert not torch.equal(la['e_loss'], lc['e_loss']) and not torch.equal(la['e_loss'], lp['e_loss'])
    assert all(torch.equal(p, q) for p, q in zip(trs[0].e_params + trs[0].d_params, trs[1].e_params + trs[1].d_params))
    assert any(not torch.equal(p, q) for p, q in zip(trs[0].e_params, trs[2].e_params))


def test_resume_continues_the_mask_stream(gweights, smpl_model, tmp_path):
    from human_dynamics_b200.objective import HMMRTrainer
    from human_dynamics_b200.optim import TFAdam
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    cfg = _cfg(7)
    straight = HMMRTrainer(cfg, gweights, smpl, optimizer=TFAdam)
    data = _data(straight.n_fake(2, 6), 3)
    la = [straight.step(*d) for d in data]
    first = HMMRTrainer(cfg, gweights, smpl, optimizer=TFAdam)
    for d in data[:2]:
        first.step(*d)
    prefix = first.save_checkpoint(str(tmp_path / ('model.ckpt-%d' % first.global_step)))
    del first
    resumed = HMMRTrainer.resume(cfg, prefix, smpl)
    assert resumed.global_step == 4
    lb = resumed.step(*data[2])
    assert all(torch.equal(la[2][k], lb[k]) for k in lb)
    va, vb = straight.tf_variables(), resumed.tf_variables()
    assert sorted(va) == sorted(vb)
    for n in va:
        assert np.array_equal(va[n], vb[n]), n


def test_mask_statistics_over_a_step():
    """Every mask of one step at B = 8, T = 20 (both calls, three heads, three stages, two layers) and of the next step: each keeps
    half its elements, and any two (sites, calls, steps) agree on half, within 6 sigma: no stream is reused."""
    N, C = 160, 1024
    n = N * C
    sigma = 0.5 / np.sqrt(n)
    t = 1234
    masks = {}
    for step, call, h, s, layer in itertools.product((t, t + 1, t + 2), (0, 1), range(3), range(3), (0, 1)):
        masks[(step, call, h, s, layer)] = _device_mask(1, step, D.site(call, h, s, layer), N, C, 0.5).astype(bool).reshape(-1)
    for k, m in masks.items():
        assert abs(m.mean() - 0.5) < 6 * sigma, k
    keys = list(masks)
    worst = 0.0
    for a, b in itertools.combinations(keys, 2):
        agree = float((masks[a] == masks[b]).mean())
        worst = max(worst, abs(agree - 0.5) / sigma)
        assert abs(agree - 0.5) < 6 * sigma, (a, b, agree)
    print('%d masks, %d pairs, worst |agreement - 0.5| = %.2f sigma' % (len(keys), len(keys) * (len(keys) - 1) // 2, worst))
