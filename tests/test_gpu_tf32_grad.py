"""GPU: the TF32 gradient mode (grad_precision='tf32').  hd_conv_wgrad_ex in 1xTF32 and the 1xTF32 data gradients against a float64
emulation of their operand rounding and against plain float64; the kernel's properties (determinism, the bias row, the impl-1 call, the
refusal of a bad impl); ResNetTrainPlan.backward in 'tf32' against the float64 oracle; HMMRTrainer in 'tf32' (phi and image input):
the forward bit-identical to 'fp32', the gradients near 'fp32''s, torch Adam's step, determinism, the checkpoint, the uint8-frame
path; a 20-step run in both modes; and 'fp32' passed explicitly equal to the default."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch

from tf32_emulation import rn_tf32
from test_gpu_resnet_grad import _batch, _gpu_choices, _mocap, _wgrad_ref

pytestmark = pytest.mark.gpu

# Bars, per-tensor relative L2 unless noted, from measurements on an NVIDIA H100 80GB HBM3 (700 W); the worst measured value is
# next to each bar (DESIGN.md section 2).  Every result is deterministic, so a rerun measures the same values.
EMU_BAR = 1e-5            # against the float64 emulation of the operand rounding, fp32 accumulation noise alone: 6.4e-7
WGRAD_F64_BAR = 1e-3      # hd_conv_wgrad_ex(impl 2) against plain float64: 3.1e-4
DGRAD_F64_BAR = 1e-3      # 1xTF32 data gradients against plain float64: 3.0e-4
TRUNK_BAR = 5e-3          # ResNetTrainPlan.backward('tf32') against the float64 oracle: 1.5e-3 (biases against their weights: 9.0e-9)
GRAD_BAR = 6e-3           # the trainer's 'tf32' gradients against its 'fp32' gradients: 5.8e-4 (phi input), 1.9e-3 (image input)
RUN_BAR = 1e-2            # 20 steps, |e_loss('tf32') - e_loss('fp32')| / e_loss('fp32') at every step: 8.9e-3 (step 6)


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.fixture(scope='module')
def golden_weights():
    from human_dynamics_b200 import synthetic
    return synthetic.make_synthetic_weights(seed=1)


# ------------------------------------------------------------------------------------------------------------------------------------
# hd_conv_wgrad_ex
# ------------------------------------------------------------------------------------------------------------------------------------
def _wgrad_ex(x, geom, pre, dy, Cout, bias, impl, dw=None, db=None):
    from human_dynamics_b200._lib import lib
    n, H, W, Cin, Ho, Wo, KH, KW, s, pt, pl = geom
    dw = torch.empty((KH * KW * Cin, Cout), device='cuda') if dw is None else dw
    db = (torch.empty(Cout, device='cuda') if bias else None) if db is None else db
    wsb = lib.hd_conv_wgrad_workspace_bytes(n * Ho * Wo, KH * KW * Cin, Cout, int(bias))
    ws = torch.empty(max(16, wsb), dtype=torch.uint8, device='cuda')
    args = (_vp(x), Cin, n, H, W, Cin, Ho, Wo, KH, KW, s, pt, pl, _vp(pre[0]) if pre else None, _vp(pre[1]) if pre else None, _vp(dy),
            Cout, Cout, _vp(dw), _vp(db), _vp(ws), ws.numel())
    rc = lib.hd_conv_wgrad(*args, _st()) if impl is None else lib.hd_conv_wgrad_ex(*args, impl, _st())
    return rc, dw, db


def _prologue_f32(x, pre):
    """relu(fma(x, scale, shift)) in fp32, as the producer computes it (the product is exact in float64, one rounding to fp32)."""
    if pre is None:
        return x
    v = (x.astype(np.float64) * pre[0].astype(np.float64) + pre[1].astype(np.float64)).astype(np.float32)
    return np.maximum(v, np.float32(0))


WGRAD_CASES = [
    (3, 28, 64, 256, 1, 1, 0, True, True),          # 1x1 (shortcut / conv3 class), bias row
    (1, 14, 256, 64, 1, 1, 0, True, False),         # n = 1
    (2, 29, 64, 64, 3, 1, 1, True, False),          # SAME 3x3 stride 1, ragged pixel count
    (3, 28, 128, 128, 3, 2, 1, True, False),        # conv2d_same 3x3 stride 2
    (1, 15, 64, 64, 3, 2, 1, False, True),          # odd size, no prologue
    (2, 64, 3, 64, 7, 2, 3, False, True),           # root conv1: 7x7 stride 2 over 3 channels
    (3, 63, 3, 64, 7, 2, 3, False, True),           # conv1, three chunks, the last ragged
    (3, 29, 64, 64, 3, 1, 1, True, True),           # SAME 3x3, two chunks, ragged
    (3, 61, 64, 64, 3, 2, 1, True, False),          # conv2d_same 3x3 stride 2, two chunks, ragged
    (5, 7, 2048, 512, 1, 1, 0, True, False)]        # block 4 shape


def _wgrad_case(n, H, Cin, Cout, K, s, pad, pre, bias):
    rng = np.random.RandomState(n * 100 + H + Cin)
    Ho = (H + 2 * pad - K) // s + 1
    geom = (n, H, H, Cin, Ho, Ho, K, K, s, pad, pad)
    x = rng.normal(0.3, 1, (n, H, H, Cin)).astype(np.float32)
    dy = (rng.normal(0, 1, (n, Ho, Ho, Cout)) * 1e-3).astype(np.float32)
    pv = (rng.uniform(0.5, 1.5, Cin).astype(np.float32), rng.normal(0, 0.5, Cin).astype(np.float32)) if pre else None
    pt = tuple(torch.from_numpy(v).cuda() for v in pv) if pre else None
    return geom, x, dy, pv, pt


@pytest.mark.parametrize('n,H,Cin,Cout,K,s,pad,pre,bias', WGRAD_CASES)
def test_wgrad_1xtf32_against_emulation_and_float64(n, H, Cin, Cout, K, s, pad, pre, bias):
    geom, x, dy, pv, pt = _wgrad_case(n, H, Cin, Cout, K, s, pad, pre, bias)
    xt, dyt = torch.from_numpy(x).cuda(), torch.from_numpy(dy).cuda()
    rc, dw, db = _wgrad_ex(xt, geom, pt, dyt, Cout, bias, 2)
    assert rc == 0
    got = dw.cpu().numpy()
    # the emulation: operands rounded as the kernel rounds them (prologue in fp32, then rn_tf32), products and sums in float64; the
    # prologue is applied before the rounding, so the reference gets it already applied
    ew, eb = _wgrad_ref(rn_tf32(_prologue_f32(x, pv)), geom, None, rn_tf32(dy))
    rw, rb = _wgrad_ref(x, geom, pv, dy)
    e_emu, e_f64 = _rel(got, ew), _rel(got, rw)
    print('wgrad 1xTF32 %s: vs emulation %.2e, vs float64 %.2e' % ((n, H, Cin, Cout, K, s), e_emu, e_f64))
    assert e_emu < EMU_BAR
    assert e_f64 < WGRAD_F64_BAR
    if bias:
        assert _rel(db.cpu().numpy(), rb) < 1e-6


@pytest.mark.parametrize('case', [WGRAD_CASES[0], WGRAD_CASES[3], WGRAD_CASES[6], WGRAD_CASES[7]])
def test_wgrad_1xtf32_properties(case):
    """Repeats are bit-identical; db is bit-identical to the 3xTF32 call's; hd_conv_wgrad is hd_conv_wgrad_ex(impl 1) bit for bit."""
    n, H, Cin, Cout, K, s, pad, pre, bias = case
    geom, x, dy, pv, pt = _wgrad_case(*case)
    xt, dyt = torch.from_numpy(x).cuda(), torch.from_numpy(dy).cuda()
    _, w2a, b2a = _wgrad_ex(xt, geom, pt, dyt, Cout, bias, 2)
    _, w2b, b2b = _wgrad_ex(xt, geom, pt, dyt, Cout, bias, 2)
    _, w1, b1 = _wgrad_ex(xt, geom, pt, dyt, Cout, bias, 1)
    _, w0, b0 = _wgrad_ex(xt, geom, pt, dyt, Cout, bias, None)
    assert torch.equal(w2a, w2b) and torch.equal(w1, w0)
    assert not torch.equal(w2a, w1)                                  # the modes differ
    if bias:
        assert torch.equal(b2a, b2b) and torch.equal(b2a, b1) and torch.equal(b1, b0)


def test_wgrad_ex_bad_impl_launches_nothing():
    from human_dynamics_b200._lib import lib
    geom, x, dy, pv, pt = _wgrad_case(*WGRAD_CASES[0])
    xt, dyt = torch.from_numpy(x).cuda(), torch.from_numpy(dy).cuda()
    dw = torch.full((64, 256), 7.0, device='cuda')
    db = torch.full((256,), 7.0, device='cuda')
    torch.cuda.synchronize()
    for impl in (0, 3, 4, -1, 5):
        lib.hd_launch_count_reset()
        rc, _, _ = _wgrad_ex(xt, geom, pt, dyt, 256, True, impl, dw, db)
        torch.cuda.synchronize()
        assert rc == 1 and lib.hd_launch_count() == 0, impl          # HD_ERR_INVALID, nothing launched
    assert bool((dw == 7).all()) and bool((db == 7).all())


# ------------------------------------------------------------------------------------------------------------------------------------
# 1xTF32 data gradients
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,Cin,Cout,K,s', [(14, 64, 64, 3, 2), (15, 128, 64, 3, 2), (9, 64, 128, 3, 1), (28, 256, 256, 3, 1),
                                            (14, 256, 1024, 1, 1)])
def test_dgrad_op_1xtf32(H, Cin, Cout, K, s):
    from human_dynamics_b200._lib import lib, check
    from human_dynamics_b200.nets import PackedConv, dgrad_op
    from human_dynamics_b200.trainable import BackwardDataPack
    from oracle.nets_ref import conv2d_same
    rng = np.random.RandomState(H + Cin + s + K)
    n = 3
    Ho = (H - 1) // s + 1
    w = (rng.normal(0, 1, (K, K, Cin, Cout)) / np.sqrt(K * K * Cin)).astype(np.float32)
    dy = rng.normal(0, 1, (n, Ho, Ho, Cout)).astype(np.float32)
    wt = torch.from_numpy(w).cuda()
    conv = PackedConv(wt, 'cuda', stride=s, pad=(K // 2, K // 2), tc='auto')
    conv.bwd = BackwardDataPack(wt, K * K, Cin, Cout)
    conv.bwd.repack(_st())
    dyt = torch.from_numpy(dy).cuda()
    src = dyt
    if s > 1:
        src = torch.empty((n, H, H, Cout), device='cuda')
        check(lib.hd_zero_insert(_vp(dyt), _vp(src), n, Ho, Ho, Cout, s, H, H, _st()), 'hd_zero_insert')
    out = torch.empty((n, H, H, Cin), device='cuda')
    op = dgrad_op(conv.bwd, src, n, H, H, K, K, out, one_pass=True)
    assert op.d.impl == 2 and not op.d.w_nk_lo and not op.d.tmap_lo
    op.run(_st())

    def ref(wv, dv):
        xt = torch.zeros((n, H, H, Cin), dtype=torch.float64, requires_grad=True)
        y = conv2d_same(xt, torch.from_numpy(wv.astype(np.float64)), s)
        g, = torch.autograd.grad(y, xt, torch.from_numpy(dv.astype(np.float64)))
        return g.numpy()
    got = out.cpu().numpy()
    e_emu, e_f64 = _rel(got, ref(rn_tf32(w), rn_tf32(dy))), _rel(got, ref(w, dy))
    print('dgrad 1xTF32 %s: vs emulation %.2e, vs float64 %.2e' % ((H, Cin, Cout, K, s), e_emu, e_f64))
    assert e_emu < EMU_BAR
    assert e_f64 < DGRAD_F64_BAR


# ------------------------------------------------------------------------------------------------------------------------------------
# the whole trunk in 'tf32' against the float64 oracle
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n,size', [(2, 224), (16, 224), (4, 64)])
def test_trunk_tf32_gradients_against_oracle(golden_weights, n, size):
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.trunk import TrainableResNet
    from oracle import nets_train_grad_ref as G
    seed = 300 + n + size
    img = synthetic.make_images(n, seed=seed, size=size)
    dphi = np.random.RandomState(seed).normal(0, 1, (n, 2048)).astype(np.float32)
    images, dphi_t = torch.from_numpy(img).cuda(), torch.from_numpy(dphi).cuda()
    nets = {gp: TrainableResNet(golden_weights, grad_precision=gp) for gp in ('fp32', 'tf32')}
    phis, plans = {}, {}
    for gp, net in nets.items():
        phis[gp], plans[gp] = net(images)
    # the forward does not depend on the mode: phis and the batch-norm moments bit for bit
    assert torch.equal(phis['fp32'], phis['tf32'])
    m32, mtf = plans['fp32'].moments(), plans['tf32'].moments()
    assert all(torch.equal(m32[k][0], mtf[k][0]) and torch.equal(m32[k][1], mtf[k][1]) for k in m32)
    net, plan = nets['tf32'], plans['tf32']
    g = torch.autograd.grad(phis['tf32'], list(net.parameters()), dphi_t)
    got = {nm: t for nm, t in zip([k for k, _ in net._params.items()], g)}
    masks = _gpu_choices(plan, n)
    ref, _ = G.trunk_gradients(img, golden_weights, dphi, masks=masks, device='cuda')

    def err(k):                               # biases against their layer's weight gradient (their exact gradient is 0)
        a, r = got[k].cpu().numpy().astype(np.float64), ref[k].cpu().numpy()
        if k.endswith('/biases'):
            return float(np.linalg.norm(a - r) / np.linalg.norm(ref[k[:-len('biases')] + 'weights'].cpu().numpy()))
        return _rel(a, r)
    errs = {k: err(k) for k in ref}
    assert len(errs) == 53 + 21 + 2 * 49
    worst = max(errs.items(), key=lambda kv: kv[1])
    print('trunk tf32 n=%d size=%d: worst per-tensor relative L2 %.3e (%s), worst bias %.3e' % (
        n, size, worst[1], worst[0], max(v for k, v in errs.items() if k.endswith('/biases'))))
    for k, v in errs.items():
        assert v < TRUNK_BAR, (k, v)
    g2 = torch.autograd.grad(net(images)[0], list(net.parameters()), dphi_t)
    assert all(torch.equal(a, b) for a, b in zip(g, g2))


# ------------------------------------------------------------------------------------------------------------------------------------
# HMMRTrainer in 'tf32'
# ------------------------------------------------------------------------------------------------------------------------------------
def _phi_batch(B, T, seed):
    b = _batch(B, T, 16, seed)
    del b['images']
    b['phis'] = torch.from_numpy(np.random.RandomState(seed + 1).normal(0, 1, (B, T, 2048)).astype(np.float32)).cuda()
    return b


def _grad_err(name, g, r, named):
    g, r = g.detach().double().cpu().numpy(), r.detach().double().cpu().numpy()
    if name.endswith('/biases') and name.startswith('resnet_v2_50'):
        return float(np.linalg.norm(g - r) / np.linalg.norm(named[name[:-len('biases')] + 'weights'].double().cpu().numpy()))
    return _rel(g, r)


@pytest.mark.parametrize('image', [False, True])
def test_trainer_tf32(weights, smpl_model, image):
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    B, T, S = 2, 6, 64
    batch = _batch(B, T, S, 5) if image else _phi_batch(B, T, 5)
    kw = dict(precomputed_phi=False, freeze_phi=False) if image else {}
    make = lambda gp: HMMRTrainer(TrainConfig(grad_precision=gp, **kw), weights, smpl)    # noqa: E731
    trs = {gp: make(gp) for gp in ('fp32', 'tf32')}
    mocap = _mocap(trs['fp32'].n_fake(B, T), 6)
    out, grads = {}, {}
    for gp, tr in trs.items():
        named, e_loss, d_loss = tr.forward(batch, mocap)
        out[gp] = (named, e_loss, d_loss)
        ge = torch.autograd.grad(e_loss, tr.e_params, retain_graph=True, allow_unused=True)
        gd = torch.autograd.grad(d_loss, tr.d_params, allow_unused=True)
        grads[gp] = (ge, gd)
    # the forward is the same: every loss bit for bit (and, from images, the phis and the batch moments behind them)
    for k in out['fp32'][0]:
        assert torch.equal(out['fp32'][0][k], out['tf32'][0][k]), k
    assert torch.equal(out['fp32'][1], out['tf32'][1]) and torch.equal(out['fp32'][2], out['tf32'][2])
    if image:
        p32, ptf = trs['fp32']._pending.moments(), trs['tf32']._pending.moments()
        assert all(torch.equal(p32[k][0], ptf[k][0]) and torch.equal(p32[k][1], ptf[k][1]) for k in p32)
    # E's and D's gradients near 'fp32''s
    names = {}
    for gp, tr in trs.items():
        e_names = [n for n, _ in tr.model.named_parameters()] + ([n for n in tr.trunk.net.names] if image else [])
        names[gp] = e_names
    trunk_named = dict(zip(names['tf32'][-172:], grads['fp32'][0][-172:])) if image else {}
    errs = []
    for i, (a, b) in enumerate(zip(grads['tf32'][0], grads['fp32'][0])):
        if a is None:
            assert b is None
            continue
        errs.append((_grad_err(names['tf32'][i], a, b, trunk_named), names['tf32'][i]))
    for i, (a, b) in enumerate(zip(grads['tf32'][1], grads['fp32'][1])):
        errs.append((_rel(a.cpu().numpy(), b.cpu().numpy()), 'D%d' % i))
    worst = max(errs)
    print('trainer tf32 (%s input): worst gradient vs fp32 %.3e (%s)' % ('image' if image else 'phi', worst[0], worst[1]))
    for e, n in errs:
        assert e < GRAD_BAR, (n, e)
    # step: parameters move by exactly torch Adam's step from the 'tf32' gradients; the moving statistics as in 'fp32'
    fresh = make('tf32')
    before = [p.detach().clone() for p in fresh.e_params + fresh.d_params]
    o1 = fresh.step(batch, mocap)
    ps = [torch.nn.Parameter(b.clone()) for b in before]
    ne = len(fresh.e_params)
    opt_e, opt_d = torch.optim.Adam(ps[:ne], fresh.config.e_lr), torch.optim.Adam(ps[ne:], fresh.config.d_lr)
    for p, g in zip(ps, list(grads['tf32'][0]) + list(grads['tf32'][1])):
        p.grad = None if g is None else g.clone()
    opt_e.step()
    opt_d.step()
    for p, q in zip(ps, fresh.e_params + fresh.d_params):
        assert torch.equal(p.detach(), q.detach())
    if image:
        ref32 = make('fp32')
        ref32.step(batch, mocap)
        m_a, m_b = fresh.trunk.bn.moving(), ref32.trunk.bn.moving()
        assert all(np.array_equal(m_a[k], m_b[k]) for k in m_a)
    # repeats: the same two steps from the same state, bit for bit
    again = make('tf32')
    o2 = again.step(batch, mocap)
    for k in o1:
        assert torch.equal(o1[k], o2[k]), k
    assert all(torch.equal(p, q) for p, q in zip(fresh.e_params + fresh.d_params, again.e_params + again.d_params))
    fresh.step(batch, mocap)
    again.step(batch, mocap)
    assert all(torch.equal(p, q) for p, q in zip(fresh.e_params + fresh.d_params, again.e_params + again.d_params))
    # the checkpoint loads in HMMREngine
    if image:
        from human_dynamics_b200.engine import HMMREngine, load_weights
        with tempfile.TemporaryDirectory() as d:
            w2 = load_weights(fresh.save_checkpoint(os.path.join(d, 'model.ckpt-2')))
        for n in fresh.trunk.net.names:
            assert np.array_equal(w2[n].reshape(-1), fresh.trunk.net.param(n).detach().cpu().numpy().reshape(-1)), n
        eng = HMMREngine(w2, smpl_model)
        phi = eng.encode_images(batch['images'].reshape(B * T, S, S, 3))
        assert bool(torch.isfinite(phi).all())


def test_trainer_tf32_from_uint8_frames(weights, smpl_model):
    from human_dynamics_b200.augment import TubeAugmentor
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    B, T, S = 2, 5, 64
    rng = np.random.RandomState(12)
    frames = rng.randint(0, 256, size=(B * T, 96, 120, 3)).astype(np.uint8)
    lab = np.stack([rng.uniform(0, 120, (B * T, 25)), rng.uniform(0, 96, (B * T, 25)), np.ones((B * T, 25))], 1).astype(np.float32)
    cen = np.stack([rng.randint(40, 80, B * T), rng.randint(30, 60, B * T)], 1).astype(np.int32)
    pose = rng.normal(0, 0.3, (B * T, 72)).astype(np.float32)
    g3 = rng.normal(0, 0.3, (B * T, 14, 3)).astype(np.float32)
    r = TubeAugmentor(img_size=S, seed=7)(frames, lab, cen, pose, g3, tube_lengths=[T] * B)
    batch = {'images': r['images'].view(B, T, S, S, 3), 'labels': r['labels'].transpose(1, 2).reshape(B, T, 25, 3).contiguous(),
             'poses': r['poses'].reshape(B, T, 72), 'shape': torch.zeros((B, 10), device='cuda'),
             'gt3ds': r['gt3ds'].reshape(B, T, 14, 3), 'has_3d': torch.ones((B, 2), device='cuda')}
    tr = HMMRTrainer(TrainConfig(precomputed_phi=False, freeze_phi=False, grad_precision='tf32'), weights, smpl)
    before = [p.detach().clone() for p in tr.trunk.net.parameters()]
    out = tr.step(batch, _mocap(tr.n_fake(B, T), 3))
    assert all(v.shape == () and torch.isfinite(v) for v in out.values())
    assert any(not torch.equal(a, b.detach()) for a, b in zip(before, tr.trunk.net.parameters()))


# ------------------------------------------------------------------------------------------------------------------------------------
# a short run, and 'fp32' unchanged
# ------------------------------------------------------------------------------------------------------------------------------------
def test_twenty_steps_in_both_modes(weights, smpl_model):
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    B, T = 2, 20
    batch = _phi_batch(B, T, 9)
    curves = {}
    for gp in ('fp32', 'tf32'):
        tr = HMMRTrainer(TrainConfig(grad_precision=gp, e_lr=1e-4), weights, smpl)
        mocap = _mocap(tr.n_fake(B, T), 10)
        curves[gp] = [float(tr.step(batch, mocap)['e_loss']) for _ in range(20)]
    a, b = np.array(curves['tf32']), np.array(curves['fp32'])
    dev = np.abs(a - b) / np.abs(b)
    print('20 steps: e_loss fp32 %.6g -> %.6g, tf32 %.6g -> %.6g, worst relative difference %.3e (step %d)'
          % (b[0], b[-1], a[0], a[-1], dev.max(), int(dev.argmax())))
    assert b[-1] < b[0] and a[-1] < a[0]
    assert dev.max() < RUN_BAR


def test_explicit_fp32_equals_the_default(weights, smpl_model):
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    B, T, S = 2, 4, 64
    batch = _batch(B, T, S, 21)
    res = []
    for kw in ({}, {'grad_precision': 'fp32'}):
        tr = HMMRTrainer(TrainConfig(precomputed_phi=False, freeze_phi=False, **kw), weights, smpl)
        out = tr.step(batch, _mocap(tr.n_fake(B, T), 22))
        res.append((out, [p.detach().clone() for p in tr.e_params + tr.d_params]))
    for k in res[0][0]:
        assert torch.equal(res[0][0][k], res[1][0][k]), k
    assert all(torch.equal(p, q) for p, q in zip(res[0][1], res[1][1]))
