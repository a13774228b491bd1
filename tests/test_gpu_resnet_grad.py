"""GPU: the trunk's backward (freeze_phi=False).  hd_conv_wgrad, hd_bn_relu_backward, pool1's backward and the strided / 2-D data
gradients against float64; ResNetTrainPlan.backward against the float64 autograd oracle (oracle/nets_train_grad_ref.py) run on the
device; and HMMRTrainer(precomputed_phi=False, freeze_phi=False): the phis' gradient, the temporal model, the trunk's Adam step,
determinism, the checkpoint and the uint8-frame path."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope='module')
def golden_weights():
    from human_dynamics_b200 import synthetic
    return synthetic.make_synthetic_weights(seed=1)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


# ------------------------------------------------------------------------------------------------------------------------------------
# hd_conv_wgrad
# ------------------------------------------------------------------------------------------------------------------------------------
def _wgrad(x, geom, pre, dy, Cout, bias):
    from human_dynamics_b200._lib import lib, check
    n, H, W, Cin, Ho, Wo, KH, KW, s, pt, pl = geom
    dw = torch.empty((KH * KW * Cin, Cout), device='cuda')
    db = torch.empty(Cout, device='cuda') if bias else None
    wsb = lib.hd_conv_wgrad_workspace_bytes(n * Ho * Wo, KH * KW * Cin, Cout, int(bias))
    ws = torch.empty(max(16, wsb), dtype=torch.uint8, device='cuda')
    check(lib.hd_conv_wgrad(_vp(x), Cin, n, H, W, Cin, Ho, Wo, KH, KW, s, pt, pl, _vp(pre[0]) if pre else None,
                            _vp(pre[1]) if pre else None, _vp(dy), Cout, Cout, _vp(dw), _vp(db), _vp(ws), ws.numel(), _st()), 'hd_conv_wgrad')
    return dw, db


def _wgrad_ref(x, geom, pre, dy):
    n, H, W, Cin, Ho, Wo, KH, KW, s, pt, pl = geom
    a = x.astype(np.float64)
    if pre is not None:
        a = np.maximum(x.astype(np.float64) * pre[0].astype(np.float64) + pre[1].astype(np.float64), 0)
    ap = np.zeros((n, H + KH + s * Ho, W + KW + s * Wo, Cin))
    ap[:, pt:pt + H, pl:pl + W] = a
    d = dy.astype(np.float64)
    out = np.zeros((KH, KW, Cin, dy.shape[-1]))
    for ky in range(KH):
        for kx in range(KW):
            patch = ap[:, ky:ky + s * (Ho - 1) + 1:s, kx:kx + s * (Wo - 1) + 1:s]
            out[ky, kx] = np.einsum('nyxc,nyxo->co', patch, d)
    return out.reshape(-1, dy.shape[-1]), d.sum((0, 1, 2))


@pytest.mark.parametrize('n,H,Cin,Cout,K,s,pad,pre,bias', [
    (3, 28, 64, 256, 1, 1, 0, True, True),          # 1x1 (shortcut / conv3 class), bias row
    (1, 14, 256, 64, 1, 1, 0, True, False),         # n = 1
    (2, 29, 64, 64, 3, 1, 1, True, False),          # SAME 3x3 stride 1, ragged pixel count
    (3, 28, 128, 128, 3, 2, 1, True, False),        # conv2d_same 3x3 stride 2
    (1, 15, 64, 64, 3, 2, 1, False, True),          # odd size, no prologue
    (2, 64, 3, 64, 7, 2, 3, False, True),           # root conv1: 7x7 stride 2 over 3 channels
    (3, 63, 3, 64, 7, 2, 3, False, True),           # conv1, three chunks, the last ragged
    (3, 29, 64, 64, 3, 1, 1, True, True),           # SAME 3x3, two chunks, ragged
    (3, 61, 64, 64, 3, 2, 1, True, False),          # conv2d_same 3x3 stride 2, two chunks, ragged
    (5, 7, 2048, 512, 1, 1, 0, True, False)])       # block 4 shape
def test_wgrad_against_float64(n, H, Cin, Cout, K, s, pad, pre, bias):
    rng = np.random.RandomState(n * 100 + H + Cin)
    Ho = (H + 2 * pad - K) // s + 1
    geom = (n, H, H, Cin, Ho, Ho, K, K, s, pad, pad)
    x = rng.normal(0.3, 1, (n, H, H, Cin)).astype(np.float32)
    dy = (rng.normal(0, 1, (n, Ho, Ho, Cout)) * 1e-3).astype(np.float32)
    pv = (rng.uniform(0.5, 1.5, Cin).astype(np.float32), rng.normal(0, 0.5, Cin).astype(np.float32)) if pre else None
    pt = tuple(torch.from_numpy(v).cuda() for v in pv) if pre else None
    dw, db = _wgrad(torch.from_numpy(x).cuda(), geom, pt, torch.from_numpy(dy).cuda(), Cout, bias)
    rw, rb = _wgrad_ref(x, geom, pv, dy)
    assert _rel(dw.cpu().numpy(), rw) < 2e-6
    if bias:
        assert _rel(db.cpu().numpy(), rb) < 1e-6
    dw2, db2 = _wgrad(torch.from_numpy(x).cuda(), geom, pt, torch.from_numpy(dy).cuda(), Cout, bias)
    assert torch.equal(dw, dw2) and (not bias or torch.equal(db, db2))


# ------------------------------------------------------------------------------------------------------------------------------------
# hd_bn_relu_backward
# ------------------------------------------------------------------------------------------------------------------------------------
def _bn_stats(x, rows, Cc, gamma, beta):
    from human_dynamics_b200._lib import lib, check
    out = [torch.empty(Cc, device='cuda') for _ in range(4)]
    ws = torch.empty(max(16, lib.hd_bn_stats_workspace_bytes(rows, Cc)), dtype=torch.uint8, device='cuda')
    check(lib.hd_bn_batch_stats(_vp(x), rows, Cc, Cc, _vp(gamma), _vp(beta), 1e-5, *[_vp(t) for t in out], None, None, 0.997, _vp(ws),
                                ws.numel(), _st()), 'hd_bn_batch_stats')
    return out


@pytest.mark.parametrize('frames,H,Cc,mean,group,stride', [
    (4, 14, 64, 0., 1, 0), (3, 8, 256, 1e3, 1, 1), (2, 7, 2048, 0., 49, 0), (5, 9, 512, 1e3, 1, 2), (1, 3, 2048, 1e3, 1, 2),
    (160, 7, 2048, 0.5, 49, 0)])
def test_bn_relu_backward_against_float64(frames, H, Cc, mean, group, stride):
    from human_dynamics_b200._lib import lib, check
    rng = np.random.RandomState(frames + Cc + H)
    rows = frames * H * H
    x = (rng.normal(mean, 1, (rows, Cc)) + rng.normal(0, 0.2, Cc)).astype(np.float32)
    gamma = rng.uniform(0.5, 1.5, Cc).astype(np.float32)
    beta = rng.normal(0, 0.5, Cc).astype(np.float32)
    dz = rng.normal(0, 1, (rows // group, Cc)).astype(np.float32)
    Hs = (H + stride - 1) // max(stride, 1)
    addend = rng.normal(0, 1, (frames, Hs, Hs, Cc) if stride > 1 else (rows, Cc)).astype(np.float32) if stride else None
    xt, gt, bt = (torch.from_numpy(v).cuda() for v in (x, gamma, beta))
    sc, sh, m, v = _bn_stats(xt, rows, Cc, gt, bt)
    dx = torch.empty((rows, Cc), device='cuda')
    dg, dbeta = torch.empty(Cc, device='cuda'), torch.empty(Cc, device='cuda')
    ws = torch.empty(lib.hd_bn_relu_backward_workspace_bytes(rows, Cc), dtype=torch.uint8, device='cuda')
    at = torch.from_numpy(addend).cuda() if addend is not None else None
    dzt = torch.from_numpy(dz).cuda()

    def run(out):
        check(lib.hd_bn_relu_backward(_vp(xt), _vp(dzt), group, rows, Cc, _vp(sc), _vp(sh), _vp(v), _vp(gt), 1e-5, _vp(at), H, H, stride,
                                      _vp(out), _vp(dg), _vp(dbeta), _vp(ws), ws.numel(), _st()), 'hd_bn_relu_backward')
    run(dx)
    # float64: the mask is the GPU forward's (fma(x, scale, shift) > 0); everything else exact
    z = x.astype(np.float64) * sc.cpu().numpy().astype(np.float64) + sh.cpu().numpy().astype(np.float64)
    g = np.repeat(dz.astype(np.float64), group, 0) / group * (z > 0)
    xd = x.astype(np.float64)
    mu, var = xd.mean(0), xd.var(0)
    rstd = 1 / np.sqrt(var + 1e-5)
    xh = (xd - mu) * rstd
    want = gamma * rstd * (g - g.mean(0) - xh * (g * xh).mean(0))
    if stride == 1:
        want = want + addend
    elif stride > 1:
        w4 = want.reshape(frames, H, H, Cc)
        w4[:, ::stride, ::stride] += addend
    assert _rel(dbeta.cpu().numpy(), g.sum(0)) < 1e-6
    assert _rel(dg.cpu().numpy(), (g * xh).sum(0)) < 1e-5
    assert _rel(dx.cpu().numpy(), want) < 1e-5
    dx2 = torch.empty_like(dx)
    run(dx2)
    assert torch.equal(dx, dx2)


# ------------------------------------------------------------------------------------------------------------------------------------
# pool1 backward, the strided data gradient, the 2-D backward-data pack
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,W', [(112, 112), (15, 9), (8, 8)])
def test_maxpool_backward_against_float64(H, W):
    from human_dynamics_b200._lib import lib, check
    from oracle.nets_train_grad_ref import max_pool_3x3_s2
    rng = np.random.RandomState(H + W)
    n, Cc = 2, 64
    x = rng.randint(0, 5, (n, H, W, Cc)).astype(np.float32)         # small integers: many exact ties inside the windows
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    dout = rng.normal(0, 1, (n, Ho, Wo, Cc)).astype(np.float32)
    din = torch.empty((n, H, W, Cc), device='cuda')
    xg, dg = torch.from_numpy(x).cuda(), torch.from_numpy(dout).cuda()
    check(lib.hd_maxpool3x3s2_same_backward(_vp(xg), _vp(dg), _vp(din), n, H, W, Cc, _st()), 'hd_maxpool3x3s2_same_backward')
    xt = torch.from_numpy(x.astype(np.float64)).requires_grad_()
    y = max_pool_3x3_s2(xt)                                          # first maximum in scan order (torch.argmax)
    want, = torch.autograd.grad(y, xt, torch.from_numpy(dout.astype(np.float64)))
    # an input chosen by two windows sums them in fp32 here, in fp64 in the reference
    np.testing.assert_allclose(din.cpu().numpy(), want.numpy(), rtol=1e-6, atol=1e-6)
    assert np.array_equal(din.cpu().numpy() != 0, want.numpy() != 0)


@pytest.mark.parametrize('H,Cin,Cout,s', [(14, 64, 64, 2), (15, 128, 64, 2), (9, 64, 128, 1), (28, 256, 256, 1)])
def test_conv3x3_data_gradient_against_float64(H, Cin, Cout, s):
    """dX of a conv2d_same 3x3 through the 2-D backward-data pack (tap flip of the flattened (ky, kx)), stride 2 via zero insertion."""
    from human_dynamics_b200._lib import lib, check
    from human_dynamics_b200.nets import PackedConv, _dgrad_op
    from human_dynamics_b200.trainable import BackwardDataPack
    from oracle.nets_ref import conv2d_same
    rng = np.random.RandomState(H + Cin + s)
    n = 3
    Ho = (H - 1) // s + 1
    w = (rng.normal(0, 1, (3, 3, Cin, Cout)) / np.sqrt(9 * Cin)).astype(np.float32)
    dy = rng.normal(0, 1, (n, Ho, Ho, Cout)).astype(np.float32)
    wt = torch.from_numpy(w).cuda()
    conv = PackedConv(wt, 'cuda', stride=s, pad=(1, 1), tc='auto')
    conv.bwd = BackwardDataPack(wt, 9, Cin, Cout)
    conv.bwd.repack(_st())
    dyt = torch.from_numpy(dy).cuda()
    z = torch.empty((n, H, H, Cout), device='cuda')
    out = torch.empty((n, H, H, Cin), device='cuda')
    src = dyt
    if s > 1:
        check(lib.hd_zero_insert(_vp(dyt), _vp(z), n, Ho, Ho, Cout, s, H, H, _st()), 'hd_zero_insert')
        src = z
    _dgrad_op(conv, src, n, H, H, 3, out).run(_st())
    xt = torch.zeros((n, H, H, Cin), dtype=torch.float64, requires_grad=True)
    y = conv2d_same(xt, torch.from_numpy(w.astype(np.float64)), s)
    want, = torch.autograd.grad(y, xt, torch.from_numpy(dy.astype(np.float64)))
    assert _rel(out.cpu().numpy(), want.numpy()) < 2e-6


# ------------------------------------------------------------------------------------------------------------------------------------
# the whole trunk against the float64 oracle
# ------------------------------------------------------------------------------------------------------------------------------------
# per-tensor relative L2; measured on an H100 80GB HBM3: worst 7.2e-6 (n = 2), 6.9e-6 (16), 1.2e-5 (160) at 224², 8.3e-6 at 64²
TRUNK_BAR = 5e-5


def _gpu_choices(plan, n):
    """The GPU forward's ReLU masks (fma(x, scale, shift) > 0 on the kept raw maps) and pool1's window choice (first maximum of the kept
    fp32 conv1 output), keyed like oracle/nets_train_grad_ref's sites."""
    from oracle.nets_train_grad_ref import max_pool_3x3_s2
    masks = {}
    for op, s in zip(plan.stats, plan.bn.scopes):
        x = op.x[:op.rows * op.C].double().view(n, -1, op.C)
        z = x * op.scale.double() + op.shift.double()
        hw = z.shape[1]
        h = int(round(hw ** 0.5))
        masks[s] = (z > 0).view(n, h, h, op.C)
    rec = {}
    max_pool_3x3_s2(plan.root_buf.view(n, plan.H1, plan.H1, 64).double(), record=rec)
    masks['pool1'] = rec['pool1']
    return masks


def _trunk_case(weights, n, size, seed, check_repeat=False):
    from human_dynamics_b200 import synthetic, _lib
    from human_dynamics_b200.trunk import TrainableResNet
    from oracle import nets_train_grad_ref as G
    img = synthetic.make_images(n, seed=seed, size=size)
    dphi = np.random.RandomState(seed).normal(0, 1, (n, 2048)).astype(np.float32)
    net = TrainableResNet(weights)
    images = torch.from_numpy(img).cuda()
    phis, plan = net(images)
    dphi_t = torch.from_numpy(dphi).cuda()
    g = torch.autograd.grad(phis, list(net.parameters()), dphi_t)
    got = {nm: t for nm, t in zip([k for k, _ in net._params.items()], g)}
    masks = _gpu_choices(plan, n)
    rec = {}
    ref, rphi = G.trunk_gradients(img, weights, dphi, masks=masks, record=rec, device='cuda')
    flips = sum(int(((rec[s] > 0) != masks[s]).sum()) for s in plan.bn.scopes)
    near = all(bool((rec[s][(rec[s] > 0) != masks[s]].abs() < 1e-3).all()) for s in plan.bn.scopes)
    assert near, 'a ReLU site where the GPU and the oracle disagree is not a near tie'
    # Every bias feeds only batch-normalised paths (a per-channel constant reaches the next batch norms through the identity shortcuts and
    # pool1, and batch norm is shift-invariant), so its exact gradient is 0 and both sides hold rounding noise: a bias is measured
    # against the weight gradient of its own layer.
    def err(k):
        g, r = got[k].cpu().numpy().astype(np.float64), ref[k].cpu().numpy()
        if k.endswith('/biases'):
            return float(np.linalg.norm(g - r) / np.linalg.norm(ref[k[:-len('biases')] + 'weights'].cpu().numpy()))
        return _rel(g, r)
    errs = {k: err(k) for k in ref}
    worst = max(v for k, v in errs.items() if not k.endswith('/biases'))
    print('n=%d size=%d: worst per-tensor relative L2 %.3e (biases against their weights %.3e), %d ReLU near-ties taken from the GPU'
          % (n, size, worst, max(v for k, v in errs.items() if k.endswith('/biases')), flips))
    for k, v in errs.items():
        assert v < TRUNK_BAR, (k, v)
    assert _rel(phis.detach().cpu().numpy(), rphi.cpu().numpy()) < 1e-4
    if check_repeat:
        _lib.lib.hd_launch_count_reset()
        phis2, plan2 = net(images)
        torch.cuda.synchronize()
        assert _lib.lib.hd_launch_count() == plan.num_launches and plan2 is plan and torch.equal(phis, phis2)
        _lib.lib.hd_launch_count_reset()
        g2 = torch.autograd.grad(phis2, list(net.parameters()), dphi_t)
        torch.cuda.synchronize()
        assert _lib.lib.hd_launch_count() == plan.num_backward_launches
        assert all(torch.equal(a, b) for a, b in zip(g, g2))
    return worst


@pytest.mark.parametrize('n,size', [(2, 224), (16, 224), (160, 224), (4, 64)])
def test_trunk_gradients_against_oracle(golden_weights, n, size):
    _trunk_case(golden_weights, n, size, 300 + n + size, check_repeat=(n == 16))


def test_keep_plan_phis_equal_the_frozen_plan(golden_weights):
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.nets import PackedResNet, ResNetBatchNorm, ResNetTrainPlan
    n = 6
    img = torch.from_numpy(synthetic.make_images(n, seed=4, size=224)).cuda()
    packed = PackedResNet(golden_weights, 'cuda', tc='auto')
    bn = ResNetBatchNorm(golden_weights, 'cuda')
    a, b = torch.empty((n, 2048), device='cuda'), torch.empty((n, 2048), device='cuda')
    ResNetTrainPlan(packed, bn, n, 224).run(img, a)
    ResNetTrainPlan(packed, bn, n, 224, keep=True).run(img, b)
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------------------------------
# HMMRTrainer with freeze_phi=False
# ------------------------------------------------------------------------------------------------------------------------------------
def _batch(B, T, S, seed):
    from human_dynamics_b200 import synthetic
    rng = np.random.RandomState(seed)
    return {'labels': torch.from_numpy(np.concatenate([rng.uniform(-1, 1, (B, T, 25, 2)), np.ones((B, T, 25, 1))], -1).astype(np.float32)).cuda(),
            'poses': torch.from_numpy(rng.normal(0, 0.3, (B, T, 72)).astype(np.float32)).cuda(),
            'shape': torch.from_numpy(rng.normal(0, 0.5, (B, 10)).astype(np.float32)).cuda(),
            'gt3ds': torch.from_numpy(rng.normal(0, 0.3, (B, T, 14, 3)).astype(np.float32)).cuda(),
            'has_3d': torch.ones((B, 2), device='cuda'),
            'images': torch.from_numpy(synthetic.make_images(B * T, seed=seed, size=S).reshape(B, T, S, S, 3)).cuda()}


def _mocap(n, seed):
    from human_dynamics_b200.smpl import batch_rodrigues
    aa = torch.from_numpy(np.random.RandomState(seed).normal(0, 0.3, size=(n * 24, 3)).astype(np.float32)).cuda()
    return batch_rodrigues(aa).reshape(n, 216)


def test_trainer_unfrozen_trunk(weights, smpl_model):
    from human_dynamics_b200.engine import HMMREngine, load_weights
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from oracle import nets_ref
    from src.tf_smpl.batch_smpl import SMPL
    smpl = SMPL(smpl_model)
    B, T, S = 2, 6, 64
    batch = _batch(B, T, S, 5)
    cfg = TrainConfig(precomputed_phi=False, freeze_phi=False, do_hallucinate=True, do_hallucinate_preds=True)
    tr = HMMRTrainer(cfg, weights, smpl)
    mocap = _mocap(tr.n_fake(B, T), 6)
    net = tr.trunk.net
    assert len(tr.e_params) == len(list(tr.model.parameters())) + 53 + 21 + 2 * 49
    # chaining: the dphi the trunk receives == d e_loss / d phis of a phi-input trainer fed those phis, bit for bit
    seen = {}
    plan = net.plan(B * T, S)
    orig = plan.backward

    def spy(dphi, images, stream=None):
        seen['dphi'] = dphi.clone()
        out = orig(dphi, images, stream)
        seen['grads'] = {k: v.clone() for k, v in out.items()}
        return out
    plan.backward = spy
    with torch.no_grad():
        phis, _ = net(batch['images'].reshape(B * T, S, S, 3))
    ref_tr = HMMRTrainer(TrainConfig(do_hallucinate=True, do_hallucinate_preds=True), weights, smpl)
    pb = {k: v for k, v in batch.items() if k != 'images'}
    pb['phis'] = phis.view(B, T, 2048).clone().requires_grad_()
    _, e_ref, _ = ref_tr.forward(pb, mocap)
    dphi_ref, = torch.autograd.grad(e_ref, pb['phis'])
    # the frozen image trainer: the temporal model and D_pose must end bit-identical
    fz = HMMRTrainer(TrainConfig(precomputed_phi=False, do_hallucinate=True, do_hallucinate_preds=True), weights, smpl)
    before = {n: p.detach().clone() for n, p in net._params.items()}
    a, b = tr.step(batch, mocap), fz.step(batch, mocap)
    assert torch.equal(seen['dphi'], dphi_ref.reshape(B * T, 2048))
    for k in b:
        assert torch.equal(a[k], b[k]), k
    for p, q in zip(tr.model.parameters(), fz.model.parameters()):
        assert torch.equal(p, q)
    for p, q in zip(tr.disc.parameters(), fz.disc.parameters()):
        assert torch.equal(p, q)
    # the trunk moved by exactly torch Adam's step from the gradients the backward returned
    ps = [torch.nn.Parameter(before[n].clone()) for n in net.names]
    opt = torch.optim.Adam(ps, cfg.e_lr)
    for p, n in zip(ps, net.names):
        p.grad = net.gradient_of(n, seen['grads']).clone()
    opt.step()
    for p, n in zip(ps, net.names):
        assert torch.equal(p.detach(), net.param(n).detach()), n
    assert not torch.equal(before['resnet_v2_50/block2/unit_1/bottleneck_v2/conv2/weights'],
                           net.param('resnet_v2_50/block2/unit_1/bottleneck_v2/conv2/weights'))
    # determinism: the same step from the same state, twice
    outs = []
    for _ in range(2):
        t2 = HMMRTrainer(cfg, weights, smpl)
        o = t2.step(batch, mocap)
        outs.append((o, [p.detach().clone() for p in t2.e_params]))
    for k in outs[0][0]:
        assert torch.equal(outs[0][0][k], outs[1][0][k]), k
    assert all(torch.equal(x, y) for x, y in zip(outs[0][1], outs[1][1]))
    # a second step repacks the changed weights; the checkpoint carries the trained trunk
    tr.step(batch, mocap)
    img = batch['images'].reshape(B * T, S, S, 3)
    with tempfile.TemporaryDirectory() as d:
        prefix = tr.save_checkpoint(os.path.join(d, 'model.ckpt-2'))
        w2 = load_weights(prefix)
    for n in net.names:
        assert np.array_equal(w2[n].reshape(-1), net.param(n).detach().cpu().numpy().reshape(-1)), n
    eng = HMMREngine(w2, smpl_model)
    phi_inf = eng.encode_images(img).cpu().numpy()
    ref = nets_ref.encoder_resnet(img.cpu().numpy(), w2, torch.float64).numpy()
    assert np.abs(phi_inf - ref).max() / np.abs(ref).max() < 1e-4


def test_trainer_unfrozen_end_to_end_from_uint8_frames(weights, smpl_model):
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
    outs = []
    for _ in range(2):
        r = TubeAugmentor(img_size=S, seed=7)(frames, lab, cen, pose, g3, tube_lengths=[T] * B)
        batch = {'images': r['images'].view(B, T, S, S, 3), 'labels': r['labels'].transpose(1, 2).reshape(B, T, 25, 3).contiguous(),
                 'poses': r['poses'].reshape(B, T, 72), 'shape': torch.zeros((B, 10), device='cuda'),
                 'gt3ds': r['gt3ds'].reshape(B, T, 14, 3), 'has_3d': torch.ones((B, 2), device='cuda')}
        tr = HMMRTrainer(TrainConfig(precomputed_phi=False, freeze_phi=False), weights, smpl)
        out = tr.step(batch, _mocap(tr.n_fake(B, T), 3))
        assert all(v.shape == () and torch.isfinite(v) for v in out.values())
        outs.append((out, [p.detach().clone() for p in tr.trunk.net.parameters()]))
    for k in outs[0][0]:
        assert torch.equal(outs[0][0][k], outs[1][0][k]), k
    assert all(torch.equal(x, y) for x, y in zip(outs[0][1], outs[1][1]))


def test_stale_graph_refuses_backward(weights):
    from human_dynamics_b200 import synthetic, _lib
    from human_dynamics_b200.trunk import TrainableResNet
    net = TrainableResNet(weights)
    img = torch.from_numpy(synthetic.make_images(2, seed=1, size=64)).cuda()
    p1, _ = net(img)
    net(img)
    with pytest.raises(_lib.HDError, match='another forward'):
        torch.autograd.grad(p1.sum(), list(net.parameters()))
    p2, _ = net(img)
    with torch.no_grad():
        net.param('resnet_v2_50/postnorm/gamma').mul_(1.5)
    with pytest.raises(_lib.HDError, match='modified in place'):
        torch.autograd.grad(p2.sum(), list(net.parameters()))
