"""GPU: the trainable temporal model (human_dynamics_b200/trainable.py, csrc/net_grad.cu + the 3xTF32 GEMM) -- forward bit-identical
to HMMREngine, gradients against the float64 oracle (oracle/nets_grad_ref.py, pinned to finite differences in
test_temporal_grad_cpu.py), device packing, determinism, a fine-tuning loop against the oracle, checkpoint round trip and errors."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F64 = torch.float64
REL = 1e-4
GUARD = 2.5e-5      # the float32 oracle must agree with the float64 one this well, else the case is too ill-conditioned to judge
MARGIN = 1e-5       # |pre-activation| below this: the GPU's ReLU sign is taken (the two forwards may legitimately disagree there)
KEYS = (-5, 5)


def rel_err(a, b):
    a, b = a.detach().double(), b.detach().double().to(a.device)
    return float((a - b).abs().max() / max(b.abs().max().item(), 1e-300))


@pytest.fixture(scope='module')
def engine(weights, smpl_model):
    from human_dynamics_b200.engine import HMMREngine
    return HMMREngine(weights, smpl_model)


@pytest.fixture(scope='module')
def model(weights):
    from human_dynamics_b200.trainable import TemporalModel
    return TemporalModel(weights)


def _phi(B, T, seed):
    rng = np.random.RandomState(seed)
    return torch.from_numpy(rng.normal(0, 1, size=(B, T, 2048)).astype(np.float32)).cuda()


@pytest.mark.parametrize('BT', [(2, 20), (32, 20), (2, 25)])      # T = 25: T*64 > 1280, the GroupNorm-statistics + prologue branch
def test_forward_bit_identical_to_engine(engine, model, BT):
    B, T = BT
    N = B * T
    phi = _phi(B, T, B).requires_grad_()
    f = model.temporal_encode(phi)
    assert f.requires_grad
    assert torch.equal(f.detach(), engine.temporal_encode(phi.detach()))
    th, dl = model.regress(f.reshape(N, 2048))
    th_e, dl_e = engine.regress(f.detach().reshape(N, 2048).contiguous())
    assert torch.equal(th.detach(), th_e)
    for k in KEYS:
        assert torch.equal(dl[k].detach(), dl_e[k])
    h = model.hallucinate(phi)
    assert torch.equal(h.detach(), engine.hallucinate(phi.detach()))
    with torch.no_grad():
        assert torch.equal(model.temporal_encode(phi), f.detach())


def _oracle(weights, names, phi, ups, masks, dtype):
    from oracle import nets_grad_ref as g
    L = g.leaves(weights, names, dtype, 'cuda')
    B, T = phi.shape[:2]
    N = B * T
    x = phi.detach().to(dtype).requires_grad_()
    f = g.fmovie(x, g.fmovie_blocks(L), masks)
    start = L['mean_param'].reshape(1, 85).expand(N, 85)
    th, dl = g.call_hmr_ief(f.reshape(N, 2048), start, {dt: g.ief_params(L, dt) for dt in (0,) + KEYS}, KEYS, masks)
    hal = g.fc2_res(x.reshape(N, 2048), tuple(L['fc2_res/fc%d/%s' % (i, k)] for i in (1, 2, 3) for k in ('weights', 'biases')), masks)
    loss = (th * ups[0].to(dtype)).sum() + sum((dl[k] * ups[1 + i].to(dtype)).sum() for i, k in enumerate(KEYS)) + \
        (hal * ups[3].to(dtype).reshape(N, 2048)).sum()
    gr =torch.autograd.grad(loss, [x] + [L[n] for n in names])
    return dict(zip(['phi'] + names, gr))


def _masks(model, phi, feats, record):
    """Oracle masks: the float64 sign everywhere except near ties, where the GPU's sign is taken.  Returns (masks, overridden, sites)."""
    gpu = model.relu_masks(phi=phi, feats=feats, hal=phi.reshape(-1, 2048))
    masks, over, sites = {}, 0, 0
    for name, pre in record.items():
        gm = gpu[name].to(pre.device).reshape(pre.shape)
        near = pre.abs() < MARGIN
        masks[name] = torch.where(near, gm, pre > 0)
        over += int((near & (gm != (pre > 0))).sum())
        sites += pre.numel()
    return masks, over, sites


@pytest.mark.parametrize('scale', [1.0, 1e-8, 1e8])
@pytest.mark.parametrize('BT', [(1, 1), (2, 20), (3, 7), (32, 20), (2, 25)])
def test_grads_match_oracle(weights, model, BT, scale):
    from human_dynamics_b200.trainable import trainable_names
    B, T = BT
    N = B * T
    names = trainable_names(weights)
    rng = np.random.RandomState(B * 100 + T)
    ups = [torch.from_numpy(rng.normal(0, scale, size=s).astype(np.float32)).cuda() for s in ((N, 85), (N, 85), (N, 85), (B, T, 2048))]
    phi = _phi(B, T, B + T).requires_grad_()
    model.zero_grad(set_to_none=True)
    f = model.temporal_encode(phi)
    th, dl = model.regress(f.reshape(N, 2048))
    hal = model.hallucinate(phi)
    loss = (th * ups[0]).sum() + sum((dl[k] * ups[1 + i]).sum() for i, k in enumerate(KEYS)) + (hal * ups[3]).sum()
    loss.backward()
    got = {'phi': phi.grad}
    got.update({n: model.param(n).grad for n in names})
    record = {}
    with torch.no_grad():
        from oracle import nets_grad_ref as g
        L = g.leaves(weights, names, F64, 'cuda')
        x = phi.detach().double()
        fo = g.fmovie(x, g.fmovie_blocks(L), None, record)
        g.call_hmr_ief(fo.reshape(N, 2048), L['mean_param'].reshape(1, 85).expand(N, 85), {dt: g.ief_params(L, dt) for dt in (0,) + KEYS},
                       KEYS, None, record)
        g.fc2_res(x.reshape(N, 2048), tuple(L['fc2_res/fc%d/%s' % (i, k)] for i in (1, 2, 3) for k in ('weights', 'biases')), None, record)
    masks, over, sites = _masks(model, phi.detach(), f.detach().reshape(N, 2048), record)
    print('BT=%s scale=%g: %d of %d ReLU sites overridden' % (BT, scale, over, sites))
    assert over <= 1e-4 * sites
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        r64 = _oracle(weights, names, phi, ups, masks, F64)
        r32 = _oracle(weights, names, phi, ups, masks, torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    # Every tensor is judged.  Where even the float32 oracle is off by GUARD or more (an ill-conditioned case), the bar is 10x the float32
    # oracle's own error instead of REL; those tensors are listed, and they may not be more than a quarter of all.
    worst, relaxed = [], []
    for n in ['phi'] + names:
        assert got[n] is not None, n
        assert torch.isfinite(got[n]).all(), n
        e32, e = rel_err(r32[n], r64[n]), rel_err(got[n], r64[n])
        bar = REL
        if e32 >= GUARD:
            bar = max(REL, 10 * e32)
            relaxed.append((n, e32, e))
        worst.append((e, n))
        assert e < bar, (n, e, e32)
    print('worst: %s; judged against 10x the float32 oracle error: %s' % (max(worst), relaxed))
    assert len(relaxed) <= len(names) // 4, relaxed


def test_device_packing_of_engine_and_model_equals_host_packing(engine, model, weights):
    """Every tensor-core pack of an engine (ResNet units, the gather and the plane conv1, f_movie, the IEF heads, fc2_res, the SMPL blend
    and dc GEMMs), of the temporal model's forward, and a tc3 / tc1 TF32 pack, as hd_pack_weight writes them on the device, equal the
    numpy restatement (oracle/pack_ref.py) byte for byte."""
    from oracle import pack_ref
    from human_dynamics_b200.nets import RESNET_BLOCKS, PackedConv

    def same(hi, lo, w_nk, kind):
        rh, rl = pack_ref.split(w_nk, kind)
        bits = np.uint16 if kind == 'f16' else np.uint32
        assert np.array_equal(hi.cpu().numpy().view(bits), rh.view(bits)) and np.array_equal(lo.cpu().numpy().view(bits), rl.view(bits))

    layers = []                                            # (PackedConv, its TF HWIO source or None for its own fp32 copy, expected packing)
    p = 'resnet_v2_50'
    layers.append((engine.resnet.conv1, weights[p + '/conv1/weights'], 'f16'))
    assert engine.resnet.conv1.gather
    i = 0
    for b, (_, units, _) in enumerate(RESNET_BLOCKS, start=1):
        for u in range(1, units + 1):
            unit = engine.resnet.units[i]
            for k in ('shortcut', 'conv1', 'conv2', 'conv3'):
                if k in unit:
                    layers.append((unit[k], weights['%s/block%d/unit_%d/bottleneck_v2/%s/weights' % (p, b, u, k)], 'f16'))
            i += 1
    for i, blk in enumerate(engine.fmovie.blocks):
        for k in (1, 2):
            layers.append((blk['conv%d' % k], weights['AZ_FC_block2_conv%dblock_%d/weights' % (k, i)], 'f16'))
    for dt, head in [(0, engine.ief.main)] + sorted(engine.ief.deltas.items()):
        q = ('single_view_ief' if dt == 0 else 'single_view_ief_%s%d' % ('future' if dt > 0 else 'past', abs(dt))) + '/3D_module'
        layers += [(head.fc1_phi, weights[q + '/fc1/weights'][:2048], 'f16'), (head.fc2, weights[q + '/fc2/weights'], 'f16'),
                   (head.fc3, weights[q + '/fc3/weights'], 'f16')]
    for k in (1, 2, 3):
        layers.append((getattr(engine.hal, 'fc%d' % k), weights['fc2_res/fc%d/weights' % k], 'f16'))
    layers += [(engine.smpl.blend, None, 'f16'), (engine.smpl.grad_state()[2], None, 'tf32')]
    for tc in ('tc3', 'tc1'):
        layers.append((PackedConv(weights['single_view_ief/3D_module/fc2/weights'], torch.device('cuda'), tc=tc), None, 'tf32'))
    for blk in model.fmovie.blocks:
        layers += [(blk['conv1'], None, 'f16'), (blk['conv2'], None, 'f16')]
    for h in [model.ief.main] + list(model.ief.deltas.values()):
        layers += [(h.fc1_phi, None, 'f16'), (h.fc2, None, 'f16'), (h.fc3, None, 'f16')]
    layers += [(getattr(model.hal, 'fc%d' % k), None, 'f16') for k in (1, 2, 3)]
    assert len(layers) == 1 + 52 + 6 + 9 + 3 + 2 + 2 + 6 + 9 + 3
    torch.cuda.synchronize()
    for pc, src, kind in layers:
        assert pc.tc == kind
        w = pc.w_kn.cpu().numpy().reshape(pc.KH, pc.KW, pc.Cin, pc.Cout)
        if src is not None:
            assert np.array_equal(w, np.asarray(src, np.float32).reshape(w.shape))
        same(pc.w_nk_hi, pc.w_nk_lo, pack_ref.nk_layout(w, pc.gather), kind)
    planes = engine.resnet.conv1_planes
    same(planes.w_nk_hi, planes.w_nk_lo, pack_ref.conv1_planes_layout(weights[p + '/conv1/weights']), 'f16')


def test_step_then_forward_equals_fresh_model(weights):
    from human_dynamics_b200.trainable import TemporalModel
    m = TemporalModel(weights)
    B, T = 2, 20
    phi = _phi(B, T, 9)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    th, dl = m.regress(m.temporal_encode(phi).reshape(B * T, 2048))
    (th.square().mean() + sum(v.square().mean() for v in dl.values()) + m.hallucinate(phi).square().mean()).backward()
    opt.step()
    assert m.sync_packs() > 0
    fresh = TemporalModel(m.tf_variables())
    with torch.no_grad():
        f1, f2 = m.temporal_encode(phi), fresh.temporal_encode(phi)
        assert torch.equal(f1, f2)
        a, b = m.regress(f1.reshape(B * T, 2048)), fresh.regress(f2.reshape(B * T, 2048))
        assert torch.equal(a[0], b[0]) and all(torch.equal(a[1][k], b[1][k]) for k in KEYS)
        assert torch.equal(m.hallucinate(phi), fresh.hallucinate(phi))
    assert m.sync_packs() == 0


def _dphi(model, phi):
    B, T = phi.shape[:2]
    phi = phi.clone().requires_grad_()
    model.zero_grad(set_to_none=True)
    th, dl = model.regress(model.temporal_encode(phi).reshape(B * T, 2048))
    w = torch.arange(85, dtype=torch.float32, device='cuda') / 85 - 0.5
    ((th * w).sum() + sum((v * w).sum() for v in dl.values()) + model.hallucinate(phi).sum()).backward()
    return phi.grad, {n: p.grad.clone() for n, p in model._params.items()}


def test_determinism_permutation_and_batch_split(model):
    phi = _phi(4, 20, 21)
    g1, w1 = _dphi(model, phi)
    g2, w2 = _dphi(model, phi)
    assert torch.equal(g1, g2) and all(torch.equal(w1[n], w2[n]) for n in w1)
    perm = torch.tensor([2, 0, 3, 1], device='cuda')
    gp, _ = _dphi(model, phi[perm])
    assert torch.equal(gp, g1[perm])
    ga, _ = _dphi(model, phi[:2])
    gb, _ = _dphi(model, phi[2:])
    assert torch.equal(torch.cat([ga, gb]), g1)


@pytest.mark.parametrize('pred_mode', ['pred', 'hal'])
def test_finetune_tracks_oracle(weights, smpl_model, pred_mode):
    """10 SGD steps on the keypoint reprojection loss of the main and delta heads (L1, as the reference's keypoint loss), through
    predict_from_features (f_movie, or fc2_res with pred_mode 'hal') and the SMPL backward, against the same loop on the float64 oracle
    (CPU).  Asserted: the loss falls and tracks the oracle's to 1e-4 at every step.  The parameter updates p - p0 are compared with the
    oracle's and reported (see the open finding below)."""
    from human_dynamics_b200.config import HMMRConfig
    from human_dynamics_b200.trainable import TemporalModel, trainable_names
    from oracle import nets_grad_ref as g
    from oracle.smpl_grad_ref import SMPLGradRef, batch_orth_proj_idrot
    from src.tf_smpl.batch_smpl import SMPL
    B, T, steps, lr = 2, 20, 10, 1e-4
    N = B * T
    model = TemporalModel(weights, HMMRConfig(pred_mode=pred_mode))
    smpl = SMPL(smpl_model)
    phi = _phi(B, T, 33)
    rng = np.random.RandomState(3)
    K = smpl.consts.num_kps
    gt = torch.from_numpy(rng.uniform(-0.8, 0.8, size=(B, T, K, 2)).astype(np.float32))
    gtd = torch.from_numpy(rng.uniform(-0.8, 0.8, size=(B, T, len(KEYS), K, 2)).astype(np.float32))
    opt = torch.optim.SGD(model.parameters(), lr=lr)
    names = trainable_names(weights)
    L = g.leaves(weights, names, F64)
    p0 = {n: model.param(n).detach().clone() for n in names}
    opt_o = torch.optim.SGD([L[n] for n in names], lr=lr)
    ref_smpl = SMPLGradRef(smpl_model)

    def oracle_loss(L, dtype, sm):
        x = phi.detach().cpu().to(dtype)
        if pred_mode == 'pred':
            f = g.fmovie(x, g.fmovie_blocks(L))
        else:
            f = g.fc2_res(x.reshape(N, 2048), tuple(L['fc2_res/fc%d/%s' % (i, k)] for i in (1, 2, 3) for k in ('weights', 'biases')))
        th, dl = g.call_hmr_ief(f.reshape(N, 2048), L['mean_param'].reshape(1, 85).expand(N, 85),
                                {dt: g.ief_params(L, dt) for dt in (0,) + KEYS}, KEYS)

        def kps(om, cam):
            _, j, _ = sm(om[:, 75:85], om[:, 3:75], get_skin=True)
            return batch_orth_proj_idrot(j, cam)
        k0 = kps(th, th[:, :3]).reshape(B, T, K, 2)
        kd = torch.stack([kps(dl[k], th[:, :3]).reshape(B, T, K, 2) for k in KEYS], 2)
        return (k0 - gt.to(dtype)).abs().mean() + (kd - gtd.to(dtype)).abs().mean()
    # conditioning of the first update: the float32 oracle's error against the float64 one (the keypoint loss reaches the temporal
    # layers through SMPL, whose float32 evaluation alone moves small, cancelling sums such as a GroupNorm gamma's gradient)
    L32 = g.leaves(weights, names, torch.float32)
    gr32 = torch.autograd.grad(oracle_loss(L32, torch.float32, SMPLGradRef(smpl_model, dtype=torch.float32)), [L32[n] for n in names],
                               allow_unused=True)
    L64 = g.leaves(weights, names, F64)
    gr64 = torch.autograd.grad(oracle_loss(L64, F64, ref_smpl), [L64[n] for n in names], allow_unused=True)
    cond = {n: rel_err(a, b) for n, a, b in zip(names, gr32, gr64) if b is not None and b.abs().max() > 0}
    losses, losses_o = [], []
    for step in range(steps):
        out = model.predict_from_features(phi, smpl)
        loss = (out['kps'] - gt.cuda()).abs().mean() + (out['kps_delta'] - gtd.cuda()).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
        lo = oracle_loss(L, F64, ref_smpl)
        opt_o.zero_grad()
        lo.backward()
        opt_o.step()
        losses_o.append(lo.item())
        if step == 0:
            first = _deltas(model, L, p0, weights, names)
    print('loss gpu %s\nloss ref %s' % (losses, losses_o))
    assert losses[-1] < losses[0]
    for a, b in zip(losses, losses_o):
        assert abs(a - b) <= 1e-4 * abs(b)
    last = _deltas(model, L, p0, weights, names)
    print('update error after step 1: %s\nafter step %d: %s\nfloat32 oracle, first update: %s' %
          (max(first.values()), steps, max(last.values()), max(cond.values())))
    assert len(first) >= len(names) // 2 and set(first) == set(cond)
    # OPEN FINDING, reported and not asserted: on the H100 the first update of this loop differs from the float64 oracle's by up to
    # 7.8e-2 ('pred') / 1.1e-1 ('hal'), max-normalised, largest in the delta heads' fc1 / fc2 biases (and 5.6e-2 in f_movie's block-0 gn1
    # gamma), reproducibly, while the float32 oracle agrees with the float64 one to ~2e-6 and the same layers' gradients under random
    # upstream gradients agree to 1e-6 (test_grads_match_oracle).  The cause (the keypoint-loss / SMPL upstream of this loop or the delta
    # heads' backward under it) is not isolated yet; the loss tracking above is what is asserted.
    print('per-tensor update error after step 1: %s' % sorted(((v, n) for n, v in first.items()), reverse=True)[:5])


def _deltas(model, L, p0, weights, names):
    """{name: max|dp_gpu - dp_ref| / max|dp_ref|} over the parameters the loss moves (dp = p - p0); a layer the loss does not reach (f_movie
    in 'hal' mode, fc2_res in 'pred') must not move on either side."""
    out = {}
    for n in names:
        d_gpu = model.param(n).detach() - p0[n]
        d_ref = L[n].detach().reshape(d_gpu.shape) - torch.from_numpy(np.asarray(weights[n], np.float64)).reshape(d_gpu.shape)
        if d_ref.abs().max() == 0:
            assert d_gpu.abs().max() == 0, n
            continue
        out[n] = rel_err(d_gpu, d_ref)
    return out


def test_checkpoint_round_trip(weights, smpl_model, tmp_path):
    from human_dynamics_b200.engine import HMMREngine
    from human_dynamics_b200.trainable import TemporalModel
    from src.tf_smpl.batch_smpl import SMPL
    model = TemporalModel(weights)
    with torch.no_grad():
        for p in model.parameters():
            p.mul_(1.001)
    prefix = model.save_checkpoint(str(tmp_path / 'model.ckpt-10'))
    eng = HMMREngine(prefix, smpl_model)
    phi = _phi(2, 20, 5)
    with torch.no_grad():
        f = model.temporal_encode(phi)
        assert torch.equal(f, eng.temporal_encode(phi))
        a, b = model.regress(f.reshape(40, 2048)), eng.regress(f.reshape(40, 2048))
        assert torch.equal(a[0], b[0]) and all(torch.equal(a[1][k], b[1][k]) for k in KEYS)
        assert torch.equal(model.hallucinate(phi), eng.hallucinate(phi))
        out = model.predict_from_features(phi, SMPL(smpl_model))
        ref = eng.predict_from_features(phi)
        for k in ('omegas', 'omegas_delta', 'shapes'):
            assert torch.equal(out[k], ref[k]), k
        for k in ('kps', 'kps_delta', 'verts'):
            assert rel_err(out[k], ref[k]) < 1e-5, k
    # ... and through Tester: its predict of images equals the trained model on the features Tester's own ResNet computes
    from human_dynamics_b200.config import HMMRConfig
    from human_dynamics_b200 import synthetic
    from src.evaluation.tester import Tester
    cfg = HMMRConfig(load_path=prefix, batch_size=1, sequence_length=20)
    cfg.smpl_model = smpl_model
    tester = Tester(cfg)
    img = torch.from_numpy(synthetic.make_images(20, seed=4).reshape(1, 20, 224, 224, 3))
    res = tester.predict(img.numpy(), copy=True)
    with torch.no_grad():
        phi_t = tester.engine.encode_images(img.cuda().reshape(20, 224, 224, 3)).clone()
        out = model.predict_from_features(phi_t.view(1, 20, 2048), SMPL(smpl_model))
    for k in ('omegas', 'omegas_delta'):
        assert np.array_equal(out[k].cpu().numpy(), np.asarray(res[k])), k


def test_unused_graph_is_freed_and_retain_graph_works(model):
    """Outputs dropped without a backward free the whole graph (nothing the Functions save refers back to their outputs); and two
    backward passes over one graph (retain_graph) give the gradients of the summed loss."""
    import gc
    B, T = 4, 20
    N = B * T
    phi = _phi(B, T, 41).requires_grad_()

    def run():
        th, dl = model.regress(model.temporal_encode(phi).reshape(N, 2048))
        return th, dl, model.hallucinate(phi)
    th, dl, h = run()
    (th.sum() + sum(v.sum() for v in dl.values()) + h.sum()).backward()      # warm-up: backward packs, lazily built
    model.zero_grad(set_to_none=True)
    phi.grad = None
    del th, dl, h
    gc.collect()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    for _ in range(3):
        th, dl, h = run()
        assert torch.cuda.memory_allocated() > base
        del th, dl, h
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() == base
    w = torch.arange(85, dtype=torch.float32, device='cuda') / 85 - 0.5
    th, dl, h = run()
    l1, l2 = (th * w).sum() + h.sum(), sum((v * w).sum() for v in dl.values())
    l1.backward(retain_graph=True)
    l2.backward()
    two = {'phi': phi.grad.clone(), **{n: p.grad.clone() for n, p in model._params.items()}}
    model.zero_grad(set_to_none=True)
    phi.grad = None
    th, dl, h = run()
    ((th * w).sum() + h.sum() + sum((v * w).sum() for v in dl.values())).backward()
    one = {'phi': phi.grad, **{n: p.grad for n, p in model._params.items()}}
    for n in one:
        assert rel_err(two[n], one[n]) < 1e-5, n
    model.zero_grad(set_to_none=True)
    del th, dl, h, l1, l2


def test_errors_and_launch_count(engine, model):
    from human_dynamics_b200 import _lib
    with pytest.raises(_lib.HDError):
        model.temporal_encode(torch.zeros(1, 2, 2048))
    with pytest.raises(_lib.HDError):
        model.regress(torch.zeros(3, 2048))
    phi = _phi(2, 20, 7).requires_grad_()
    f = model.temporal_encode(phi)
    (gphi,) = torch.autograd.grad(f.sum(), phi, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(gphi.sum(), phi)
    x = phi.detach()
    with torch.no_grad():
        model.regress(model.temporal_encode(x).reshape(40, 2048))
        model.hallucinate(x)
        engine.regress(engine.temporal_encode(x).reshape(40, 2048))
        engine.hallucinate(x)
        torch.cuda.synchronize()
        counts = []
        for m in (model, engine):
            _lib.lib.hd_launch_count_reset()
            m.regress(m.temporal_encode(x).reshape(40, 2048))
            m.hallucinate(x)
            counts.append(int(_lib.lib.hd_launch_count()))
    assert counts[0] == counts[1], counts
    with torch.no_grad():
        out = model.temporal_encode(x)
    assert not out.requires_grad and out.grad_fn is None
