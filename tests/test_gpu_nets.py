"""GPU parity: fused conv/FC kernel, ResNet-v2-50, f_movie, IEF and the full Tester window vs the CPU oracle."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

REL = 1e-4


def rel_err(a, b):
    b = np.asarray(b, np.float64)
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


def _conv_case(rng, n, H, W, Cin, Cout, KH, KW, stride, pad, pre=None, res=None, post_scale=True, relu=True, impl='simt'):
    """Run hd_conv_gemm through PackedConv and compare with an fp64 torch reference."""
    from human_dynamics_b200.nets import PackedConv
    x = rng.normal(0, 1, size=(n, H, W, Cin)).astype(np.float32)
    w = (rng.normal(0, 1, size=(KH, KW, Cin, Cout)) / np.sqrt(KH * KW * Cin)).astype(np.float32)
    ps = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32) if post_scale else None
    pb = rng.normal(0, 0.2, size=Cout).astype(np.float32)
    dev = torch.device('cuda')
    pc = PackedConv(w, dev, ps, pb, relu, stride=stride, pad=pad, tc=(impl if impl != 'simt' else False))
    xt = torch.from_numpy(x).to(dev)
    pre_t = None
    a = torch.from_numpy(x).double()
    if pre == 'bn':
        s = rng.uniform(0.5, 1.5, size=Cin).astype(np.float32); b = rng.normal(0, 0.3, size=Cin).astype(np.float32)
        pre_t = (torch.from_numpy(s).to(dev), torch.from_numpy(b).to(dev), 0, 1)
        a = torch.relu(a * torch.from_numpy(s).double() + torch.from_numpy(b).double())
    elif pre == 'gn':
        s = rng.uniform(0.5, 1.5, size=(n, Cin)).astype(np.float32); b = rng.normal(0, 0.3, size=(n, Cin)).astype(np.float32)
        pre_t = (torch.from_numpy(s).to(dev), torch.from_numpy(b).to(dev), Cin, 1)
        a = torch.relu(a * torch.from_numpy(s).double()[:, None, None, :] + torch.from_numpy(b).double()[:, None, None, :])
    ac = F.pad(a.permute(0, 3, 1, 2), (pad[1], pad[1], pad[0], pad[0]))
    y = F.conv2d(ac, torch.from_numpy(w).double().permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)
    Ho, Wo = y.shape[1], y.shape[2]
    if ps is not None:
        y = y * torch.from_numpy(ps).double()
    y = y + torch.from_numpy(pb).double()
    res_t, res_geom = None, None
    if res is not None:
        rs = res
        r = rng.normal(0, 1, size=(n, Ho * rs, Wo * rs, Cout)).astype(np.float32)
        res_t = torch.from_numpy(r).to(dev)
        res_geom = (Cout, Ho * rs, Wo * rs, rs)
        y = y + torch.from_numpy(r).double()[:, ::rs, ::rs, :]
    if relu:
        y = torch.relu(y)
    out = torch.empty((n, Ho, Wo, Cout), dtype=torch.float32, device=dev)
    op = pc.bind(xt, n, H, W, out, pre=pre_t, res=res_t, res_geom=res_geom, impl=impl)
    assert op.out_hw == (Ho, Wo)
    op.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rel_err(out.cpu().numpy(), y.numpy()), op


CASES = [
    # n, H, W, Cin, Cout, KH, KW, stride, pad, pre, res, post_scale, relu
    (2, 14, 14, 64, 64, 1, 1, 1, (0, 0), 'bn', None, True, True),
    (2, 14, 14, 64, 256, 1, 1, 1, (0, 0), None, 1, False, False),
    (3, 9, 9, 32, 96, 3, 3, 1, (1, 1), None, None, True, True),
    (2, 14, 14, 64, 64, 3, 3, 2, (1, 1), None, None, True, True),
    (2, 8, 8, 128, 512, 1, 1, 1, (0, 0), None, 2, False, False),       # strided identity shortcut
    (3, 20, 1, 128, 128, 3, 1, 1, (1, 0), 'gn', 1, False, False),       # temporal conv + GN prologue + residual
    (37, 1, 1, 85, 1024, 1, 1, 1, (0, 0), None, 1, False, True),        # ragged K (IEF fc1 theta part)
    (37, 1, 1, 1024, 85, 1, 1, 1, (0, 0), None, 1, False, False),       # ragged N (IEF fc3)
    (2, 12, 12, 3, 64, 7, 7, 2, (3, 3), None, None, False, False),      # conv1 geometry
    (1, 5, 5, 40, 24, 3, 3, 1, (1, 1), 'bn', None, True, True),         # nothing aligned
]


@pytest.mark.parametrize('case', CASES)
def test_conv_gemm_simt(case):
    rng = np.random.RandomState(hash(case) % (2 ** 31))
    err, _ = _conv_case(rng, *case, impl='simt')
    assert err < 2e-5, err


TC_CASES = [c for c in CASES if c[3] % 32 == 0] + [
    (4, 28, 28, 128, 128, 3, 3, 1, (1, 1), None, None, True, True),
    (4, 28, 28, 256, 64, 1, 1, 1, (0, 0), 'bn', None, True, True),
    (2, 7, 7, 512, 2048, 1, 1, 1, (0, 0), None, 1, False, False),
    (5, 20, 1, 2048, 2048, 3, 1, 1, (1, 0), 'gn', 1, False, False),
    (640, 1, 1, 2048, 1024, 1, 1, 1, (0, 0), None, None, False, False),
]


@pytest.mark.parametrize('case', TC_CASES)
def test_conv_gemm_tcgen05_3xtf32(case):
    from human_dynamics_b200 import _lib
    rng = np.random.RandomState(hash(case) % (2 ** 31))
    err, op = _conv_case(rng, *case, impl='tc3')
    assert op.d.impl == _lib.HD_IMPL_TC_3XTF32, 'tensor-core path was not selected'
    print('tc3 rel err %.3e (K=%d)' % (err, case[3] * case[5] * case[6]))
    assert err < 5e-5, err        # tensor-core fp32 accumulation truncates: grows slowly with K (K=6144 -> ~3e-5)


F16_CASES = [c for c in TC_CASES if c[3] % 64 == 0] + [
    (2, 12, 12, 3, 64, 7, 7, 2, (3, 3), None, None, False, False),      # conv1: ragged K=147 through the gather producer
    (3, 224, 224, 3, 64, 7, 7, 2, (3, 3), None, None, False, False),
]


@pytest.mark.parametrize('case', F16_CASES)
def test_conv_gemm_tcgen05_3xf16(case):
    """fp16 head/remainder split (11+11 significant bits, remainder scaled by 2^11): same accuracy class as 3xTF32."""
    from human_dynamics_b200 import _lib
    rng = np.random.RandomState(hash(case) % (2 ** 31))
    err, op = _conv_case(rng, *case, impl='tc3h')
    assert op.d.impl == _lib.HD_IMPL_TC_3XF16, 'fp16 tensor-core path was not selected'
    print('tc3h rel err %.3e (K=%d)' % (err, case[3] * case[5] * case[6]))
    assert err < 5e-5, err


@pytest.mark.parametrize('shape', [
    # n, H, Cin, Cout, k, stride, with_res, fp32_out
    (3, 14, 64, 256, 1, 1, True, True),      # K <= 256: conv3-style, residual + fp32 + split outputs
    (2, 28, 128, 64, 3, 1, False, False),    # 3x3, split output only, BN=64 tile
    (2, 14, 256, 128, 3, 2, False, False),   # strided 3x3 through the cp.async gather (zero-fill padding)
    (5, 7, 512, 2048, 1, 1, True, True),     # many N tiles, ragged M (245 rows)
    (7, 28, 64, 256, 1, 1, True, True),      # K=64: 43 M-tiles x 4 N-tiles on 132 CTAs, ragged last tile (5488 rows)
    (640, 7, 256, 64, 1, 1, False, False),   # 245 tiles > 132 CTAs: several tiles per CTA through the operand ring
    (9, 14, 128, 512, 1, 1, True, False),    # residual + split output only (no fp32 store)
    (4, 14, 256, 1024, 1, 1, True, False),   # same at K = 256 (last unit of block3: the next unit's shortcut is a conv)
    (9, 14, 256, 1024, 1, 1, False, True),   # no residual, both outputs
    (300, 14, 64, 256, 1, 1, True, True),    # 460 M-tiles x 2: every CTA walks ~6 tiles (ring wrap-around, barrier phases)
    (5, 14, 128, 96, 1, 1, True, True),      # Cout = 96: the second 64-wide N tile is half outside the tensor
    (6, 14, 256, 160, 1, 1, False, True),    # Cout = 160: the third N tile has 32 valid columns of 64
])
@pytest.mark.parametrize('tma', [True, False])
def test_conv_gemm_presplit_activations_tma_flag(shape, tma):
    """A operand as a pre-activated fp16 head/remainder pair (cp.async producer) and the epilogue's second output
    relu(v*s2+b2) as such a pair, against an fp64 reference of the same arithmetic."""
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.nets import PackedConv
    n, H, Cin, Cout, k, stride, with_res, fp32_out = shape
    rng = np.random.RandomState(sum(shape))
    dev = torch.device('cuda')
    x = np.maximum(rng.normal(0, 1, size=(n, H, H, Cin)), 0).astype(np.float32)          # already pre-activated
    w = (rng.normal(0, 1, size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(np.float32)
    bias = rng.normal(0, 0.2, size=Cout).astype(np.float32)
    s2 = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32); b2 = rng.normal(0, 0.3, size=Cout).astype(np.float32)
    pc = PackedConv(w, dev, post_shift=bias, stride=stride, pad=(k // 2, k // 2), tc='tc3h')
    xt = torch.from_numpy(x).to(dev)
    hi = xt.half(); lo = ((xt - hi.float()) * 2048).half()
    Ho = (H + 2 * (k // 2) - k) // stride + 1
    out = torch.zeros((n, Ho, Ho, Cout), device=dev) if fp32_out else None
    oh = torch.zeros((n, Ho, Ho, Cout), dtype=torch.float16, device=dev); ol = torch.zeros_like(oh)
    r = rng.normal(0, 1, size=(n, Ho, Ho, Cout)).astype(np.float32) if with_res else None
    rt = torch.from_numpy(r).to(dev) if with_res else None
    op = pc.bind(None, n, H, H, out, inp_split=(hi, lo), out_split=(oh, ol), res=rt,
                 post2=(torch.from_numpy(s2).to(dev), torch.from_numpy(b2).to(dev), 1), impl='tc3h')
    if not tma:                                          # with / without HD_CONV_NO_TMA_EPILOGUE: results must not depend on it
        op.d.flags |= _lib.HD_CONV_NO_TMA_EPILOGUE
    assert op.d.impl == _lib.HD_IMPL_TC_3XF16
    assert bool(op.d.tmap_out_hi) and bool(op.d.flags & _lib.HD_CONV_NO_TMA_EPILOGUE) == (not tma)
    op.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ac = F.pad(torch.from_numpy(x).double().permute(0, 3, 1, 2), (k // 2,) * 4)
    v = F.conv2d(ac, torch.from_numpy(w).double().permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1) + torch.from_numpy(bias).double()
    if with_res:
        v = v + torch.from_numpy(r).double()
    y = torch.relu(v * torch.from_numpy(s2).double() + torch.from_numpy(b2).double())
    if fp32_out:
        assert rel_err(out.cpu().numpy(), v.numpy()) < 2e-5
    got = oh.float().cpu().double() + ol.float().cpu().double() / 2048.0       # the pair represents y to ~2^-22
    assert rel_err(got.numpy(), y.numpy()) < 2e-5


def test_conv_gemm_refuses_half_a_pair_of_n64_weight_maps():
    """tmap_hi_n64 without tmap_lo_n64 would pair the head map with the remainder operand: refused, not run."""
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.nets import PackedConv
    dev = torch.device('cuda')
    w = np.random.RandomState(5).normal(0, 0.1, size=(1, 1, 64, 128)).astype(np.float32)
    pc = PackedConv(w, dev, tc='tc3h')
    x = torch.zeros((2, 8, 8, 64), device=dev)
    out = torch.zeros((2, 8, 8, 128), device=dev)
    op = pc.bind(x, 2, 8, 8, out, impl='tc3h')
    assert op.d.impl == _lib.HD_IMPL_TC_3XF16
    op.d.tmap_hi_n64 = op.d.tmap_hi
    assert _lib.lib.hd_conv_gemm(op.ref, _lib.current_stream()) == 1          # HD_ERR_INVALID
    op.d.tmap_lo_n64 = op.d.tmap_lo
    assert _lib.lib.hd_conv_gemm(op.ref, _lib.current_stream()) == 0
    torch.cuda.synchronize()


def test_conv_gemm_tcgen05_1xtf32_is_tf32_accurate():
    rng = np.random.RandomState(3)
    err, _ = _conv_case(rng, 4, 28, 28, 128, 128, 3, 3, 1, (1, 1), None, None, True, True, impl='tc1')
    assert 1e-5 < err < 5e-3, err          # single-pass TF32: ~1e-3, NOT the parity mode


@pytest.mark.parametrize('impl', ['simt', 'tc3', 'auto'])
@pytest.mark.parametrize('n,size', [(3, 64), (2, 224)])
def test_resnet_matches_oracle(weights, impl, n, size):
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.nets import PackedResNet, ResNetPlan
    from oracle import nets_ref
    img = synthetic.make_images(n, seed=n, size=size)
    dev = torch.device('cuda')
    plan = ResNetPlan(PackedResNet(weights, dev, tc=(impl if impl != 'simt' else False)), n, size, impl)
    phi = torch.empty((n, 2048), dtype=torch.float32, device=dev)
    plan.run(torch.from_numpy(img).to(dev), phi)
    torch.cuda.synchronize()
    ref = nets_ref.encoder_resnet(img, weights).numpy()
    ref64 = nets_ref.encoder_resnet(img, weights, torch.float64).numpy()
    assert rel_err(ref, ref64) < 1e-5
    assert rel_err(phi.cpu().numpy(), ref) < REL


def _run_whole_and_stages(packed, img, size, cut, next_has_shortcut):
    """phi of the whole split plan, and of two stage plans cut in front of unit `cut` and chained the way engine._trunk chains them
    (stage A writes the fp32 map and the pre-activated pair that stage B reads): (whole plan, stage A, stage B, phi, stage phi)."""
    from human_dynamics_b200.nets import ResNetPlan, f16_pair
    n, dev = img.shape[0], img.device
    whole = ResNetPlan(packed, n, size, 'auto')
    pa = ResNetPlan(packed, n, size, 'auto', units=(0, cut), root=True, tail=False, next_pre=packed.units[cut]['pre'],
                    next_has_shortcut=next_has_shortcut)
    pb = ResNetPlan(packed, n, size, 'auto', units=(cut, len(packed.units)), root=False)
    assert whole.split and pa.split and pb.split
    mid = torch.full((n, pa.out_hw, pa.out_hw, pa.out_depth), float('nan'), device=dev)
    mid_split = f16_pair(mid.shape, dev, 'auto')
    pa.set_output(mid, mid_split)
    pb.set_input(mid, mid_split)
    phi, phi_s = (torch.empty((n, 2048), dtype=torch.float32, device=dev) for _ in range(2))
    whole.run(img, phi)
    pa.run(img, None)
    pb.run(None, phi_s)
    torch.cuda.synchronize()
    return whole, pa, pb, phi, phi_s


def _out_subsample_ops(plan):
    return sum(1 for op in plan.ops if getattr(op, 'd', None) is not None and op.d.out_subsample > 1)


@pytest.mark.parametrize('size', [224, 72])
def test_resnet_epilogue_subsample_equals_stage_subsample_pass(weights, size):
    """The unit in front of a strided identity unit writes x[:, ::s, ::s] from its conv3 epilogue (hd_conv_desc.out_subsample) instead of
    the full fp32 map + an hd_subsample pass: same bits, three passes fewer (size 72 walks odd maps: 9 -> 5 -> 3).  A stage plan that
    starts at block 1's strided identity unit has no unit in front of it and runs the hd_subsample pass."""
    from human_dynamics_b200 import synthetic, _lib
    from human_dynamics_b200.nets import PackedResNet, SubsampleOp
    from oracle import nets_ref
    dev = torch.device('cuda')
    img_h = synthetic.make_images(3, seed=8, size=size)
    img = torch.from_numpy(img_h).to(dev)
    packed = PackedResNet(weights, dev, tc='auto')
    plan, pa, pb, phi, phi_s = _run_whole_and_stages(packed, img, size, 2, False)
    assert not any(isinstance(op, SubsampleOp) for op in plan.ops) and _out_subsample_ops(plan) == 3
    assert isinstance(pb.ops[0], SubsampleOp) and sum(isinstance(op, SubsampleOp) for op in pa.ops + pb.ops) == 1
    assert _out_subsample_ops(pa) + _out_subsample_ops(pb) == 2
    assert torch.equal(phi, phi_s)
    assert rel_err(phi.cpu().numpy(), nets_ref.encoder_resnet(img_h, weights).numpy()) < REL
    # descriptors outside the activation-map contract refuse the flag instead of silently writing the full map
    op = next(op for op in plan.ops if getattr(op, 'd', None) is not None and op.d.out and op.d.res)
    op.d.out_subsample = 2
    op.d.flags |= _lib.HD_CONV_NO_TMA_EPILOGUE
    assert _lib.lib.hd_conv_gemm(op.ref, _lib.current_stream()) == 4          # HD_ERR_UNSUPPORTED
    op.d.out_subsample = 0


def test_resnet_dead_fp32_outputs_are_dead_across_stages(weights):
    """Skipping the fp32 copies nobody reads (pool1 output, block outputs in front of a conv shortcut) must not change a bit: the whole
    plan against stage plans cut in front of block 2's conv shortcut, whose stage A skips its fp32 output or writes it."""
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.nets import PackedResNet
    dev = torch.device('cuda')
    img = torch.from_numpy(synthetic.make_images(3, seed=5, size=224)).to(dev)
    packed = PackedResNet(weights, dev, tc='auto')
    assert 'shortcut' in packed.units[3]

    def dead(plan):
        return sum(1 for op in plan.ops if getattr(op, 'd', None) is not None and not op.d.out and op.d.res)
    outs = []
    for skip in (True, False):
        plan, pa, pb, phi, phi_s = _run_whole_and_stages(packed, img, 224, 3, skip)
        assert plan.pool_f32_dead and pa.pool_f32_dead
        assert dead(plan) == 3 and dead(pa) + dead(pb) == (3 if skip else 2)
        outs += [phi, phi_s]
    assert all(torch.equal(outs[0], o) for o in outs[1:])


@pytest.mark.parametrize('impl', ['simt', 'auto'])
def test_fmovie_matches_oracle(weights, impl):
    from human_dynamics_b200.nets import PackedFMovie, FMoviePlan
    from oracle import nets_ref
    B, T = 3, 20
    x = np.random.RandomState(0).normal(0, 1, size=(B, T, 2048)).astype(np.float32)
    dev = torch.device('cuda')
    plan = FMoviePlan(PackedFMovie(weights, dev, 3, tc=(impl if impl != 'simt' else False)), B, T, impl)
    y = plan.run(torch.from_numpy(x).to(dev))
    torch.cuda.synchronize()
    ref = nets_ref.az_fc2_groupnorm(x, weights, 3).numpy()
    assert rel_err(y.cpu().numpy(), ref) < REL


@pytest.mark.parametrize('impl', ['simt', 'auto'])
def test_ief_matches_oracle(weights, impl):
    from human_dynamics_b200.nets import PackedIEF, IEFPlan
    from oracle import nets_ref
    N = 45
    phi = np.random.RandomState(1).normal(0, 1, size=(N, 2048)).astype(np.float32)
    dev = torch.device('cuda')
    packed = PackedIEF(weights, dev, tc=(impl if impl != 'simt' else False))
    plan = IEFPlan(packed, N, impl=impl)
    theta0 = packed.mean_param.expand(N, 85).contiguous()
    theta, deltas = plan.run(torch.from_numpy(phi).to(dev), theta0)
    torch.cuda.synchronize()
    om = np.tile(weights['mean_param'].reshape(1, 85), (N, 1))
    rt, rd = nets_ref.call_hmr_ief(phi, om, weights, 'single_view_ief', 85, 3, (0, -5, 5), True, True)
    assert rel_err(theta.cpu().numpy(), rt.numpy()) < REL
    for dt in (-5, 5):
        assert rel_err(deltas[dt].cpu().numpy(), rd[dt].numpy()) < REL


def _check_predict(got, ref, keys=None):
    for k, v in ref.items():
        if k.startswith('_') or (keys and k not in keys):
            continue
        g = got[k].cpu().numpy() if isinstance(got[k], torch.Tensor) else got[k]
        assert g.shape == v.shape, (k, g.shape, v.shape)
        assert rel_err(g, v) < REL, (k, rel_err(g, v))


@pytest.mark.parametrize('impl', ['simt', 'tc3', 'auto'])
def test_full_window_matches_oracle(weights, smpl_model, impl):
    """BASELINE config 3 wiring at B=2, T=20, 224x224 (oracle ResNet on 40 frames takes ~10 s)."""
    from human_dynamics_b200 import synthetic, HMMRConfig
    from human_dynamics_b200.engine import HMMREngine
    from oracle import nets_ref
    B, T = 2, 20
    img = synthetic.make_images(B * T, seed=0).reshape(B, T, 224, 224, 3)
    eng = HMMREngine(weights, smpl_model, HMMRConfig(batch_size=B, sequence_length=T, frame_chunk=16), impl=impl)
    got = eng.predict(torch.from_numpy(img).cuda())
    torch.cuda.synchronize()
    ref = nets_ref.hmmr_predict(img, weights, smpl_model)
    assert rel_err(got['_phi'].cpu().numpy(), ref['_phi']) < REL
    assert rel_err(got['_movie_strips'].cpu().numpy(), ref['_movie_strips']) < REL
    _check_predict(got, ref)


def test_single_frame_path_matches_oracle(weights, smpl_model):
    """BASELINE config 2 wiring (ResNet + 3-iter IEF + SMPL, no temporal encoder) at batch 8."""
    from human_dynamics_b200 import synthetic, HMMRConfig
    from human_dynamics_b200.engine import HMMREngine
    from oracle import nets_ref
    n = 8
    img = synthetic.make_images(n, seed=4)
    eng = HMMREngine(weights, smpl_model, HMMRConfig(batch_size=n, sequence_length=1))
    got = eng.predict(torch.from_numpy(img).cuda().view(n, 1, 224, 224, 3), single_frame=True)
    torch.cuda.synchronize()
    ref = nets_ref.single_frame_predict(img, weights, smpl_model)
    for k in ('omegas', 'verts', 'joints', 'kps', 'poses'):
        assert rel_err(got[k].cpu().numpy().reshape(ref[k].shape), ref[k]) < REL, k


def test_tester_surface_and_sliding_window(weights, smpl_model):
    """src.evaluation.tester.Tester: predict() dict contract and predict_all_images windowing (tester.py:260-312)."""
    from human_dynamics_b200 import synthetic, HMMRConfig
    from src.evaluation.tester import Tester
    from oracle import nets_ref
    B, T, S = 2, 20, 64
    cfg = HMMRConfig(batch_size=B, sequence_length=T, img_size=S, weights=weights, smpl_model=smpl_model, pred_mode='pred')
    tester = Tester(cfg)
    N = 19                                        # -> count = ceil(19 / (8*2)) = 2 passes, ragged tail
    frames = synthetic.make_images(N, seed=9, size=S)
    res = tester.predict_all_images(frames)                         # cached per-frame features (default)
    res_literal = tester.predict_all_images(frames, cache_features=False)   # the reference's literal image windows
    for k in res:
        assert np.array_equal(res[k], res_literal[k]), 'feature cache changed ' + k
    margin, g = 6, 8
    count = int(np.ceil(N / (g * B)))
    padded = np.concatenate([np.zeros((margin, S, S, 3), np.float32), frames,
                             np.zeros((count * B * g + T - N, S, S, 3), np.float32)])
    ref_chunks = []
    for c in range(count):
        batch = np.stack([padded[(c * B + i) * g:(c * B + i) * g + T] for i in range(B)])
        ref_chunks.append(nets_ref.hmmr_predict(batch, weights, smpl_model))
    for k in ('verts', 'omegas', 'kps', 'joints', 'poses', 'cams', 'shapes', 'verts_delta', 'omegas_delta', 'kps_delta'):
        v = np.array([r[k] for r in ref_chunks])[:, :, margin:-margin]
        v = v.reshape((-1,) + v.shape[3:])[:N]
        assert res[k].shape == v.shape, k
        assert rel_err(res[k], v) < REL, k
    assert set(res.keys()) == {a + b for a in ('cams', 'joints', 'kps', 'poses', 'shapes', 'verts', 'omegas') for b in ('', '_delta')}
    with pytest.raises(ValueError):
        tester.predict(np.zeros((1, T, S, S, 3), np.float32))     # static shapes, like the TF placeholder


def test_hal_mode_and_models_surface(weights, smpl_model):
    """pred_mode='hal' (fc2_res) and the reference-named functions in src.models / src.omega."""
    from human_dynamics_b200 import synthetic, HMMRConfig
    from src.evaluation.tester import Tester
    import src.models as M
    from src.omega import OmegasPred, f_movie
    from oracle import nets_ref
    B, T, S = 2, 5, 64
    cfg = HMMRConfig(batch_size=B, sequence_length=T, img_size=S, weights=weights, smpl_model=smpl_model, pred_mode='hal')
    tester = Tester(cfg)
    img = synthetic.make_images(B * T, seed=2, size=S).reshape(B, T, S, S, 3)
    got = tester.predict(img)
    ref = nets_ref.hmmr_predict(img, weights, smpl_model, pred_mode='hal')
    _check_predict(got, ref)
    # stateless functions resolve weights through the active engine
    x = torch.from_numpy(img.reshape(B * T, S, S, 3)).cuda()
    phi, scope = M.get_image_encoder()(x, is_training=False, reuse=False)
    assert scope == 'resnet_v2_50'
    assert rel_err(phi.cpu().numpy(), ref['_phi'].reshape(B * T, -1)) < REL
    strips = M.get_temporal_encoder()(is_training=False, net=phi.view(B, T, -1), num_conv_layers=3)
    assert f_movie is M.az_fc2_groupnorm
    assert rel_err(strips.cpu().numpy(), nets_ref.az_fc2_groupnorm(ref['_phi'], weights, 3).numpy()) < REL
    om = torch.from_numpy(np.tile(weights['mean_param'].reshape(1, 85), (B * T, 1))).cuda()
    theta, deltas = M.call_hmr_ief(phi, om, 'single_view_ief', 85, 3, False, (0, -5, 5), True, True)
    rt, rd = nets_ref.call_hmr_ief(ref['_phi'].reshape(B * T, -1), om.cpu().numpy(), weights, 'single_view_ief', 85, 3,
                                   (0, -5, 5), True, True)
    assert rel_err(theta.cpu().numpy(), rt.numpy()) < REL
    assert rel_err(deltas[5].cpu().numpy(), rd[5].numpy()) < REL
    # OmegasPred container: append_batched -> compute_smpl -> getters (omega.py:237-304)
    from src.tf_smpl.batch_smpl import SMPL
    op = OmegasPred(cfg, SMPL(smpl_model), use_optcam=False, vis_max_batch=B, batch_size=B, is_training=False)
    op.append_batched(theta.view(B, T, 85))
    OmegasPred.compute_all_smpl([op])
    from oracle.smpl_ref import SMPLRef
    raw = rt.numpy()
    v_ref, _, _ = SMPLRef(smpl_model)(raw[:, 75:], raw[:, 3:75], get_skin=True)
    assert rel_err(op.get_verts().cpu().numpy().reshape(v_ref.shape), v_ref) < REL
    assert op.get_kps().shape == (B, T, 25, 2) and op.get_poses_rot().shape == (B, T, 24, 3, 3)


@pytest.mark.parametrize('n,size', [(2, 24), (3, 224), (5, 64)])
@pytest.mark.parametrize('tma', [True, False])
def test_conv1_from_padded_fp16_planes_tma_flag(n, size, tma):
    """ResNet root conv1 (7x7/2, explicit pad 3+3, bias) through the plane-input tensor-core path: hd_pack_conv1_planes
    + hd_conv_gemm(HD_CONV_INPUT_PLANES) against an fp64 convolution."""
    from human_dynamics_b200 import nets, _lib
    from human_dynamics_b200._lib import lib, check, fptr
    import ctypes as C
    rng = np.random.RandomState(n * 1000 + size)
    dev = torch.device('cuda')
    x = rng.uniform(-1, 1, size=(n, size, size, 3)).astype(np.float32)
    w = (rng.normal(0, 1, size=(7, 7, 3, 64)) / np.sqrt(147)).astype(np.float32)
    b = rng.normal(0, 0.2, size=64).astype(np.float32)
    pc = nets.PackedConv1Planes(w, b, dev)
    planes = pc.alloc_planes(n, size)
    out = torch.zeros((n, size // 2, size // 2, 64), device=dev)
    op = pc.bind(planes, n, size, out)
    if not tma:                                          # results must not depend on HD_CONV_NO_TMA_EPILOGUE
        op.d.flags |= _lib.HD_CONV_NO_TMA_EPILOGUE
    assert bool(op.d.tmap_out) and bool(op.d.flags & 1) == (not tma)
    st = torch.cuda.current_stream().cuda_stream
    xt = torch.from_numpy(x).to(dev)
    for _ in range(2):          # twice: the zero border must survive the first pass
        check(lib.hd_pack_conv1_planes(fptr(xt), C.c_void_p(planes[0].data_ptr()), C.c_void_p(planes[1].data_ptr()), n, size, size,
                                       planes[0].shape[2], st), 'pack')
        op.run(st)
    torch.cuda.synchronize()
    ac = F.pad(torch.from_numpy(x).double().permute(0, 3, 1, 2), (3, 3, 3, 3))
    y = F.conv2d(ac, torch.from_numpy(w).double().permute(3, 2, 0, 1), stride=2).permute(0, 2, 3, 1) + torch.from_numpy(b).double()
    assert tuple(out.shape) == tuple(y.shape)
    assert rel_err(out.cpu().numpy(), y.numpy()) < 2e-5
    # the planes represent the image to ~2^-22 and keep a zero border
    rec = planes[0].float() + planes[1].float() / 2048.0
    assert float((rec[:, 3:3 + size, 3:3 + size, :3] - xt).abs().max()) < 1e-6
    assert float(rec[:, :3].abs().max()) == 0 and float(rec[:, :, :3].abs().max()) == 0 and float(rec[..., 3].abs().max()) == 0


@pytest.mark.parametrize('n,H,C,s', [(3, 56, 256, 2), (5, 7, 128, 2), (2, 9, 64, 3), (1, 28, 512, 2)])
def test_subsample_is_strided_slice(n, H, C, s):
    """slim's identity shortcut of a strided unit: x[:, ::s, ::s, :] (pixel counts that are not multiples of the 4 pixels a warp copies)."""
    from human_dynamics_b200._lib import lib, check, fptr
    x = torch.randn((n, H, H, C), device='cuda')
    Ho = (H - 1) // s + 1
    out = torch.full((n, Ho, Ho, C), float('nan'), device='cuda')
    guard = torch.zeros(64, device='cuda')          # directly behind `out` in most allocators; the tail warp must not write past the end
    check(lib.hd_subsample(fptr(x), fptr(out), n, H, H, C, s, torch.cuda.current_stream().cuda_stream), 'hd_subsample')
    torch.cuda.synchronize()
    assert torch.equal(out, x[:, ::s, ::s, :].contiguous())
    assert float(guard.abs().sum()) == 0.0


def test_weight_packing_layouts_and_split_precision():
    """What the tensor-core kernels are fed, as hd_pack_weight writes it on the device: K-major [Cout_pad, K] with K = (ky, kx, ci) (TF
    HWIO flattened), each weight as an fp16 head + 2^11-scaled fp16 remainder that together carry >= 21 significant bits; conv1's 7x7x3
    filter re-laid as 8 x 8 x 4 taps with zero weights on the padding taps."""
    from human_dynamics_b200 import nets
    rng = np.random.RandomState(3)
    w = (rng.normal(0, 1, size=(3, 3, 64, 96)) / 24).astype(np.float32)
    pc = nets.PackedConv(w, torch.device('cuda'), tc='auto')
    assert pc.tc == 'f16' and (pc.K, pc.K_pad, pc.Cout) == (576, 576, 96)
    torch.cuda.synchronize()
    hi, lo = pc.w_nk_hi.cpu().numpy(), pc.w_nk_lo.cpu().numpy()
    assert hi.shape == lo.shape == (128, 576) and hi.dtype == lo.dtype == np.float16          # rows padded to the 128-wide N tile
    assert not hi[96:].any() and not lo[96:].any()
    rec = hi[:96].astype(np.float64) + lo[:96].astype(np.float64) / 2048.0
    ref = w.reshape(576, 96).T.astype(np.float64)                                            # [co, (ky, kx, ci)]
    assert np.abs(rec - ref).max() <= np.abs(ref).max() * 2.0 ** -21
    assert np.array_equal(hi[:96], ref.astype(np.float16))                                   # head = RN_f16(w)
    assert np.array_equal(pc.w_kn.cpu().numpy(), w.reshape(576, 96))                         # exact-FP32 path keeps TF's [K, Cout]
    small = nets.PackedConv(w[:, :, :, :64], torch.device('cuda'), tc='auto')
    assert small.w_nk_hi.shape == (64, 576)                                                  # Cout <= 64: 64-wide tile, no padding rows
    # conv1 planes
    w1 = rng.normal(0, 0.1, size=(7, 7, 3, 64)).astype(np.float32)
    p1 = nets.PackedConv1Planes(w1, np.zeros(64, np.float32), torch.device('cuda'))
    torch.cuda.synchronize()
    t = (p1.w_nk_hi.cpu().numpy().astype(np.float64) + p1.w_nk_lo.cpu().numpy().astype(np.float64) / 2048.0).reshape(64, 8, 8, 4)
    assert not t[:, 7].any() and not t[:, :, 7].any() and not t[:, :, :, 3].any()            # phantom kernel row / pixel / channel
    assert np.abs(t[:, :7, :7, :3] - w1.transpose(3, 0, 1, 2)).max() <= np.abs(w1).max() * 2.0 ** -21
    assert p1.plane_width(224) == 232 and p1.plane_width(64) == 72
