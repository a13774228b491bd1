"""The half-precision inference mode (impl 'tc1h', HD_IMPL_TC_1XF16: fp16 heads only, one MMA per product).

Kernel: for every variant launch_conv_tc selects under impl 4 (planes conv1, gather conv1, the register-staged prologue path, the
pre-split 64- / 128-wide and SHORT tiles with and without the TMA residual, the pair output, out_subsample, ragged M), the outputs equal
impl 3's bit for bit when impl 3 is given the same heads with zero remainders (activation lo = 0 and a weight pack whose remainder is 0:
the weights rounded to fp16 first).  Both modes then run the same rounded operations; impl 3 only adds +-0 * 2^-11 to its sums, so the
sign of an exact zero is the one allowed difference (values are compared, not bits).  The same outputs are within 1e-5 of float64 sums
of the fp16 operands.  The layer shapes pick the variants by the dispatch rules of conv_tc.cu: K <= 128 1x1 layers with a pair or a
residual take SHORT, Cout > 64 layers with 133..264 64-wide tiles take the 128-wide tile, the rest the 64-wide one.

Networks: HMMREngine / Tester in 'tc1h' against the float64 oracle and the reference-executed golden file at the mode's bars, repeats,
graph replay, trunk chunking and the uint8 frame path.  Measured errors are printed (pytest -s) for DESIGN.md section 2."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# bars of the mode, max |err| / max |ref| (about 4x the CPU estimate of rounding every conv's operands to fp16)
BARS = {'_phi': 2e-3, '_movie_strips': 2e-3, 'omegas': 2e-3, 'kps': 1e-2, 'joints': 1e-2, 'verts': 2.5e-2, 'verts_delta': 2.5e-2}


def rel_err(a, b):
    b = np.asarray(b, np.float64)
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


def _f16(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def _same_values(a, b):
    """Equal as numbers (+0 == -0), no NaN."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and not np.isnan(a).any() and bool((a == b).all())


# --------------------------------------------------------------------------------------------------------------------- kernel
def _run_layer(n, H, KH, Cin, Cout, mode, sub=0):
    """One conv (KH x KH, SAME, stride 1) over pre-split fp16 input, in impl 4 and in impl 3 with zero remainders.  mode: a set of
    'out' (fp32 output), 'pair' (the next layer's fp16 pair) and 'res' (a row-aligned residual).  Returns {key: (impl4, impl3)} and the
    float64 reference of the fp32 output and the pair's pre-activation."""
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.nets import PackedConv
    rng = np.random.RandomState(n * 7919 + H * 131 + KH * 17 + Cin * 7 + Cout + 3 * len(mode) + sub)
    dev = torch.device('cuda')
    M = n * H * H
    x = _f16(np.maximum(rng.normal(0, 1, size=(n, H, H, Cin)), 0))
    w = rng.normal(0, 1, size=(KH, KH, Cin, Cout)) / np.sqrt(KH * KH * Cin)
    w16 = _f16(w)
    sc = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32)
    bias = rng.normal(0, 0.2, size=Cout).astype(np.float32)
    s2 = rng.uniform(0.5, 1.5, size=Cout).astype(np.float32)
    b2 = rng.normal(0, 0.3, size=Cout).astype(np.float32)
    r = rng.normal(0, 1, size=(M, Cout)).astype(np.float32)
    pad = (KH // 2, KH // 2)
    pc4 = PackedConv(w.astype(np.float32), dev, post_scale=sc, post_shift=bias, pad=pad, tc='tc1h')   # head = RN_f16(w) = w16
    pc3 = PackedConv(w16, dev, post_scale=sc, post_shift=bias, pad=pad, tc='tc3h')                    # head w16, remainder 0
    assert float(pc3.w_nk_lo.float().abs().max()) == 0 and torch.equal(pc3.w_nk_hi, pc4.w_nk_hi)
    hi = torch.from_numpy(x).to(dev).half()
    lo = torch.zeros_like(hi)
    post2 = (torch.from_numpy(s2).to(dev), torch.from_numpy(b2).to(dev), 1)
    rt = torch.from_numpy(r).to(dev) if 'res' in mode else None
    Hs = (H + sub - 1) // sub if sub > 1 else H
    got = {}
    for impl, pc in (('tc1h', pc4), ('tc3h', pc3)):
        out = torch.full((n * Hs * Hs, Cout), float('nan'), device=dev) if 'out' in mode else None
        oh = torch.full((M, Cout), float('nan'), dtype=torch.float16, device=dev) if 'pair' in mode else None
        ol = torch.full_like(oh, float('nan')) if 'pair' in mode and impl == 'tc3h' else None
        op = pc.bind(None, n, H, H, out, inp_split=(hi, lo if impl == 'tc3h' else None),
                     out_split=(oh, ol) if 'pair' in mode else None, post2=post2 if 'pair' in mode else None,
                     res=rt, res_geom=(Cout, H, H, 1) if rt is not None else None, out_subsample=sub, impl=impl)
        assert op.d.impl == (_lib.HD_IMPL_TC_1XF16 if impl == 'tc1h' else _lib.HD_IMPL_TC_3XF16)
        op.run(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        if out is not None:
            got.setdefault('out', []).append(out.cpu().numpy())
        if oh is not None:
            got.setdefault('hi', []).append(oh.float().cpu().numpy())
    xt = torch.from_numpy(x).double().permute(0, 3, 1, 2)
    wt = torch.from_numpy(w16).double().permute(3, 2, 0, 1)
    v = F.conv2d(xt, wt, padding=KH // 2).permute(0, 2, 3, 1).reshape(M, Cout)
    v = v * torch.from_numpy(sc).double() + torch.from_numpy(bias).double()
    if rt is not None:
        v = v + torch.from_numpy(r).double()
    y = torch.relu(v * torch.from_numpy(s2).double() + torch.from_numpy(b2).double())
    v = v.numpy()
    if sub > 1:
        v = v.reshape(n, H, H, Cout)[:, ::sub, ::sub].reshape(-1, Cout)
    return got, v, y.numpy()


# (n, H, KH, Cin, Cout): K = KH^2 Cin in {64, 128, 256, 576, 1152, 2304, 4608}, Cout in {64, 128, 256, 2048}; M = n H^2 is never a
# multiple of 128.  The small-M rows run 64-wide tiles; the others have 133..264 64-wide tiles (the 128-wide tile when Cout > 64).
LAYERS = [
    (2, 14, 1, 64, 64), (8, 28, 1, 64, 256),
    (2, 14, 1, 128, 128), (12, 28, 1, 128, 128),
    (2, 14, 1, 256, 64), (8, 28, 1, 256, 256), (1, 28, 1, 256, 2048),
    (2, 14, 3, 64, 64), (8, 28, 3, 64, 256),
    (2, 14, 3, 128, 128), (12, 28, 3, 128, 128),
    (2, 14, 3, 256, 256), (8, 28, 3, 256, 256),
    (2, 7, 3, 512, 2048), (1, 28, 3, 512, 2048),
]
MODES = [('out',), ('pair',), ('res', 'pair'), ('out', 'res', 'pair')]


@pytest.mark.parametrize('n,H,KH,Cin,Cout', LAYERS)
@pytest.mark.parametrize('mode', MODES, ids='+'.join)
def test_presplit_impl4_equals_impl3_on_zero_remainders(n, H, KH, Cin, Cout, mode):
    got, v, y = _run_layer(n, H, KH, Cin, Cout, set(mode))
    for k, (g4, g3) in got.items():
        assert _same_values(g4, g3), k + ': impl 4 differs from impl 3 on zero remainders'
    if 'out' in got:
        assert rel_err(got['out'][0], v) < 1e-5
    if 'hi' in got:          # the head alone: fp16 rounding of the pre-activation
        assert np.abs(got['hi'][0] - y).max() <= 2 ** -11 * np.abs(y).max() + 1e-5 * np.abs(y).max()


@pytest.mark.parametrize('n,H,Cin,Cout', [(40, 14, 64, 256), (41, 15, 128, 96), (8, 28, 256, 512), (3, 14, 512, 1024)])
def test_presplit_impl4_subsample(n, H, Cin, Cout):
    """out_subsample: the fp32 rows x[:, ::2, ::2] from registers, the head staged; impl 4 needs no tmap_out_lo."""
    got, v, _ = _run_layer(n, H, 1, Cin, Cout, {'out', 'res', 'pair'}, sub=2)
    for k, (g4, g3) in got.items():
        assert _same_values(g4, g3), k
    assert rel_err(got['out'][0], v) < 1e-5


@pytest.mark.parametrize('n,K,Cout', [(40, 2048, 2048), (37, 1024, 1024), (40, 2048, 64)])
def test_register_staged_impl4(n, K, Cout):
    """fp32 input through the register-staged producer (fc2_res, the non-fast f_movie / IEF): the split keeps the head only."""
    from human_dynamics_b200.nets import PackedConv
    rng = np.random.RandomState(n + K + Cout)
    dev = torch.device('cuda')
    x = _f16(rng.normal(0, 1, size=(n, K)))
    w = rng.normal(0, 1, size=(K, Cout)) / np.sqrt(K)
    bias = rng.normal(0, 0.2, size=Cout).astype(np.float32)
    res = rng.normal(0, 1, size=(n, Cout)).astype(np.float32)
    outs = []
    for impl, wp in (('tc1h', w.astype(np.float32)), ('tc3h', _f16(w))):
        pc = PackedConv(wp, dev, post_shift=bias, post_relu=True, tc=impl)
        out = torch.full((n, Cout), float('nan'), device=dev)
        op = pc.bind(torch.from_numpy(x).to(dev), n, 1, 1, out, res=torch.from_numpy(res).to(dev), res_geom=(Cout, 1, 1, 1), impl=impl)
        assert op.d.impl == (4 if impl == 'tc1h' else 3) and op.d.in_ and not op.d.in_hi
        op.run(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        outs.append(out.cpu().numpy())
    assert _same_values(outs[0], outs[1])
    ref = np.maximum(x.astype(np.float64) @ _f16(w).astype(np.float64) + bias + res, 0)
    assert rel_err(outs[0], ref) < 1e-5


@pytest.mark.parametrize('n,size', [(2, 64), (3, 224), (5, 38)])
def test_conv1_planes_and_gather_impl4(n, size):
    """The ResNet root conv1 in impl 4: from the head plane alone (HD_CONV_INPUT_PLANES) and through the ragged-Cin gather producer."""
    from human_dynamics_b200 import nets
    from human_dynamics_b200._lib import lib, check, fptr
    rng = np.random.RandomState(n * 1000 + size)
    dev = torch.device('cuda')
    st = torch.cuda.current_stream().cuda_stream
    x = _f16(rng.uniform(-1, 1, size=(n, size, size, 3)))
    w = rng.normal(0, 1, size=(7, 7, 3, 64)) / np.sqrt(147)
    b = rng.normal(0, 0.2, size=64).astype(np.float32)
    xt = torch.from_numpy(x).to(dev)
    ac = F.pad(torch.from_numpy(x).double().permute(0, 3, 1, 2), (3, 3, 3, 3))
    ref = (F.conv2d(ac, torch.from_numpy(_f16(w)).double().permute(3, 2, 0, 1), stride=2).permute(0, 2, 3, 1) +
           torch.from_numpy(b).double()).numpy()
    res = {}
    for impl, wp in (('tc1h', w.astype(np.float32)), ('tc3h', _f16(w))):
        pc = nets.PackedConv1Planes(wp, b, dev)
        planes = pc.alloc_planes(n, size, impl)
        assert (planes[1] is None) == (impl == 'tc1h')
        out = torch.full((n, size // 2, size // 2, 64), float('nan'), device=dev)
        op = pc.bind(planes, n, size, out, impl)
        for _ in range(2):
            check(lib.hd_pack_conv1_planes(fptr(xt), C.c_void_p(planes[0].data_ptr()),
                                           C.c_void_p(planes[1].data_ptr()) if planes[1] is not None else None,
                                           n, size, size, planes[0].shape[2], st), 'hd_pack_conv1_planes')
            op.run(st)
        g = nets.PackedConv(wp, dev, post_shift=b, stride=2, pad=(3, 3), tc=impl)
        assert g.gather
        out_g = torch.full((n, size // 2, size // 2, 64), float('nan'), device=dev)
        if size % 2 == 0:
            gop = g.bind(xt, n, size, size, out_g, in_ld=3, impl=impl)
            assert gop.d.impl == (4 if impl == 'tc1h' else 3)
            gop.run(st)
        torch.cuda.synchronize()
        res[impl] = (out.cpu().numpy(), out_g.cpu().numpy())
    assert _same_values(res['tc1h'][0], res['tc3h'][0])
    assert rel_err(res['tc1h'][0], ref) < 1e-5
    if size % 2 == 0:
        assert _same_values(res['tc1h'][1], res['tc3h'][1])
        assert rel_err(res['tc1h'][1], ref) < 1e-5


def test_head_only_pair_writers_write_the_heads():
    """maxpool, GroupNorm + ReLU, the IEF fc1-theta kernel, the fp16 split and process_image with a NULL remainder write the same
    heads as with one."""
    from human_dynamics_b200._lib import lib, check, fptr
    dev = torch.device('cuda')
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.RandomState(5)
    vp = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None     # noqa: E731

    def both(call, shape, fill=float('nan')):      # planes: the zero border is the caller's, the kernels write the interior
        out = []
        for with_lo in (True, False):
            hi = torch.full(shape, fill, dtype=torch.float16, device=dev)
            lo = torch.full(shape, fill, dtype=torch.float16, device=dev) if with_lo else None
            check(call(vp(hi), vp(lo)), 'pair writer')
            torch.cuda.synchronize()
            out.append(hi.cpu())
        assert torch.equal(out[0], out[1]) and not torch.isnan(out[1].float()).any()

    x = torch.from_numpy(rng.normal(0, 1, size=(2, 17, 17, 64)).astype(np.float32)).to(dev)
    sc = torch.from_numpy(rng.uniform(0.5, 1.5, 64).astype(np.float32)).to(dev)
    sh = torch.from_numpy(rng.normal(0, 1, 64).astype(np.float32)).to(dev)
    both(lambda h, l: lib.hd_maxpool3x3s2_same(fptr(x), None, 2, 17, 17, 64, fptr(sc), fptr(sh), h, l, st), (2, 9, 9, 64))
    g = torch.from_numpy(rng.normal(0, 1, size=(2, 20, 2048)).astype(np.float32)).to(dev)
    ga = torch.from_numpy(rng.uniform(0.5, 1.5, 2048).astype(np.float32)).to(dev)
    be = torch.from_numpy(rng.normal(0, 1, 2048).astype(np.float32)).to(dev)
    both(lambda h, l: lib.hd_groupnorm_relu_split(fptr(g), fptr(ga), fptr(be), h, l, 2, 20, 2048, 32, 1e-6, st), (40, 2048))
    both(lambda h, l: lib.hd_split_f16(fptr(g), h, l, g.numel(), st), (40, 2048))
    P = torch.from_numpy(rng.normal(0, 1, size=(40, 1024)).astype(np.float32)).to(dev)
    th = torch.from_numpy(rng.normal(0, 1, size=(40, 85)).astype(np.float32)).to(dev)
    W = torch.from_numpy((rng.normal(0, 1, size=(85, 1024)) / 10).astype(np.float32)).to(dev)
    both(lambda h, l: lib.hd_ief_fc1_theta(fptr(P), fptr(th), 85, fptr(W), 85, 1024, h, l, None, 40, st), (40, 1024))
    fr = torch.from_numpy(rng.randint(0, 256, size=(3, 40, 50, 3)).astype(np.uint8)).to(dev)
    geom = torch.tensor([[60, 70, -5, 3]] * 3, dtype=torch.int32, device=dev)
    S, WP = 32, 40
    both(lambda h, l: lib.hd_process_image(vp(fr), 3, 40, 50, vp(geom), None, S, h, l, WP, st), (3, S + 6, WP, 4), 0.0)
    img = torch.from_numpy(rng.uniform(-1, 1, size=(3, S, S, 3)).astype(np.float32)).to(dev)
    both(lambda h, l: lib.hd_pack_conv1_planes(fptr(img), h, l, 3, S, S, WP, st), (3, S + 6, WP, 4), 0.0)


# --------------------------------------------------------------------------------------------------------------------- networks
def _engine(weights, smpl_model, B, T, S=224, **kw):
    from human_dynamics_b200 import HMMRConfig
    from human_dynamics_b200.engine import HMMREngine
    return HMMREngine(weights, smpl_model, HMMRConfig(batch_size=B, sequence_length=T, img_size=S, impl='tc1h', **kw))


def _check_bars(out, ref, tag, keys=None):
    errs = {}
    for k in (keys or BARS):
        g = out[k].cpu().numpy() if isinstance(out[k], torch.Tensor) else out[k]
        errs[k] = rel_err(g, ref[k])
    print('\n[tc1h %s] ' % tag + '  '.join('%s %.2e' % kv for kv in errs.items()))
    for k, e in errs.items():
        assert e <= BARS[k], (tag, k, e)
    return errs


def test_engine_tc1h_b2_synthetic_weights_vs_oracle(smpl_model):
    """B = 2, T = 20, 224 x 224, synthetic weights of another seed than the fixture, against the float64 oracle."""
    from human_dynamics_b200 import synthetic
    from oracle import nets_ref
    w = synthetic.make_synthetic_weights(seed=3, with_hal=True)
    img = synthetic.make_images(40, seed=5, size=224).reshape(2, 20, 224, 224, 3)
    eng = _engine(w, smpl_model, 2, 20)
    out = eng.predict(torch.from_numpy(img).cuda())
    torch.cuda.synchronize()
    ref = nets_ref.hmmr_predict(img, w, smpl_model)
    _check_bars(out, ref, 'B=2 T=20 seed 3')


def test_tester_tc1h_vs_reference_executed_golden(weights, smpl_model):
    """Tester.predict in 'tc1h' on the weights and frames of tests/golden/ref_exec_v1.npz (outputs of the reference's own source)."""
    import os
    from human_dynamics_b200 import HMMRConfig, synthetic
    from src.evaluation.tester import Tester
    with np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_exec_v1.npz')) as z:
        gold = {k: z[k] for k in z.files if k.startswith('tester_') or k == 'vert_ids'}
    img = synthetic.make_images(40, seed=21, size=224).reshape(2, 20, 224, 224, 3)
    tester = Tester(HMMRConfig(batch_size=2, sequence_length=20, weights=weights, smpl_model=smpl_model, impl='tc1h'))
    assert tester.engine.impl == 'tc1h'
    got = tester.predict(img)
    ids = gold['vert_ids']
    got = dict(got)
    got['verts'] = got['verts'][:, :, ids]
    got['verts_delta'] = got['verts_delta'][:, :, :, ids]
    ref = {k: gold['tester_' + k] for k in ('omegas', 'kps', 'joints', 'verts', 'verts_delta')}
    _check_bars(got, ref, 'Tester vs reference-executed golden', keys=list(ref))


@pytest.fixture(scope='module')
def c3_tc1h(weights, smpl_model):
    from human_dynamics_b200 import synthetic
    B, T = 32, 20
    img = synthetic.make_images(B * T, seed=11).reshape(B, T, 224, 224, 3)
    eng = _engine(weights, smpl_model, B, T)
    assert (eng.config.frame_chunk, eng.config.late_chunk) == (160, 640)
    x = torch.from_numpy(img).cuda()
    out = {k: v.clone() for k, v in eng.predict(x).items()}
    again = {k: v.clone() for k, v in eng.predict(x).items()}
    torch.cuda.synchronize()
    return eng, img, out, again


def test_c3_tc1h_first_and_last_clip_vs_oracle(c3_tc1h, weights, smpl_model):
    from oracle import nets_ref
    eng, img, out, _ = c3_tc1h
    sel = [0, img.shape[0] - 1]
    ref = nets_ref.hmmr_predict(img[sel], weights, smpl_model)
    _check_bars({k: v[sel] for k, v in out.items()}, ref, 'C3 clips 0, 31')


def test_c3_tc1h_repeats_and_chunking_are_bit_identical(c3_tc1h, weights, smpl_model):
    eng, img, out, again = c3_tc1h
    for k in out:
        assert torch.equal(out[k], again[k]), k         # repeats: bit-identical
    B, T = 4, img.shape[1]
    eng2 = _engine(weights, smpl_model, B, T, frame_chunk=16, late_chunk=32)
    o2 = eng2.predict(torch.from_numpy(img[:B]).cuda())
    torch.cuda.synchronize()
    for k in ('_phi', '_movie_strips', 'omegas', 'omegas_delta', 'cams', 'shapes'):
        assert torch.equal(o2[k], out[k][:B]), k
    for k in ('verts', 'kps', 'verts_delta'):      # SMPL picks its kernel by batch size: same numbers to 1e-5 (as in the parity mode)
        assert rel_err(o2[k].cpu().numpy(), out[k][:B].cpu().numpy()) < 2e-5, k


def test_tc1h_graph_replay_equals_eager(weights, smpl_model):
    from human_dynamics_b200 import synthetic
    B, T, S = 2, 20, 64
    eng = _engine(weights, smpl_model, B, T, S)
    a = torch.from_numpy(synthetic.make_images(B * T, seed=1, size=S)).cuda().view(B, T, S, S, 3)
    eager = {k: v.clone() for k, v in eng.predict(a).items() if not k.startswith('_')}
    buf = a.clone()
    out, nodes = eng.predict_graphed(buf)
    torch.cuda.synchronize()
    assert nodes > 100
    for k in eager:
        assert torch.equal(out[k], eager[k]), k


def test_tc1h_uint8_frames_and_feature_extractor(weights, smpl_model):
    """Tester.predict_frames (process_image writing the head plane) equals predict on the GPU crops; FeatureExtractor in 'tc1h'
    gives the engine's phis."""
    from human_dynamics_b200 import HMMRConfig
    from human_dynamics_b200.preprocess import process_images
    from src.datasets.resnet_extractor import FeatureExtractor
    from src.evaluation.tester import Tester
    B, T, H, W = 2, 20, 120, 160
    tester = Tester(HMMRConfig(batch_size=B, sequence_length=T, weights=weights, smpl_model=smpl_model, impl='tc1h'))
    rng = np.random.RandomState(8)
    frames = rng.randint(0, 256, size=(B, T, H, W, 3), dtype=np.uint8)
    boxes = np.stack([rng.uniform(60, 100, B * T), rng.uniform(40, 80, B * T), rng.uniform(0.8, 1.4, B * T)], 1).reshape(B, T, 3)
    got = {k: v.copy() for k, v in tester.predict_frames(frames, boxes).items()}
    crops, _ = process_images(frames.reshape(B * T, H, W, 3), boxes.reshape(-1, 3))
    dev = tester.predict(crops.view(B, T, 224, 224, 3), as_numpy=True)
    for k in dev:
        assert np.array_equal(got[k], dev[k]), k
    fx = FeatureExtractor(weights, img_size=224, batch_size=T, impl='tc1h')
    phis = fx.compute_all_phis(crops.cpu().numpy()[:T])
    eng_phi = tester.engine.encode_images(crops[:T].contiguous()).cpu().numpy()
    assert rel_err(phis, eng_phi) < 1e-6
