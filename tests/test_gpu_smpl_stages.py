"""GPU: the SMPL forward kernels one entry point at a time, against oracle/smpl_stages_ref.py in float64.

Every stage is fed the kernel's own upstream outputs (the reference skins the GPU's v_posed with the GPU's A12, regresses the GPU's
verts, and so on) and the float32 constants the kernels read, so each error is that stage's own and the bars sit near float32
rounding.  Every output starts as NaN inside a larger buffer (guard rows, unused interleave slots, padded pitches): a test asserts
that each stage writes all of its footprint and nothing else.  Every launch runs twice and must give the same bits.

Covered: hd_smpl_pose (all seven outputs, the fp16 operand splits bit for bit), the kinematic trees the FK accepts (SMPL's, a
depth-23 chain, a star, random trees) through hd_smpl_pose / hd_global_rigid / hd_smpl_forward, hd_rodrigues at its edges, the
fused hd_smpl_forward in all four template instances (8 or 32 poses per CTA x 4 or runtime non-zeros), the staged path (blend
GEMM, hd_smpl_lbs, hd_smpl_lbs_tc across run counts, V and pitches, hd_smpl_joints), hd_orth_proj, and the per-device
shared-memory opt-in with two GPUs."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import smpl_stages_ref as sr

pytestmark = pytest.mark.gpu

# Bars: max |err| / max |ref| per tensor (absolute for Rs, whose entries are bounded by 1), set at 3-5x the worst value measured on
# an NVIDIA H100 80GB HBM3 (700 W power limit, max SM clock 1980 MHz), which is next to each bar.  Every kernel here is deterministic,
# so a rerun measures the same values.  `pytest -s` prints the worst value per bar.
RS_BAR = 1e-6             # Rodrigues (hd_smpl_pose, hd_rodrigues, the forwards), absolute: 3.3e-7
FK_BAR = 1.5e-6           # Jtr, A12 / A44 from the GPU's Rs, every tree including the depth-23 chain: 3.5e-7 (A12)
BLEND_BAR = 6e-7          # v_posed of the tensor-core blend GEMM: 1.6e-7
SKIN_BAR = 8e-7           # CUDA-core skinning (hd_smpl_lbs) of the GPU's v_posed and A12: 1.9e-7
SKIN_TC_BAR = 1.5e-6      # tensor-core skinning (hd_smpl_lbs_tc), weights and A as unscaled fp16 pairs: 3.3e-7
JOINTS_BAR = 4e-7         # keypoint regression of the GPU's verts: 8.4e-8
FWD_BAR = 5e-6            # whole forward, fused or staged, against float64 of the same inputs and float32 constants, and staged
                          # against fused: 1.3e-6 (verts; joints 8.7e-7, kps 5.1e-7, Jtr 4.6e-7)
# The pose-blend part of the fused verts (verts minus the same forward without posedirs; about 1e-2 at most) against float64: 6.8e-5.
# This is the absolute error of verts (~1e-6) over a small part: smpl_skin_kernel starts its blend accumulator at v_template, so each
# of the 217 blend terms is added at the template's magnitude and rounded there, where the reference adds the blend sum to v_shaped
# once.  The bar therefore sees a pose-blend error of a few 1e-4 of that part, and no finer.
POSE_PART_BAR = 3e-4

NAN = float('nan')
WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print('worst %-28s %.2e' % (k, WORST[k]))


def _bar(name, value, bar, tag):
    WORST[name] = max(WORST.get(name, 0.0), value)
    assert value < bar, (tag, name, value, bar)


def _lib():
    from human_dynamics_b200._lib import lib, check
    return lib, check


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, NAN, dtype=dtype, device='cuda')


def _rel(got, ref):
    ref = ref.double()
    return float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300))


def _abs(got, ref):
    return float((got.double() - ref.double()).abs().max())


def _bits(t):
    return t.contiguous().view({torch.float32: torch.int32, torch.float16: torch.int16, torch.uint8: torch.uint8}[t.dtype])


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


def _all_nan(t):
    return bool(torch.isnan(t).all())


def _others(buf, rows):
    """The rows of buf not in `rows` (which the stage must leave NaN)."""
    keep = torch.ones(buf.shape[0], dtype=torch.bool, device=buf.device)
    keep[rows] = False
    return buf[keep]


def _slot_rows(N, mul, off):
    return torch.arange(N, device='cuda') * mul + off


def _omega(N, seed, ld=91):
    """beta (N,10), theta (N,72), cam (N,3) as column views of one [N, ld] buffer (the engine's omega layout, padded pitch)."""
    from human_dynamics_b200 import synthetic
    beta, theta = synthetic.make_smpl_inputs(N, seed=seed)
    rng = np.random.RandomState(seed + 1000)
    om = np.full((N, ld), np.nan, np.float32)
    om[:, 0] = rng.uniform(0.5, 1.5, N)
    om[:, 1:3] = rng.uniform(-0.3, 0.3, (N, 2))
    om[:, 3:75] = theta
    om[:, 75:85] = beta
    om = torch.from_numpy(om).cuda()
    return om[:, 75:85], om[:, 3:75], om[:, 0:3]


# ------------------------------------------------------------------------------------------------------------------------------------
# models: SMPL-sized ones with 4, 8 (5-6 real) and 24 skinning non-zeros per vertex, small ones with a ragged last vertex tile, and one
# without keypoints
# ------------------------------------------------------------------------------------------------------------------------------------
def _five_or_six_weights(model, seed):
    rng = np.random.RandomState(seed)
    V = model['v_template'].shape[0]
    W = np.zeros((V, 24))
    for v in range(V):
        k = rng.randint(5, 7)
        W[v, rng.choice(24, size=k, replace=False)] = rng.rand(k) + 0.05
    m = dict(model)
    m['weights'] = W / W.sum(1, keepdims=True)
    return m


@functools.lru_cache(maxsize=None)
def _model(name):
    from human_dynamics_b200 import synthetic
    V = {'v128': 128, 'v130': 130}.get(name.split('_')[-1], 6890)
    kind = name.split('_')[0]
    if kind == 'nnz4':
        return synthetic.make_synthetic_smpl(seed=2, num_verts=V)
    if kind == 'nnz24':
        return synthetic.make_synthetic_smpl(seed=7, dense_weights=True, num_kps=19, num_verts=V)
    if kind == 'nnz8':
        return _five_or_six_weights(synthetic.make_synthetic_smpl(seed=3, num_verts=V), seed=4)
    if kind == 'nokp':
        m = dict(synthetic.make_synthetic_smpl(seed=5, num_verts=V))
        m['cocoplus_regressor'] = np.zeros((0, V))
        return m
    raise KeyError(name)


_CONSTS = {}


def _consts(name, joint_type='cocoplus', tc=False, tree=None):
    key = (name, joint_type, tc, tree)
    if key not in _CONSTS:
        from human_dynamics_b200.smpl import SMPLConstants
        m = _model(name) if tree is None else sr.with_tree(_model(name), sr.test_trees()[tree])
        _CONSTS[key] = SMPLConstants(m, joint_type=joint_type, tc=tc)
    return _CONSTS[key]


def _k64(c):
    """The float32 constants SMPLConstants uploaded, as float64 on the device, in smpl_stages_ref's keys (skinning weights and the
    keypoint regressor densified from their ELL / CSC forms)."""
    V, K = c.num_verts, c.num_kps
    W = torch.zeros((V, 24), dtype=torch.float64, device='cuda')
    W.scatter_add_(1, c.lbs_idx.long(), c.lbs_w.double())
    reg = torch.zeros((K, V), dtype=torch.float64, device='cuda')
    if K:
        ptr = c.kp_ptr.long()
        rows = torch.repeat_interleave(torch.arange(K, device='cuda'), ptr[1:] - ptr[:-1])
        reg[rows, c.kp_vidx.long()[:len(rows)]] = c.kp_w.double()[:len(rows)]
    return {'v_template': c.v_template.double(), 'dirs': c.dirs.double(), 'J_template': c.J_template.double(),
            'J_shapedirs': c.J_shapedirs.double(), 'weights': W, 'regressor': reg, 'parents': c.parents, 'num_verts': V}


def test_models_have_the_intended_shapes():
    assert _consts('nnz4').lbs_nnz == 4 and _consts('nnz8').lbs_nnz == 8 and _consts('nnz24').lbs_nnz == 24
    assert _consts('nnz8_v130').lbs_nnz == 8 and _consts('nokp').num_kps == 0
    c = _consts('nnz8')
    real = (c.lbs_w != 0).sum(1)
    assert int(real.min()) == 5 and int(real.max()) == 6
    assert bool((c.lbs_idx[c.lbs_w == 0] == 0).all())       # padding entries: joint 0, weight 0


# ------------------------------------------------------------------------------------------------------------------------------------
# hd_smpl_pose
# ------------------------------------------------------------------------------------------------------------------------------------
def _pose_run(c, beta, theta, N, mul, off, coef_ld):
    """hd_smpl_pose with every output requested, each in a NaN buffer with guard rows (slotted outputs: N * mul + 2 rows)."""
    lib, check = _lib()
    o = {'rs': _nan((N + 1, 216)), 'Rs': _nan((N * mul + 2, 24, 9)), 'Jtr': _nan((N * mul + 2, 24, 3)), 'A12': _nan((N + 1, 288)),
         'coef': _nan((N + 1, coef_ld)), 'coef_hi': _nan((N + 1, coef_ld), torch.float16),
         'coef_lo': _nan((N + 1, coef_ld), torch.float16), 'a12t_hi': _nan((N + 1, 12, 32), torch.float16),
         'a12t_lo': _nan((N + 1, 12, 32), torch.float16)}
    check(lib.hd_smpl_pose(C.byref(c.c), _vp(beta), beta.stride(0), _vp(theta), theta.stride(0), N, _vp(o['Rs']), _vp(o['Jtr']),
                           _vp(o['A12']), _vp(o['coef']), coef_ld, _vp(o['coef_hi']), _vp(o['coef_lo']), _vp(o['a12t_hi']),
                           _vp(o['a12t_lo']), mul, off, _vp(o['rs']), N * 216 * 4, _st()), 'hd_smpl_pose')
    torch.cuda.synchronize()
    return o


def _pose_twice(c, beta, theta, N, mul=1, off=0, coef_ld=256):
    o = _pose_run(c, beta, theta, N, mul, off, coef_ld)
    o2 = _pose_run(c, beta, theta, N, mul, off, coef_ld)
    for k in o:
        assert _same_bits(o[k], o2[k]), 'hd_smpl_pose rerun differs: ' + k
    return o


def _split_f16x2(x):
    """conv_common.cuh split_f16x2: clamp to the finite fp16 range, head = RN_f16(x), lo = RN_f16((x - head) * 2^11)."""
    x = x.clamp(-65504.0, 65504.0)
    hi = x.half()
    return hi, ((x - hi.float()) * 2048.0).half()


def _check_fk(tag, c, beta, R, Jtr, A12, tree_parents=None, rotate_base=False):
    k = _k64(c)
    J = sr.rest_joints(beta.double(), k['J_template'], k['J_shapedirs'])
    jtr, A = sr.forward_kinematics(R.double(), J, c.parents if tree_parents is None else tree_parents, rotate_base)
    _bar('Jtr', _rel(Jtr, jtr), FK_BAR, tag)
    _bar('A12', _rel(A12.reshape(-1, 24, 3, 4), A), FK_BAR, tag)


@pytest.mark.parametrize('slot', [(1, 0), (3, 1), (3, 2)])
@pytest.mark.parametrize('N', [1, 3, 4, 5, 257])
def test_pose_kernel_all_outputs(N, slot):
    c = _consts('nnz4')
    mul, off = slot
    beta, theta, _ = _omega(N, seed=N)
    rows = _slot_rows(N, mul, off)
    eye = torch.eye(3, device='cuda')
    for coef_ld in (217, 256, 260):
        tag = 'N=%d slot=%s coef_ld=%d' % (N, slot, coef_ld)
        o = _pose_twice(c, beta, theta, N, mul, off, coef_ld)
        for k in ('rs', 'A12', 'coef', 'coef_hi', 'coef_lo', 'a12t_hi', 'a12t_lo'):
            assert not torch.isnan(o[k][:N]).any() and _all_nan(o[k][N:]), (tag, k)
        for k in ('Rs', 'Jtr'):
            assert not torch.isnan(o[k][rows]).any() and _all_nan(_others(o[k], rows)), (tag, k)
        R = o['rs'][:N].reshape(N, 24, 3, 3)
        _bar('Rs', _abs(R, sr.rodrigues(theta.double().reshape(N, 24, 3))), RS_BAR, tag)
        assert _same_bits(o['Rs'][rows].reshape(N, 24, 3, 3), R), tag
        _check_fk(tag, c, beta, R, o['Jtr'][rows], o['A12'][:N])
        # the blend operand row [beta | R_j - I, j = 1..23 | 0], formed in float32 from the kernel's own Rs, and its fp16 split
        row = torch.cat([beta, (R[:, 1:] - eye).reshape(N, 207), torch.zeros((N, coef_ld - 217), device='cuda')], 1)
        assert _same_bits(o['coef'][:N], row), tag
        hi, lo = _split_f16x2(row)
        assert _same_bits(o['coef_hi'][:N], hi) and _same_bits(o['coef_lo'][:N], lo), tag
        # A^T as an unscaled fp16 pair, joints 24..31 of K exactly zero
        A = o['A12'][:N].reshape(N, 24, 12).transpose(1, 2)
        ahi = torch.zeros((N, 12, 32), dtype=torch.float16, device='cuda')
        alo = torch.zeros((N, 12, 32), dtype=torch.float16, device='cuda')
        ahi[:, :, :24] = A.half()
        alo[:, :, :24] = (A - A.half().float()).half()
        assert _same_bits(o['a12t_hi'][:N], ahi) and _same_bits(o['a12t_lo'][:N], alo), tag


# ------------------------------------------------------------------------------------------------------------------------------------
# kinematic trees
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('tree', ['smpl', 'chain', 'star', 'random1', 'random2'])
def test_trees(tree):
    """The level-by-level FK (fk_chain) on trees from depth 1 to depth 23, in all three kernels that run it."""
    lib, check = _lib()
    parents = sr.test_trees()[tree]
    c = _consts('nnz4_v130', tree=tree)
    assert list(c.parents) == [-1] + list(parents[1:])
    N = 37
    beta, theta, cam = _omega(N, seed=40)
    o = _pose_twice(c, beta, theta, N)
    R = o['rs'][:N].reshape(N, 24, 3, 3)
    _check_fk('pose ' + tree, c, beta, R, o['Jtr'][:N], o['A12'][:N])
    # hd_global_rigid on the same rotations and other joints, with and without the base flip
    Js = torch.from_numpy(np.random.RandomState(41).normal(0, 0.3, size=(N, 24, 3)).astype(np.float32)).cuda()
    par = (C.c_int * 24)(*[int(p) for p in c.parents])
    for rb in (0, 1):
        outs = []
        for _ in range(2):
            nj, A44 = _nan((N + 1, 24, 3)), _nan((N + 1, 24, 16))
            check(lib.hd_global_rigid(_vp(R.contiguous()), _vp(Js), par, _vp(nj), _vp(A44), N, rb, _st()), 'hd_global_rigid')
            torch.cuda.synchronize()
            outs.append((nj, A44))
        nj, A44 = outs[0]
        assert _same_bits(nj, outs[1][0]) and _same_bits(A44, outs[1][1])
        assert not torch.isnan(nj[:N]).any() and _all_nan(nj[N:]) and _all_nan(A44[N:])
        A44 = A44[:N].reshape(N, 24, 4, 4)
        assert torch.equal(A44[:, :, 3], torch.tensor([0.0, 0.0, 0.0, 1.0], device='cuda').expand(N, 24, 4))
        jtr, A = sr.forward_kinematics(R.double(), Js.double(), parents, rotate_base=bool(rb))
        _bar('Jtr', _rel(nj[:N], jtr), FK_BAR, 'global_rigid %s rb=%d' % (tree, rb))
        _bar('A12', _rel(A44[:, :, :3], A), FK_BAR, 'global_rigid %s rb=%d' % (tree, rb))
    # the fused forward of a model with this tree
    got = _forward_run(c, beta, theta, cam, N, 1, 0)
    _check_forward('forward ' + tree, c, beta, theta, cam, got)


# ------------------------------------------------------------------------------------------------------------------------------------
# hd_rodrigues
# ------------------------------------------------------------------------------------------------------------------------------------
def test_rodrigues_edges():
    from oracle import smpl_ref
    lib, check = _lib()
    rng = np.random.RandomState(9)
    rows = [np.zeros(3)] * 5
    for mag in (1e-7, 1e-4, 1.0, np.pi, 2 * np.pi - 1e-3, 10.0):
        d = rng.normal(size=(6, 3))
        rows += list(d / np.linalg.norm(d, axis=1, keepdims=True) * mag)
        for i in range(3):                                           # axis-aligned, both signs
            rows += [np.eye(3)[i] * mag, -np.eye(3)[i] * mag]
    rows += [[-1e-8, 0.5, 0.2], [0.3, -1e-8, -1e-8], [-1e-8, -1e-8, 0.7], [-1e-8, 0.0, 0.0], [-1e-8, -1e-8, -1e-8]]
    rows += list(rng.normal(0, 1.0, size=(300, 3)))                  # M = 524: a ragged second block of 256
    th = np.asarray(rows, np.float32)
    M = th.shape[0]
    t = torch.from_numpy(th).cuda()
    outs = []
    for _ in range(2):
        R = _nan((M + 3, 9))
        check(lib.hd_rodrigues(_vp(t), _vp(R), M, _st()), 'hd_rodrigues')
        torch.cuda.synchronize()
        outs.append(R)
    assert _same_bits(outs[0], outs[1]) and _all_nan(outs[0][M:])
    R = outs[0][:M].reshape(M, 3, 3)
    assert torch.equal(R[:5], torch.eye(3, device='cuda').expand(5, 3, 3))              # theta = 0: exactly I
    # at theta = -1e-8 (1, 1, 1) the shifted angle is exactly 0 in float32 and the reference formula divides 0 by 0: NaN exactly
    # where the float32 restatement of the reference gives NaN
    with np.errstate(divide='ignore', invalid='ignore'):
        ref32 = smpl_ref.batch_rodrigues(th, np.float32)
    nan_ref = torch.from_numpy(np.isnan(ref32)).cuda()
    assert bool(nan_ref.any()) and torch.equal(torch.isnan(R), nan_ref)
    ok = ~nan_ref.reshape(M, 9).any(1)
    _bar('Rs', _abs(R[ok], sr.rodrigues(t.double())[ok]), RS_BAR, 'hd_rodrigues')


# ------------------------------------------------------------------------------------------------------------------------------------
# fused hd_smpl_forward: smpl_skin_kernel<8 | 32, 4 | runtime>
# ------------------------------------------------------------------------------------------------------------------------------------
def _forward_run(c, beta, theta, cam, N, mul, off, consts=None):
    """hd_smpl_forward into NaN buffers with one guard row past N * mul (NaN workspace too), twice; -> the first run's buffers."""
    lib, check = _lib()
    V, K = c.num_verts, c.num_kps
    outs = []
    for _ in range(2):
        o = {'verts': _nan((N * mul + 1, V, 3)), 'joints': _nan((N * mul + 1, K, 3)), 'Rs': _nan((N * mul + 1, 24, 3, 3)),
             'Jtr': _nan((N * mul + 1, 24, 3)), 'kps': _nan((N * mul + 1, K, 2))}
        wsb = int(lib.hd_smpl_workspace_bytes(N))
        ws = torch.full((wsb,), 255, dtype=torch.uint8, device='cuda')
        check(lib.hd_smpl_forward(C.byref(c.c if consts is None else consts), _vp(beta), beta.stride(0), _vp(theta), theta.stride(0),
                                  N, _vp(o['verts']), _vp(o['joints']), _vp(o['Rs']), _vp(o['Jtr']), _vp(cam), cam.stride(0),
                                  _vp(o['kps']), mul, off, _vp(ws), wsb, _st()), 'hd_smpl_forward')
        torch.cuda.synchronize()
        outs.append(o)
    rows = _slot_rows(N, mul, off)
    for k in outs[0]:
        assert _same_bits(outs[0][k], outs[1][k]), 'hd_smpl_forward rerun differs: ' + k
        assert not torch.isnan(outs[0][k][rows]).any() and _all_nan(_others(outs[0][k], rows)), k
    return {k: v[rows] for k, v in outs[0].items()}


def _check_forward(tag, c, beta, theta, cam, got, k64=None, bar=FWD_BAR):
    ref = sr.smpl_forward(_k64(c) if k64 is None else k64, beta, theta, cam)
    _bar('Rs', _abs(got['Rs'], ref['Rs']), RS_BAR, tag)
    for k in ('verts', 'joints', 'Jtr', 'kps'):
        _bar('forward ' + k, _rel(got[k], ref[k]), bar, tag)
    return ref


FUSED_CASES = ([('nnz4_v130', n) for n in (1, 7, 9, 4223, 4224, 4231)] + [('nnz8_v130', n) for n in (1, 7, 9, 4223, 4224, 4231)] +
               [('nnz24_v130', n) for n in (9, 4224)] + [('nnz8_v128', n) for n in (7, 4224)] +
               [('nnz4', 9), ('nnz4', 4223), ('nnz4', 4224), ('nnz8', 7), ('nnz8', 4231), ('nnz24', 9), ('nnz24', 4224)])


@pytest.mark.parametrize('name,N', FUSED_CASES)
def test_fused_forward(name, N):
    """N >= 4224 takes 32 poses per CTA (64.6 KB of dynamic shared memory), below 8; lbs_nnz 4 the unrolled instance, 8 and 24 the
    runtime one.  The pose-blend part of verts (N(0, 1e-3) posedirs: about 1e-3 of |verts|) is checked on its own against a twin of the
    model without posedirs."""
    c = _consts(name)
    mul, off = (2, 1) if N > 1000 else (3, 2)
    beta, theta, cam = _omega(N, seed=N)
    got = _forward_run(c, beta, theta, cam, N, mul, off)
    ref = _check_forward('%s N=%d' % (name, N), c, beta, theta, cam, got)
    # the same forward without posedirs: the difference is the pose-blend part of verts
    dirs0 = c.dirs.clone()
    dirs0[10:] = 0
    c0 = type(c.c).from_buffer_copy(c.c)
    c0.dirs = dirs0.data_ptr()
    got0 = _forward_run(c, beta, theta, cam, N, mul, off, consts=c0)
    k0 = _k64(c)
    k0['dirs'] = dirs0.double()
    ref0 = sr.smpl_forward(k0, beta, theta, cam)
    _bar('fused pose part', _rel(got['verts'].double() - got0['verts'].double(), ref['verts'] - ref0['verts']), POSE_PART_BAR,
         '%s N=%d' % (name, N))
    del ref, ref0, got, got0


# ------------------------------------------------------------------------------------------------------------------------------------
# staged path: blend GEMM -> hd_smpl_lbs | hd_smpl_lbs_tc -> hd_smpl_joints
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,N', [('nnz4', 300), ('nnz4', 2113), ('nnz8_v130', 257)])
def test_blend_gemm(name, N):
    """v_posed of SMPLConstants' bound tensor-core blend GEMM against float64 v_template + [beta | R - I] . dirs of the GPU's Rs;
    the pitch padding [3V, vp_ld) is exactly zero."""
    c = _consts(name, tc=True)
    V = c.num_verts
    beta, theta, cam = _omega(N, seed=N + 7)
    c.forward(beta, theta, cam)                                       # binds the per-N buffers
    coef, vpos, a12, rsw, op, a12t = c._tc_bufs[N]
    res = []
    for _ in range(2):
        for t in (coef[0], coef[1], vpos, a12, rsw):
            t.fill_(NAN)
        c.forward(beta, theta, cam)
        torch.cuda.synchronize()
        res.append(vpos.clone())
    assert _same_bits(res[0], res[1])
    assert torch.equal(vpos[:, 3 * V:], torch.zeros((N, c.vp_ld - 3 * V), device='cuda'))
    R = rsw.reshape(N, 24, 3, 3)
    k = _k64(c)
    _bar('blend v_posed', _rel(vpos[:, :3 * V], sr.blend(beta, R, k['v_template'], k['dirs'])), BLEND_BAR, '%s N=%d' % (name, N))


def _v_posed(N, V, ld, seed):
    """float32 [N, ld] rows of a v_posed-like field (|x| ~ 1), the pitch padding NaN."""
    vp = np.full((N, ld), np.nan, np.float32)
    vp[:, :3 * V] = np.random.RandomState(seed).uniform(-1, 1, size=(N, 3 * V))
    return torch.from_numpy(vp).cuda()


@pytest.mark.parametrize('name,N', [('nnz4', 5), ('nnz4', 300), ('nnz8', 300), ('nnz24', 37), ('nnz4_v130', 17), ('nnz8_v130', 33),
                                    ('nnz24_v130', 16)])
def test_lbs_cuda_core(name, N):
    """hd_smpl_lbs (smpl_lbs_kernel<16, 4 | runtime>) against float64 skinning of the same v_posed and the GPU's A12."""
    lib, check = _lib()
    c = _consts(name)
    V = c.num_verts
    beta, theta, _ = _omega(N, seed=N + 3)
    A12 = _pose_twice(c, beta, theta, N)['A12'][:N].contiguous()
    ld = 3 * V + 5
    vp = _v_posed(N, V, ld, seed=N)
    mul, off = 3, 1
    rows = _slot_rows(N, mul, off)
    outs = []
    for _ in range(2):
        verts = _nan((N * mul + 1, V, 3))
        check(lib.hd_smpl_lbs(C.byref(c.c), _vp(vp), ld, _vp(A12), _vp(verts), N, mul, off, _st()), 'hd_smpl_lbs')
        torch.cuda.synchronize()
        outs.append(verts)
    assert _same_bits(outs[0], outs[1]) and _all_nan(_others(outs[0], rows))
    ref = sr.skin(vp[:, :3 * V].reshape(N, V, 3), A12.reshape(N, 24, 3, 4), _k64(c)['weights'])
    _bar('lbs', _rel(outs[0][rows], ref), SKIN_BAR, '%s N=%d' % (name, N))


def _weights(V, seed):
    if V == 6890:
        return _k64(_consts('nnz4'))['weights'].float()
    rng = np.random.RandomState(seed)
    W = np.zeros((V, 24))
    for v in range(V):
        k = rng.randint(1, 5)
        W[v, rng.choice(24, size=k, replace=False)] = rng.rand(k) + 0.05
    return torch.from_numpy((W / W.sum(1, keepdims=True)).astype(np.float32)).cuda()


LBS_TC_CASES = ([(n, 6890, i % 2, 1 + i % 2) for i, n in enumerate((1, 15, 16, 17, 2112, 2113, 16 * 133 + 5, 16 * 264 + 3))] +
                [(n, V, (i + j) % 2, 1 + (i + j + 1) % 2) for j, V in enumerate((128, 130, 2)) for i, n in enumerate((1, 17, 2113, 4227))])


@pytest.mark.parametrize('N,V,pad,off', LBS_TC_CASES)
def test_lbs_tensor_core(N, V, pad, off):
    """hd_smpl_lbs_tc: runs (16-pose batches) below and above the SM count, so a CTA takes a second batch and the v_posed prefetch
    crosses a run boundary; ragged last batches and vertex tiles; vp_ld at roundup4(3V) and 4 more; three output slots, odd ones only
    8-byte aligned.  Against float64 skinning of the same v_posed, the GPU's A12 and the float32 weights."""
    lib, check = _lib()
    c = _consts('nnz4')
    beta, theta, _ = _omega(N, seed=N + 11)
    o = _pose_twice(c, beta, theta, N)
    A12 = o['A12'][:N]
    W = _weights(V, seed=V)
    wd = torch.zeros(((V + 127) // 128 * 128, 32), device='cuda')
    wd[:V, :24] = W
    w_hi = wd.half()
    w_lo = (wd - w_hi.float()).half()
    ld = (3 * V + 3) // 4 * 4 + 4 * pad
    vp = _v_posed(N, V, ld, seed=N + V)
    mul = 3
    rows = _slot_rows(N, mul, off)
    outs = []
    for _ in range(2):
        verts = _nan((N * mul + 1, V, 3))
        check(lib.hd_smpl_lbs_tc(_vp(w_hi), _vp(w_lo), _vp(o['a12t_hi']), _vp(o['a12t_lo']), _vp(vp), ld, _vp(verts), N, V, mul, off,
                                 _st()), 'hd_smpl_lbs_tc')
        torch.cuda.synchronize()
        outs.append(verts)
    assert _same_bits(outs[0], outs[1])
    assert not torch.isnan(outs[0][rows]).any() and _all_nan(_others(outs[0], rows))
    ref = sr.skin(vp[:, :3 * V].reshape(N, V, 3), A12.reshape(N, 24, 3, 4), W)
    _bar('lbs_tc', _rel(outs[0][rows], ref), SKIN_TC_BAR, 'N=%d V=%d pad=%d off=%d' % (N, V, pad, off))


@pytest.mark.parametrize('name,jt', [('nnz4', 'cocoplus'), ('nnz4', 'lsp'), ('nnz24_v130', 'cocoplus'), ('nokp', 'cocoplus')])
def test_joints_kernel(name, jt):
    """hd_smpl_joints: the keypoint regression of the kernel's input verts against float64; kps bit for bit s * (x + t) in float32 of
    the kernel's own joints (an add, then a multiply: nothing to contract).  A model without keypoints writes nothing."""
    lib, check = _lib()
    c = _consts(name, joint_type=jt)
    V, K = c.num_verts, c.num_kps
    N, mul, off = 37, 3, 2
    rows = _slot_rows(N, mul, off)
    _, _, cam = _omega(N, seed=12)
    verts = _nan((N * mul, V, 3))                      # slots other than `off` are NaN: reading them would poison the sums
    verts[rows] = torch.from_numpy(np.random.RandomState(13).uniform(-1, 1, size=(N, V, 3)).astype(np.float32)).cuda()
    outs = []
    for _ in range(2):
        joints, kps = _nan((N * mul + 1, max(K, 1), 3)), _nan((N * mul + 1, max(K, 1), 2))
        check(lib.hd_smpl_joints(C.byref(c.c), _vp(verts), _vp(cam), cam.stride(0), _vp(joints), _vp(kps), N, mul, off, _st()),
              'hd_smpl_joints')
        torch.cuda.synchronize()
        outs.append((joints, kps))
    joints, kps = outs[0]
    assert _same_bits(joints, outs[1][0]) and _same_bits(kps, outs[1][1])
    if K == 0:
        assert _all_nan(joints) and _all_nan(kps)
        return
    assert _all_nan(_others(joints, rows)) and _all_nan(_others(kps, rows))
    j = joints[rows]
    _bar('joints', _rel(j, sr.regress(verts[rows], _k64(c)['regressor'])), JOINTS_BAR, '%s %s' % (name, jt))
    want = (j[..., :2] + cam[:, None, 1:3]) * cam[:, None, 0:1]
    assert _same_bits(kps[rows], want)


@pytest.mark.parametrize('name,N,lbs_tc', [('nnz4', 300, False), ('nnz8', 257, False), ('nnz4', 2113, True), ('nnz24', 2112, True)])
def test_staged_against_fused_and_float64(name, N, lbs_tc):
    """SMPLConstants' staged path (pose, blend GEMM, CUDA-core or tensor-core skinning, joints) against the fused kernel and float64."""
    from human_dynamics_b200.smpl import SMPLConstants
    cf = _consts(name)
    ct = _consts(name, tc=True)
    ct.lbs_tc_min_batch = 0 if lbs_tc else 1 << 30
    ct._tc_bufs.clear()
    beta, theta, cam = _omega(N, seed=N + 5)
    staged = {k: v.clone() for k, v in ct.forward(beta, theta, cam).items()}
    assert ct._tc_bufs[N][5] is not None if lbs_tc else ct._tc_bufs[N][5] is None
    fused = cf.forward(beta, theta, cam)
    torch.cuda.synchronize()
    tag = '%s N=%d lbs_tc=%d' % (name, N, lbs_tc)
    _check_forward('staged ' + tag, ct, beta, theta, cam, staged)
    for k in ('verts', 'joints', 'Jtr', 'kps'):
        _bar('staged vs fused ' + k, _rel(staged[k], fused[k]), FWD_BAR, tag)
    assert _same_bits(staged['Rs'], fused['Rs'])                 # the same pose kernel
    ct.lbs_tc_min_batch = 2112
    ct._tc_bufs.clear()


# ------------------------------------------------------------------------------------------------------------------------------------
# hd_orth_proj
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,P', [(1, 1), (7, 25), (13, 37), (300, 14)])
def test_orth_proj(N, P):
    lib, check = _lib()
    rng = np.random.RandomState(N * P)
    X = torch.from_numpy(rng.normal(0, 0.5, size=(N, P, 3)).astype(np.float32)).cuda()
    cam = torch.from_numpy(np.concatenate([rng.uniform(0.5, 1.5, (N, 1)), rng.uniform(-0.3, 0.3, (N, 2))], 1).astype(np.float32)).cuda()
    outs = []
    for _ in range(2):
        out = _nan((N * P * 2 + 7,))
        check(lib.hd_orth_proj(_vp(X), _vp(cam), _vp(out), N, P, _st()), 'hd_orth_proj')
        torch.cuda.synchronize()
        outs.append(out)
    assert _same_bits(outs[0], outs[1]) and _all_nan(outs[0][N * P * 2:])
    want = (X[..., :2] + cam[:, None, 1:3]) * cam[:, None, 0:1]
    assert _same_bits(outs[0][:N * P * 2].reshape(N, P, 2), want)


# ------------------------------------------------------------------------------------------------------------------------------------
# per-device shared-memory opt-in
# ------------------------------------------------------------------------------------------------------------------------------------
def test_opt_in_per_device():
    """The kernels above 48 KB of dynamic shared memory (smpl_skin_kernel<32, *>, smpl_lbs_backward_kernel, wgrad_kernel) opt in per
    device: in one process, the first launch on a second GPU must not skip it.  Each device's results equal device 0's bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs in one process')
    from human_dynamics_b200.smpl import SMPLConstants
    from human_dynamics_b200._lib import lib, check
    N = 4224
    model = _model('nnz4')
    res = []
    for d in (0, 1):
        with torch.cuda.device(d):
            dev = torch.device('cuda', d)
            beta, theta, _ = (t.to(dev) for t in _omega(N, seed=50))
            fwd = SMPLConstants(model, tc=False, device=dev).forward(beta, theta)
            ct = SMPLConstants(model, tc=True, device=dev)
            dverts = torch.from_numpy(np.random.RandomState(51).normal(size=(64, 6890, 3)).astype(np.float32)).to(dev)
            dbeta, dtheta = ct.backward(beta[:64].contiguous(), theta[:64].contiguous(), dverts=dverts)
            rng = np.random.RandomState(52)
            x = torch.from_numpy(rng.normal(size=(2, 29, 29, 64)).astype(np.float32)).to(dev)
            dy = torch.from_numpy(rng.normal(size=(2, 29, 29, 64)).astype(np.float32)).to(dev)
            dw = torch.empty((9 * 64, 64), device=dev)
            wsb = lib.hd_conv_wgrad_workspace_bytes(2 * 29 * 29, 9 * 64, 64, 0)
            ws = torch.empty(max(16, wsb), dtype=torch.uint8, device=dev)
            check(lib.hd_conv_wgrad(_vp(x), 64, 2, 29, 29, 64, 29, 29, 3, 3, 1, 1, 1, None, None, _vp(dy), 64, 64, _vp(dw), None,
                                    _vp(ws), ws.numel(), _st()), 'hd_conv_wgrad')
            torch.cuda.synchronize(dev)
            res.append({'verts': fwd['verts'].cpu(), 'joints': fwd['joints'].cpu(), 'dbeta': dbeta.cpu(), 'dtheta': dtheta.cpu(),
                        'dw': dw.cpu()})
    for k in res[0]:
        assert _same_bits(res[0][k], res[1][k]), k
