"""Host-side wiring of the ResNet layer plan checked WITHOUT a GPU: device allocations and library calls are stubbed, the descriptors
the plan fills are real.  Catches plan-logic mistakes (buffer roles, dead outputs, epilogue subsampling, launch counts) on the CPU."""
import ctypes as C

import numpy as np
import pytest
import torch


@pytest.fixture
def fake_device(monkeypatch):
    from human_dynamics_b200 import nets

    class FakeLib(object):
        def __getattr__(self, name):
            return lambda *a, **k: 0
    monkeypatch.setattr(nets, 'lib', FakeLib())
    monkeypatch.setattr(nets, '_dev', lambda a, device, dtype=np.float32: torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)))
    monkeypatch.setattr(torch.Tensor, 'to', lambda self, *a, **k: self)
    e, z = torch.empty, torch.zeros
    monkeypatch.setattr(torch, 'empty', lambda *a, **k: e(*a, **{kk: v for kk, v in k.items() if kk != 'device'}))
    monkeypatch.setattr(torch, 'zeros', lambda *a, **k: z(*a, **{kk: v for kk, v in k.items() if kk != 'device'}))
    return nets


def _convs(plan):
    return [o for o in plan.ops if getattr(o, 'd', None) is not None]


def test_resnet_plan_and_stage_wiring(fake_device):
    nets = fake_device
    from human_dynamics_b200 import synthetic
    packed = nets.PackedResNet(synthetic.make_resnet_weights(seed=1), 'cpu', tc='auto')
    assert len(packed.units) == 16
    plan = nets.ResNetPlan(packed, 2, 64, 'auto')
    assert plan.split and plan.pool_f32_dead
    convs = _convs(plan)
    assert len(convs) == 52                                            # 16 units x 3 + 4 shortcut convs (conv1 of the root is separate)
    subs = [o for o in plan.ops if isinstance(o, nets.SubsampleOp)]
    epis = [(o.d.Cout, o.d.Ho, o.d.out_subsample) for o in convs if o.d.out_subsample > 1]
    # the units in front of the three strided identity units write x[:, ::2, ::2] themselves (maps 16 -> 8 -> 4 -> 2 at size 64)
    assert (len(subs), epis) == (0, [(256, 16, 2), (512, 8, 2), (1024, 4, 2)])
    assert sum(1 for o in convs if not o.d.out and o.d.res) == 3       # fp32 outputs in front of a conv shortcut are never written
    assert plan.num_launches == 3 + len(plan.ops) + 1
    for o in convs:
        d = o.d
        assert d.in_hi and d.in_lo and not d.in_ and d.impl == 3       # every trunk conv reads a pre-split pair
        if d.res:
            assert (d.res_stride, d.res_H, d.res_W, d.res_ld) == (1, d.Ho, d.Wo, d.Cout)   # residual rows == output rows (TMA slabs)
        if d.out_subsample > 1:
            assert d.out and not d.tmap_out and d.tmap_out_hi and d.res                      # dense subsample: no fp32 TMA store
    # the residual of a strided identity unit is the dense subsampled buffer
    strided = [o for o in convs if o.d.KH == 1 and o.d.res and o.d.res == plan.bufS.data_ptr() and o.d.Cout in (256, 512, 1024)]
    assert len(strided) >= 3

    # cut in front of block 1's strided identity unit: stage A writes its fp32 output, and stage B subsamples it in one hd_subsample
    # pass that reads the stage input
    nxt = packed.units[2]
    pa = nets.ResNetPlan(packed, 2, 64, 'auto', units=(0, 2), root=True, tail=False, next_pre=nxt['pre'], next_has_shortcut=False)
    pb = nets.ResNetPlan(packed, 2, 64, 'auto', units=(2, 16), root=False)
    assert _convs(pa)[-1].d.out and not any(o.d.out_subsample > 1 for o in _convs(pa))
    assert isinstance(pb.ops[0], nets.SubsampleOp) and (pb.ops[0], 'res', 2) in pb.in_refs
    assert sum(isinstance(o, nets.SubsampleOp) for o in pb.ops) == 1
    assert [o.d.out_subsample for o in _convs(pb) if o.d.out_subsample > 1] == [2, 2]
    assert _convs(pb)[2].d.res == pb.bufS.data_ptr()                  # the strided unit's conv3 reads the dense copy


def test_root_conv1_choice(fake_device):
    """bind_root_conv1: the fp16 impls read padded fp16 planes at even sizes and gather the fp32 images at odd ones; 'simt' has no
    conv1 op (hd_conv1_7x7s2)."""
    nets = fake_device
    from human_dynamics_b200 import _lib, synthetic
    w = synthetic.make_resnet_weights(seed=1)
    packed = nets.PackedResNet(w, 'cpu', tc='auto')
    even = nets.ResNetPlan(packed, 2, 64, 'auto')
    assert even.planes is not None and even.conv1_op.d.flags & _lib.HD_CONV_INPUT_PLANES
    assert even.conv1_op.d.out == even.root_buf.data_ptr() and even.num_launches == 3 + len(even.ops) + 1
    odd = nets.ResNetPlan(packed, 2, 63, 'auto')
    d = odd.conv1_op.d
    assert odd.planes is None and d.impl == _lib.HD_IMPL_TC_3XF16 and not d.flags & _lib.HD_CONV_INPUT_PLANES
    assert (d.KH, d.KW, d.Cin, d.in_ld, d.H) == (7, 7, 3, 3, 63) and d.out == odd.root_buf.data_ptr()
    assert odd.num_launches == 2 + len(odd.ops) + 1
    simt = nets.ResNetPlan(nets.PackedResNet(w, 'cpu', tc=False), 2, 64, 'simt')
    assert simt.planes is None and simt.conv1_op is None and simt.num_launches == 2 + len(simt.ops) + 1


def test_stage_plans_keep_the_pairs_inside_a_stage(fake_device):
    """The engine cuts the trunk after unit 7 (block 2): every (unit, strided identity unit) pair lies inside one stage, so neither
    stage needs an hd_subsample pass; the stage-A output in front of block 3's conv shortcut has no fp32 copy."""
    nets = fake_device
    from human_dynamics_b200 import synthetic
    packed = nets.PackedResNet(synthetic.make_resnet_weights(seed=1), 'cpu', tc='auto')
    nxt = packed.units[7]
    pa = nets.ResNetPlan(packed, 2, 64, 'auto', units=(0, 7), root=True, tail=False, next_pre=nxt['pre'], next_has_shortcut='shortcut' in nxt)
    pb = nets.ResNetPlan(packed, 2, 64, 'auto', units=(7, 16), root=False, tail=True)
    assert not any(isinstance(o, nets.SubsampleOp) for o in pa.ops + pb.ops)
    assert sum(1 for o in _convs(pa) + _convs(pb) if o.d.out_subsample > 1) == 3
    last_a = _convs(pa)[-1].d
    assert not last_a.out and last_a.out_hi and last_a.post2_relu == 1
    assert (pb.in_hw, pb.in_depth) == (pa.out_hw, pa.out_depth) == (4, 512)


def test_fmovie_and_ief_plan_wiring(fake_device):
    """f_movie fast path: per block GN+ReLU+split -> conv (k=3 over T, pad 1) -> GN+ReLU+split -> conv + residual; IEF fast path: phi split
    once, per head one hoisted phi.W1 GEMM, per stage fc1-theta / fc2 (tensor cores) / fc3; delta heads write into the [N, D, 85] stack."""
    nets = fake_device
    from human_dynamics_b200 import synthetic
    w = synthetic.make_synthetic_weights(seed=1)
    B, T = 2, 20
    fm = nets.FMoviePlan(nets.PackedFMovie(w, 'cpu', 3, tc='auto'), B, T, 'auto')
    x = torch.zeros((B, T, 2048))
    fm._bind(x)
    assert [s[0] for s in fm.steps] == ['gns', 'conv'] * 6 and fm.num_launches == 12
    convs = [s[1].d for s in fm.steps if s[0] == 'conv']
    for i, d in enumerate(convs):
        assert (d.n_img, d.H, d.W, d.KH, d.KW, d.pad_t, d.pad_l, d.Ho, d.Wo, d.Cin, d.Cout) == (B, T, 1, 3, 1, 1, 0, T, 1, 2048, 2048)
        assert d.in_hi == fm.act[0].data_ptr() and d.impl == 3 and d.post_shift and not d.post_relu
        assert bool(d.res) == (i % 2 == 1)                                   # the block's second conv adds the block input
    assert convs[1].res == x.data_ptr() and convs[3].res == convs[1].out and convs[5].res == convs[3].out
    assert fm.out.data_ptr() == convs[5].out

    N = B * T
    ief = nets.IEFPlan(nets.PackedIEF(w, 'cpu', tc='auto'), N, 3, None, 'auto')
    assert ief.fast and ief.delta_keys == [-5, 5] and ief.num_launches == 33
    phi, theta0 = torch.zeros((N, 2048)), torch.zeros((N, 85))
    ief._bind(phi, theta0)
    kinds = [op[0] for op in ief.main_ops]
    assert kinds == ['conv'] + ['fc1t', 'conv', 'fc3'] * 3
    # stage 0 starts from theta0, later stages from the running theta; the delta heads run in place on columns 3:75 of their slot
    assert ief.main_ops[1][1].data_ptr() == theta0.data_ptr() and ief.main_ops[4][1].data_ptr() == ief.theta.data_ptr()
    for i, dt in enumerate(ief.delta_keys):
        ops = ief.delta_ops[dt]
        view = ops[1][1]
        assert view.data_ptr() == ief.delta_all.data_ptr() + (i * 85 + 3) * 4 and ops[1][2] == 2 * 85 and ops[3][4] == 2 * 85
        assert ops[3][5].d == 72
    assert ief.main_ops[3][5].d == 85
    assert all(op[4] is None for op in ief.main_ops if op[0] == 'fc1t')             # no fp32 h1
    assert {op[6].data_ptr() for op in ief.main_ops if op[0] == 'fc3'} == {ief.h2.data_ptr()}

    # keep=True (training): the same launches over per-block buffers of their own, and `saved` = [(block input, conv1 output)], in both
    # f_movie branches (T = 25: T*64 > 1280, GroupNorm statistics + prologue)
    def fields(d):
        return tuple(getattr(d, f) for f, t in d._fields_ if t is not C.c_void_p)
    for TT in (T, 25):
        fm = nets.FMoviePlan(nets.PackedFMovie(w, 'cpu', 3, tc='auto'), B, TT, 'auto')
        fk = nets.FMoviePlan(fm.p, B, TT, 'auto', keep=True)
        x = torch.zeros((B, TT, 2048))
        fm._bind(x)
        fk._bind(x)
        assert [s[0] for s in fk.steps] == [s[0] for s in fm.steps] == (['gns', 'conv'] if TT == T else ['gn', 'conv']) * 6
        ck, cf = [s[1].d for s in fk.steps if s[0] == 'conv'], [s[1].d for s in fm.steps if s[0] == 'conv']
        assert [fields(d) for d in ck] == [fields(d) for d in cf]
        assert len({d.out for d in ck} | {x.data_ptr()}) == 7                          # three conv1 outputs, three block outputs
        assert [(a.data_ptr(), m.data_ptr()) for a, m in fk.saved] == [(x.data_ptr(), ck[0].out), (ck[1].out, ck[2].out),
                                                                        (ck[3].out, ck[4].out)]
        assert [d.res for d in ck[1::2]] == [x.data_ptr(), ck[1].out, ck[3].out] and fk.out.data_ptr() == ck[5].out
        if TT == 25:
            assert [d.in_ for d in ck] == [x.data_ptr(), ck[0].out, ck[1].out, ck[2].out, ck[3].out, ck[4].out]
    # IEF keep=True: per stage an fp32 h1 and an h2 of its own; stages 0 and 1 write separate outputs that feed the next stage; the delta
    # heads write (N, 85) outputs of their own
    ik = nets.IEFPlan(ief.p, N, 3, None, 'auto', keep=True)
    ik._bind(phi, theta0)
    assert ik.num_launches == ief.num_launches and not hasattr(ik, 'delta_all')
    for j, (ops, d) in enumerate([(ik.main_ops, 85)] + [(ik.delta_ops[dt], 72) for dt in ik.delta_keys]):
        assert [op[0] for op in ops] == kinds
        h1, h2, out0, out1 = ik.saved[j]
        assert h1.shape == h2.shape == (3, N, 1024) and out0.shape == out1.shape == (N, d)
        fc1t, fc2, fc3 = ops[1::3], ops[2::3], ops[3::3]
        assert [op[4].data_ptr() for op in fc1t] == [h1[s].data_ptr() for s in range(3)]
        assert [op[1].d.out for op in fc2] == [op[6].data_ptr() for op in fc3] == [h2[s].data_ptr() for s in range(3)]
        state = ik.theta if j == 0 else ik.delta_out[ik.delta_keys[j - 1]][:, 3:75]
        assert [op[3].data_ptr() for op in fc3] == [out0.data_ptr(), out1.data_ptr(), state.data_ptr()]
        assert [op[1].data_ptr() for op in fc1t] == [op[1].data_ptr() for op in fc3]
        assert [op[1].data_ptr() for op in fc1t[1:]] == [out0.data_ptr(), out1.data_ptr()]
        assert [op[2] for op in fc1t] == [op[2] for op in fc3] == [85, d, d] and [op[4] for op in fc3] == [d, d, 85]
    assert ik.main_ops[1][1].data_ptr() == theta0.data_ptr()
    assert all(ik.delta_out[dt].shape == (N, 85) and ik.delta_out[dt].is_contiguous() for dt in ik.delta_keys)
    assert len({t.data_ptr() for s in ik.saved for t in s}) == 4 * 3


@pytest.mark.parametrize('dense', [False, True])
def test_smpl_constant_packing_is_exact(smpl_model, smpl_model_dense, dense):
    """SMPLConstants (the device layout of the SMPL pickle, built here on the CPU without the tensor-core packing): the integer tables
    -- kinematic parents, ELL joint ids of the skinning weights, CSC vertex ids of the keypoint regressor -- and the weights they carry
    reproduce the pickle's dense matrices exactly; the pre-composed joint regressor equals batch_smpl.py:110-118 evaluated in float64."""
    from human_dynamics_b200.smpl import SMPLConstants
    m = smpl_model_dense if dense else smpl_model
    c = SMPLConstants(m, device='cpu', tc=False)
    V = m['v_template'].shape[0]
    assert c.num_verts == V == 6890 and c.num_kps == m['cocoplus_regressor'].shape[0]
    # kintree_table[0] is stored as uint32 with 4294967295 for the root; batch_smpl.py:66 casts with astype(np.int32) -> -1
    assert m['kintree_table'].dtype == np.uint32 and int(m['kintree_table'][0, 0]) == 4294967295
    assert c.parents.dtype == np.int32 and c.parents.tolist() == [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]
    assert [c.c.parents[i] for i in range(24)] == c.parents.tolist()
    # ELL skinning weights -> dense (V, 24)
    W = np.asarray(m['weights'], np.float64)
    idx, w = c.lbs_idx.numpy(), c.lbs_w.numpy()
    assert idx.shape == w.shape == (V, c.lbs_nnz) and c.lbs_nnz == (24 if dense else 4) and idx.dtype == np.int32
    rec = np.zeros((V, 24), np.float32)
    np.add.at(rec, (np.repeat(np.arange(V), c.lbs_nnz), idx.reshape(-1)), w.reshape(-1))
    assert np.array_equal(rec, W.astype(np.float32))
    nz = w != 0
    assert np.all(idx[~nz] == 0)                                               # padding entries: joint 0 with weight 0
    for v in (0, 17, V - 1):
        assert list(idx[v][nz[v]]) == sorted(idx[v][nz[v]])                    # fixed (ascending joint) summation order
    # CSC keypoint regressor -> dense (K, V)
    K = c.num_kps
    ptr, vid, kw = c.kp_ptr.numpy(), c.kp_vidx.numpy(), c.kp_w.numpy()
    assert ptr[0] == 0 and np.all(np.diff(ptr) > 0) and ptr[-1] == len(vid) == len(kw) == c.c.kp_nnz_total
    rec = np.zeros((K, V), np.float32)
    for k in range(K):
        rec[k, vid[ptr[k]:ptr[k + 1]]] = kw[ptr[k]:ptr[k + 1]]
        assert np.all(np.diff(vid[ptr[k]:ptr[k + 1]]) > 0)
    assert np.array_equal(rec, np.asarray(m['cocoplus_regressor'], np.float32))
    lsp = SMPLConstants(m, joint_type='lsp', device='cpu', tc=False)
    assert lsp.num_kps == 14 and lsp.c.kp_nnz_total == int(ptr[14])          # batch_smpl.py:81-82: the first 14 columns
    with pytest.raises(ValueError):
        SMPLConstants(m, joint_type='coco', device='cpu', tc=False)           # the reference prints 'BAD!!' and drops into ipdb
    # blend basis rows: 10 shape rows then 207 pose rows, flattened like batch_smpl.py:45-48,60-63
    dirs = c.dirs.numpy()
    assert dirs.shape == (217, V * 3)
    assert np.array_equal(dirs[:10], np.reshape(m['shapedirs'], [-1, 10]).T.astype(np.float32))
    assert np.array_equal(dirs[10:], np.reshape(m['posedirs'], [-1, 207]).T.astype(np.float32))
    # J(beta) = (beta . shapedirs + v_template) . J_regressor, pre-composed
    beta = np.random.RandomState(0).normal(0, 2, size=(5, 10))
    v_shaped = (beta @ np.reshape(m['shapedirs'], [-1, 10]).T).reshape(5, V, 3) + m['v_template']
    J_ref = np.stack([v_shaped[:, :, k] @ np.asarray(m['J_regressor']).T for k in range(3)], axis=2)
    J = c.J_template.numpy().astype(np.float64).reshape(1, 24, 3) + (beta @ c.J_shapedirs.numpy().astype(np.float64)).reshape(5, 24, 3)
    assert np.abs(J - J_ref).max() < 1e-6


def test_fold_bn_in_float64(fake_device):
    """BatchNorm folded in float64; the conv1 plane width (the packed layouts and splits are checked on the GPU, test_gpu_nets.py)."""
    nets = fake_device
    assert nets.PackedConv1Planes.plane_width(224) == 232 and nets.PackedConv1Planes.plane_width(64) == 72
    rng = np.random.RandomState(3)
    wd = {'p/gamma': rng.uniform(0.5, 1.5, 8).astype(np.float32), 'p/beta': rng.normal(size=8).astype(np.float32),
          'p/moving_mean': rng.normal(size=8).astype(np.float32), 'p/moving_variance': rng.uniform(0.5, 1.5, 8).astype(np.float32)}
    s, b = nets.fold_bn(wd, 'p')
    x = rng.normal(size=(5, 8))
    ref = wd['p/gamma'] * (x - wd['p/moving_mean']) / np.sqrt(wd['p/moving_variance'].astype(np.float64) + 1e-5) + wd['p/beta']
    assert s.dtype == b.dtype == np.float32 and np.abs(x * s + b - ref).max() < 1e-6


@pytest.mark.parametrize('dense,lsp', [(False, False), (True, False), (False, True)])
def test_c_smpl_pack_equals_python_packing(smpl_model, smpl_model_dense, dense, lsp):
    """hd_smpl_pack (csrc/smpl_pack.cu, host-only C: what a C consumer calls to fill hd_smpl_consts) against the Python packing of
    SMPLConstants: integer tables and plain casts bit for bit, the pre-composed joint regressor to float32 rounding."""
    import ctypes as C
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.smpl import SMPLConstants
    m = smpl_model_dense if dense else smpl_model
    ref = SMPLConstants(m, joint_type='lsp' if lsp else 'cocoplus', device='cpu', tc=False)
    V = m['v_template'].shape[0]
    kreg = np.ascontiguousarray(np.asarray(m['cocoplus_regressor'], np.float64)[:14] if lsp else np.asarray(m['cocoplus_regressor'], np.float64))
    K = kreg.shape[0]
    f64 = lambda a: np.ascontiguousarray(a, np.float64)              # noqa: E731
    vt, sd, pd, jr, w = f64(m['v_template']), f64(m['shapedirs']), f64(m['posedirs']), f64(m['J_regressor']), f64(m['weights'])
    kin = np.ascontiguousarray(m['kintree_table'][0], np.uint32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)                     # noqa: E731
    nnz, tot = C.c_int(), C.c_int()
    assert _lib.lib.hd_smpl_pack_sizes(V, K, ptr(w), ptr(kreg), C.byref(nnz), C.byref(tot)) == 0
    assert (nnz.value, tot.value) == (ref.lbs_nnz, ref.c.kp_nnz_total)
    out = {'vt': np.empty(V * 3, np.float32), 'dirs': np.empty((217, V * 3), np.float32), 'Jt': np.empty(72, np.float32),
           'Js': np.empty((10, 72), np.float32), 'idx': np.empty((V, nnz.value), np.int32), 'w': np.empty((V, nnz.value), np.float32),
           'kp_ptr': np.empty(K + 1, np.int32), 'kp_vidx': np.empty(tot.value, np.int32), 'kp_w': np.empty(tot.value, np.float32),
           'parents': np.empty(24, np.int32)}
    rc = _lib.lib.hd_smpl_pack(V, K, ptr(vt), ptr(sd), ptr(pd), ptr(jr), ptr(w), ptr(kreg), ptr(kin), ptr(out['vt']), ptr(out['dirs']),
                               ptr(out['Jt']), ptr(out['Js']), ptr(out['idx']), ptr(out['w']), nnz.value, ptr(out['kp_ptr']),
                               ptr(out['kp_vidx']), ptr(out['kp_w']), ptr(out['parents']))
    assert rc == 0, _lib.lib.hd_last_error()
    assert np.array_equal(out['vt'], ref.v_template.numpy()) and np.array_equal(out['dirs'], ref.dirs.numpy())
    assert np.array_equal(out['idx'], ref.lbs_idx.numpy()) and np.array_equal(out['w'], ref.lbs_w.numpy())
    assert np.array_equal(out['kp_ptr'], ref.kp_ptr.numpy()) and np.array_equal(out['kp_vidx'], ref.kp_vidx.numpy())
    assert np.array_equal(out['kp_w'], ref.kp_w.numpy()) and out['parents'].tolist() == ref.parents.tolist()
    assert np.allclose(out['Jt'], ref.J_template.numpy(), rtol=3e-7, atol=1e-9)
    assert np.allclose(out['Js'], ref.J_shapedirs.numpy(), rtol=3e-7, atol=1e-9)
    assert _lib.lib.hd_smpl_pack(V, K, ptr(vt), ptr(sd), ptr(pd), ptr(jr), ptr(w), ptr(kreg), ptr(kin), ptr(out['vt']), ptr(out['dirs']),
                                 ptr(out['Jt']), ptr(out['Js']), ptr(out['idx']), ptr(out['w']), nnz.value + 4, ptr(out['kp_ptr']),
                                 ptr(out['kp_vidx']), ptr(out['kp_w']), ptr(out['parents'])) == 1       # wrong lbs_nnz: HD_ERR_INVALID
