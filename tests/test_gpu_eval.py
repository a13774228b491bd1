"""GPU: the evaluation kernels (csrc/eval.cu) and human_dynamics_b200.evaluate.Evaluator against the float64 oracle
(oracle/eval_ref.py), their determinism and launch structure, and src.evaluation.eval.main end to end on tfrecords."""
import json
import os
import pickle

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
    pytest.skip('needs a CUDA device', allow_module_level=True)

from human_dynamics_b200 import _lib                     # noqa: E402
from human_dynamics_b200.evaluate import Evaluator        # noqa: E402
from human_dynamics_b200.smpl import SMPLConstants        # noqa: E402
from oracle import eval_cases, eval_ref                   # noqa: E402

FRAME_KEYS = ('accel', 'kp', 'kp_pa', 'kp_pck', 'accel_error', 'joints', 'joints_pa')


@pytest.fixture(scope='module')
def consts(smpl_model):
    return SMPLConstants(smpl_model)


def _lens(N):
    if N <= 3:
        return [N]
    if N == 777:
        return [1, 2, 3, 50, 721]
    return [N // 40 + (1 if i < N % 40 else 0) for i in range(40)]


def _close(got, want, rtol, key):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (key, got.shape, want.shape)
    assert np.array_equal(np.isnan(got), np.isnan(want)), key
    ok = ~np.isnan(want)
    if key == 'kp_pck':
        assert np.array_equal(got[ok], want[ok]), key
    else:
        err = np.abs(got[ok] - want[ok]) / np.maximum(np.abs(want[ok]), 1e-12)
        assert err.size == 0 or err.max() <= rtol, (key, err.max())


@pytest.mark.parametrize('K', [14, 19, 25])
@pytest.mark.parametrize('N', [1, 2, 3, 777, 35000])
def test_frames_match_oracle(N, K):
    """Every per-frame metric of every tube against the float64 oracle on the same float32 inputs, 1e-10 relative; PCK and the NaN
    positions exact.  Tubes of length 1, 2 and 3 and the edge-case frames are part of the split."""
    tubes = eval_ref.make_eval_tubes(_lens(N), K=K, seed=N + K)
    ev = Evaluator()
    for has_3d in (True, False):
        got = ev.errors_many(tubes, img_size=224, has_3d=has_3d, min_visible=6)
        for t, g in zip(tubes, got):
            want = eval_ref.compute_errors_batched(img_size=224, has_3d=has_3d, min_visible=6, **t)
            assert sorted(g) == sorted(want)
            for k in FRAME_KEYS:
                if k in want:
                    _close(g[k], want[k], 1e-10, k)
            if has_3d:
                assert g['pose'] == g['shape'] == g['mesh_posed'] == g['mesh_tpose'] == -1


def test_meshes_match_oracle(smpl_model, consts):
    """mesh_posed / mesh_tpose (float32 SMPL on the device, rotation matrices through hd_rot2aa) against the float64 oracle: 1e-6 m,
    and 1e-5 m for the frame whose rotations lie within 1e-3 rad of pi (there the float32 axis-angle of hd_rot2aa carries ~1e-6 rad
    of rounding, measured 4e-6 m of mesh distance on an H100)."""
    tubes = eval_ref.make_eval_tubes([1, 2, 3, 9, 30], seed=5)
    got = Evaluator(consts, mesh_chunk=16).errors_many(tubes, has_3d=True, compute_mesh=True)
    for t, g in zip(tubes, got):
        want = eval_ref.compute_errors_batched(has_3d=True, compute_mesh=True, smpl_model=smpl_model, **t)
        vis = np.sum(t['kps_gt'][:, :14, 2], axis=1) > 6
        cos = (np.trace(t['poses_pred'].astype(np.float64), axis1=2, axis2=3) - 1) / 2
        tol = np.where((cos < np.cos(np.pi - 1e-2)).any(axis=1), 1e-5, 1e-6)[vis]
        for k in ('mesh_posed', 'mesh_tpose'):
            assert g[k].shape == want[k].shape, k
            assert (np.abs(g[k] - want[k]) < tol).all(), (k, np.abs(g[k] - want[k]))
        for k in FRAME_KEYS:
            _close(g[k], want[k], 1e-10, k)
    assert sum((np.trace(t['poses_pred'], axis1=2, axis2=3) < -0.99).any() for t in tubes) == 1   # the near-pi frame is in the split


@pytest.mark.parametrize('dense', [False, True])
def test_tpose_closed_form_matches_smpl_forward(dense, smpl_model, smpl_model_dense):
    """hd_eval_mesh_tpose against hd_smpl_forward at theta = 0 + hd_eval_verts_error, on the sparse and the dense-weight model."""
    c = SMPLConstants(smpl_model_dense if dense else smpl_model)
    rng = np.random.RandomState(1)
    N = 64
    bg = torch.from_numpy(rng.normal(0, 1.5, size=(N, 10)).astype(np.float32)).cuda()
    bp = torch.from_numpy(rng.normal(0, 1.5, size=(N, 10)).astype(np.float32)).cuda()
    zero = torch.zeros((N, 72), device='cuda')
    va = c.forward(bg, zero, want_joints=False)['verts']
    vb = c.forward(bp, zero, want_joints=False)['verts']
    ref = torch.empty(N, dtype=torch.float64, device='cuda')
    got = torch.empty(N, dtype=torch.float64, device='cuda')
    st = _lib.current_stream()
    V = c.num_verts
    _lib.check(_lib.lib.hd_eval_verts_error(_lib.fptr(va), 3 * V, _lib.fptr(vb), 3 * V, N, V, _lib.dptr(ref), st))
    _lib.check(_lib.lib.hd_eval_mesh_tpose(_lib.C.byref(c.c), _lib.fptr(bg), 10, _lib.fptr(bp), 10, N, _lib.dptr(got), st))
    assert (got - ref).abs().max().item() < 1e-6
    assert got.min().item() > 1e-3


def _flat(results):
    return [np.asarray(r[k], np.float64).tobytes() for r in results for k in sorted(r)]


def test_bit_identical_across_repeats_batching_and_chunks(consts):
    tubes = eval_ref.make_eval_tubes([3, 1, 40, 2, 17], seed=9)
    kw = dict(img_size=224, has_3d=True, min_visible=6, compute_mesh=True)
    base = Evaluator(consts, mesh_chunk=1024).errors_many(tubes, **kw)
    assert _flat(base) == _flat(Evaluator(consts, mesh_chunk=1024).errors_many(tubes, **kw))
    for chunk in (1, 7, 4096):
        assert _flat(base) == _flat(Evaluator(consts, mesh_chunk=chunk).errors_many(tubes, **kw)), chunk
    one = [Evaluator(consts).errors(**t, **kw) for t in tubes]
    assert _flat(base) == _flat(one)
    # torch input on the device, joints read in place from a wider [n, 25, 3] prediction
    t = tubes[2]
    wide = torch.zeros((40, 25, 3), device='cuda')
    wide[:, :14] = torch.from_numpy(t['joints_pred']).cuda()
    dev = dict(t, joints_pred=wide[:, :14], kps_pred=torch.from_numpy(t['kps_pred']).cuda())
    assert _flat([Evaluator(consts).errors(**dev, **kw)]) == _flat([base[2]])


def test_launch_count_and_no_host_sync(consts):
    """One launch for the frame metrics; with meshes 3 more plus 5 per chunk (2 x hd_smpl_forward + hd_eval_verts_error), and no
    host synchronisation between upload and fetch."""
    tubes = eval_ref.make_eval_tubes([5, 30, 12], seed=2)
    N = 47
    for compute_mesh, chunk, want in ((False, 1024, 1), (True, 1024, 3 + 5), (True, 10, 3 + 5 * 5)):
        ev = Evaluator(consts, mesh_chunk=chunk)
        staged = ev._stage(tubes, True, compute_mesh)
        torch.cuda.synchronize()
        _lib.lib.hd_launch_count_reset()
        torch.cuda.set_sync_debug_mode('error')
        try:
            out = ev._launch(staged, 224, 6)
        finally:
            torch.cuda.set_sync_debug_mode('default')
        assert _lib.lib.hd_launch_count() == want, (compute_mesh, chunk)
        assert tuple(out.shape) == (N, _lib.HD_EVAL_COLS + (2 if compute_mesh else 0))


def test_invalid_arguments_rejected():
    a = _lib.EvalFramesArgs()
    assert _lib.lib.hd_eval_frames(_lib.C.byref(a), None) == 1
    x = torch.zeros(16, device='cuda')
    a.N, a.n_seq, a.K, a.J, a.img_size, a.min_visible = 1, 1, 33, 14, 224.0, 6
    for f in ('seq_start', 'kps_gt', 'kps_pred', 'joints_pred', 'out'):
        setattr(a, f, x.data_ptr())
    a.kps_gt_ld, a.kps_pred_ld, a.joints_pred_ld = 99, 66, 42
    assert _lib.lib.hd_eval_frames(_lib.C.byref(a), None) == 1                 # K > 32
    a.K = 25
    a.joints_pred_ld = 41
    assert _lib.lib.hd_eval_frames(_lib.C.byref(a), None) == 1                 # short joint rows
    with pytest.raises(ValueError):
        Evaluator().errors_many([])
    with pytest.raises(ValueError):
        Evaluator().errors(np.zeros((3, 25, 3)), np.zeros((2, 25, 2)), joints_pred=np.zeros((3, 14, 3)))
    with pytest.raises(ValueError):
        Evaluator().errors(np.zeros((3, 25, 3)), np.zeros((3, 25, 2)), joints_pred=np.zeros((3, 14, 3)), has_3d=True,
                           compute_mesh=True)


# ------------------------------------------------------------------------------------------------- against the reference's own eval.py
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'eval_v1.npz')
PIXEL_KEYS = ('kp', 'kp_pa')


def _golden_tol(t, mode):
    """Metres 1e-6, pixels 1e-4 (absolute); mesh_posed 5e-5 m on the frame with rotations within 1e-3 rad of pi, where the
    reference's float32 Rodrigues and this float32 SMPL each carry ~1e-5 m."""
    tol = {k: (0, 1e-4) for k in PIXEL_KEYS}
    if mode == 'mesh':
        vis = np.sum(t['kps_gt'][:, :14, 2], axis=1) > 6
        tol['mesh_posed'] = (0, np.where(eval_cases.near_pi(t['poses_pred']), 5e-5, 1e-6)[vis])
    return tol


def test_evaluator_matches_reference_golden(consts):
    """Evaluator on the reference's inputs as eval.py feeds them (float64 ground truth, float32 predictions) against the values the
    reference's compute_errors_batched produced: with and without 3-D, with meshes; PCK and NaN positions exact."""
    g = np.load(GOLDEN)
    tubes = eval_cases.golden_tubes(g, 'nat')
    ev = Evaluator(consts)
    for mode, has_3d, mesh in (('2d', False, False), ('3d', True, False), ('mesh', True, True)):
        feeds = [dict(t, kps_gt=t['kps_gt'].astype(np.float64), joints_gt=t['joints_gt'].astype(np.float64)) for t in tubes]
        got = ev.errors_many(feeds, img_size=224, has_3d=has_3d, min_visible=6, compute_mesh=mesh)
        for i, (t, e) in enumerate(zip(tubes, got)):
            eval_cases.assert_errors_close(e, eval_cases.golden_errors(g, 'nat/t%d/%s' % (i, mode)), 0, 1e-6, _golden_tol(t, mode))


def test_sequence_const_and_hal_match_reference_golden(tmp_path):
    """test_sequence_const (delta_t = 2) and test_sequence with pred_mode 'hal' on predictions that carry the '_hal' keys, against
    the reference's functions on the same dicts."""
    from src.evaluation import eval as ev
    g = np.load(GOLDEN)
    n = int(g['const_in/kps_gt'].shape[0])
    preds = {k: g['const_in/' + k] for k in ('kps_hal', 'joints_hal', 'poses_hal', 'shapes_hal')}
    data = {'kps': g['const_in/kps_gt'].astype(np.float64), 'gt3ds': g['const_in/joints_gt'].astype(np.float64),
            'poses': g['const_in/poses_gt'].astype(np.float64).reshape(n, 24, 3), 'shape': g['const_in/shape_gt'].astype(np.float64),
            'images': np.zeros((n, 224, 224, 3), np.uint8)}
    const = ev.test_sequence_const(data, preds, str(tmp_path / 'const.pkl'), has_3d=True, min_visible=6, delta_t=2)
    assert sorted(const) == sorted(ev.CONST_KEYS)
    for group, e in const.items():
        eval_cases.assert_errors_close(e, eval_cases.golden_errors(g, 'const/' + group), 0, 1e-6, _golden_tol(None, '3d'))
    hal = ev.test_sequence(data, preds, str(tmp_path / 'hal.pkl'), pred_mode='hal', has_3d=True, min_visible=6)
    eval_cases.assert_errors_close(hal, eval_cases.golden_errors(g, 'hal'), 0, 1e-6, _golden_tol(None, '3d'))
    with open(str(tmp_path / 'hal.pkl'), 'rb') as f:
        assert _flat([pickle.load(f)]) == _flat([hal])


# ------------------------------------------------------------------------------------------------------------- eval.main end to end
def _write_split(root, smpl_model, seed=0):
    from oracle.tfrecord_writer import make_test_example, write_tfrecord
    rng = np.random.RandomState(seed)
    layout = {('3dpw', 'vidA'): [3, 25], ('3dpw', 'vidB'): [1], ('penn_action', 'vidC'): [2, 4]}
    for (ds, vid), lens in layout.items():
        d = os.path.join(root, ds, 'test')
        os.makedirs(d, exist_ok=True)
        recs = []
        for n in lens:
            t = eval_ref.make_eval_tubes([n], seed=int(rng.randint(1 << 30)), special=False)[0]
            imgs = rng.randint(0, 256, size=(n, 224, 224, 3)).astype(np.uint8)
            gt3 = np.concatenate([t['joints_gt'], np.zeros((n, 5, 3), np.float32)], axis=1)
            recs.append(make_test_example(imgs, t['kps_gt'], gt3, t['poses_gt'], t['shape_gt']))
        write_tfrecord(os.path.join(d, vid + '.tfrecord'), recs)
    return layout


def test_eval_main_end_to_end(tmp_path, weights, smpl_model):
    from human_dynamics_b200 import tf_checkpoint
    from human_dynamics_b200.config import HMMRConfig
    from src.datasets.common import read_from_example, tf_record_iterator
    from src.evaluation import eval as ev
    from src.evaluation.eval_util import extend_dict_entries, mean_of_dict_values, update_dict_entries
    from src.evaluation.tester import Tester
    tf_dir = str(tmp_path / 'tf')
    _write_split(tf_dir, smpl_model)
    prefix = str(tmp_path / 'model' / 'model.ckpt-3')
    os.makedirs(os.path.dirname(prefix))
    tf_checkpoint.save_checkpoint(prefix, {k: v for k, v in weights.items()})
    smpl_path = str(tmp_path / 'smpl.pkl')
    with open(smpl_path, 'wb') as f:
        pickle.dump(smpl_model, f)
    cfg = HMMRConfig(batch_size=1, sequence_length=20, load_path=prefix, smpl_model_path=smpl_path)
    extra = dict(tf_dir=tf_dir, pred_dir=str(tmp_path / 'cache'), test_datasets=['3dpw', 'penn_action'], split='test', min_visible=6,
                 reverse=False, resnet_path='', T=20, precomputed_phi=False, delta_t=5)
    for k, v in extra.items():
        setattr(cfg, k, v)
    model = Tester(cfg, sequence_length=20)
    got = ev.main(cfg, model=model)
    json_path = os.path.join(str(tmp_path / 'cache'), 'model.ckpt-3', 'results_test_pred_3dpw-penn_action.json')
    with open(json_path) as f:
        assert json.load(f) == got

    # expected: Tester.predict_all_images + the float64 oracle, aggregated like the reference
    want = {}
    for ds in ('3dpw', 'penn_action'):
        ds_res = {}
        for fname in ev.tfrecord_paths(cfg, ds):
            path_res = {}
            for s_ex in tf_record_iterator(fname):
                data = read_from_example(s_ex)
                images = (np.array(data['images']) / 255) * 2 - 1
                preds = model.predict_all_images(images)
                e = eval_ref.compute_errors_batched(
                    kps_gt=data['kps'], kps_pred=preds['kps'], joints_gt=data['gt3ds'], joints_pred=preds['joints'][:, :14],
                    poses_gt=data['poses'], poses_pred=preds['poses'], shape_gt=data['shape'], shapes_pred=preds['shapes'],
                    img_size=images.shape[1], has_3d=ds in ev.DATASETS_3D, min_visible=6, compute_mesh=ds == '3dpw',
                    smpl_model=smpl_model)
                extend_dict_entries(path_res, e)
            update_dict_entries(ds_res, path_res)
        mean_of_dict_values(ds_res)
        want[ds] = ds_res
    assert sorted(got) == sorted(want)
    for ds in want:
        assert sorted(got[ds]) == sorted(want[ds]), ds
        for k in want[ds]:
            assert abs(got[ds][k] - want[ds][k]) <= 1.01e-5 or (np.isnan(got[ds][k]) and np.isnan(want[ds][k])), (ds, k)
    assert got['3dpw']['mesh_posed'] > 0 and 'mesh_posed' not in got['penn_action']

    # second run: predictions from the cache (no model), errors recomputed, same JSON
    os.remove(json_path)
    for p in os.listdir(os.path.dirname(json_path)):
        if p.startswith('results_'):
            os.remove(os.path.join(os.path.dirname(json_path), p))

    class NoModel(object):
        smpl = model.smpl

        def predict_all_images(self, images):
            raise AssertionError('prediction cache missed')
    again = ev.main(cfg, model=NoModel())
    assert again == got

    # pred_mode 'hal' from the same prediction cache: Tester's predictions have no '_hal' keys, so the ordinary keys are scored
    cfg.pred_mode = 'hal'
    hal = ev.main(cfg, model=NoModel())
    assert hal == got
    assert os.path.exists(os.path.join(os.path.dirname(json_path), 'results_test_hal_3dpw-penn_action.json'))
