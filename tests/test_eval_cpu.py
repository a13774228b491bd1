"""CPU: the tfrecord / tf.train.Example reader (src/datasets/common.py), the evaluation's cache paths, aggregation and summary table
(src/evaluation/prediction.py, eval.py), the float64 oracle (oracle/eval_ref.py) -- all against the values the reference's own
eval.py / common.py produced (tests/golden/eval_v1.npz, fixture eval_v1.tfrecord) -- and argument checks of the evaluation C-ABI."""
import ctypes
import io
import os
from contextlib import redirect_stdout

import numpy as np
import pytest

from src.datasets.common import crc32c, masked_crc32c, parse_example, read_from_example, tf_record_iterator
from oracle.tfrecord_writer import make_test_example, serialize_example, write_tfrecord


def test_crc32c_known_answers():
    assert crc32c(b'123456789') == 0xE3069283
    assert crc32c(b'') == 0
    assert crc32c(b'\x00' * 32) == 0x8A9136AA                       # RFC 3720 B.4
    assert crc32c(bytes(range(32))) == 0x46DD794E
    data = bytes(np.random.RandomState(0).randint(0, 256, 1001).astype(np.uint8))
    assert crc32c(data[500:], crc32c(data[:500])) == crc32c(data)   # continuation across an unaligned split
    assert masked_crc32c(b'') == 0xA282EAD8


def _tube(n, seed=0, S=32):
    rng = np.random.RandomState(seed)
    kps = rng.uniform(0, S, size=(n, 25, 3)).astype(np.float32)
    kps[:, :14, 2] = rng.rand(n, 14) > 0.3
    imgs = rng.randint(0, 256, size=(n, S, S, 3)).astype(np.uint8)
    return imgs, kps, rng.normal(size=(n, 19, 3)), rng.normal(size=(n, 72)), rng.normal(size=10)


@pytest.mark.parametrize('packed', [True, False])
def test_read_from_example_layout(tmp_path, packed):
    import cv2
    imgs, kps, gt3ds, poses, shape = _tube(4, seed=1)
    path = str(tmp_path / 'x.tfrecord')
    ex = make_test_example(imgs, kps, gt3ds, poses, shape, packed=packed)
    write_tfrecord(path, [ex, make_test_example(imgs[:1], kps[:1], gt3ds[:1], poses[:1], shape)])
    recs = list(tf_record_iterator(path))
    assert len(recs) == 2 and recs[0] == ex
    d = read_from_example(recs[0])
    assert d['N'] == 4 and d['kps'].shape == (4, 25, 3) and d['kps'].dtype == np.float64
    # common.py:135-144: dstack(hstack(xys, vis), face, toe), transposed
    xys = kps[:, :14, :2].transpose(0, 2, 1).astype(np.float64)
    vis = kps[:, :14, 2].astype(np.int64).astype(np.float64)[:, None]
    want = np.transpose(np.dstack((np.hstack((xys, vis)), kps[:, 14:19].transpose(0, 2, 1), kps[:, 19:].transpose(0, 2, 1))), (0, 2, 1))
    assert np.array_equal(d['kps'], want)
    assert np.array_equal(d['gt3ds'], gt3ds.astype(np.float32).astype(np.float64)[:, :14])
    assert np.array_equal(d['poses'], poses.astype(np.float32).astype(np.float64).reshape(4, 24, 3))
    assert np.array_equal(d['shape'], shape.astype(np.float32).astype(np.float64))
    assert d['time_pts'] == [0, 4] and d['im_shapes'].tolist() == [[32, 32]] * 4 and d['im_paths'][1] == b'frame00001.jpg'
    feats = parse_example(recs[0])
    for i, im in enumerate(d['images']):
        enc = feats['image/encoded'][1][i]
        assert np.array_equal(im, cv2.imdecode(np.frombuffer(enc, np.uint8), cv2.IMREAD_COLOR)[:, :, ::-1])
    lazy = read_from_example(recs[0], decode_images=False)
    assert lazy['images'] == feats['image/encoded'][1]
    assert read_from_example(recs[1])['N'] == 1


def test_example_wire_format_negative_ints_and_unknown_fields():
    ex = serialize_example({'a': ('int64', [-1, 0, 2 ** 40]), 'b': ('float', [1.5, -2.0]), 'c': ('bytes', [b'', b'xy'])}, packed=False)
    ex += bytes([0x10, 0x05])                                        # an unknown varint field after the features
    f = parse_example(ex)
    assert f['a'][0] == 'int64' and f['a'][1].tolist() == [-1, 0, 2 ** 40]
    assert f['b'][1].tolist() == [1.5, -2.0] and f['c'][1] == [b'', b'xy']


def test_corrupt_records_raise(tmp_path):
    imgs, kps, gt3ds, poses, shape = _tube(2)
    path = str(tmp_path / 'c.tfrecord')
    write_tfrecord(path, [make_test_example(imgs, kps, gt3ds, poses, shape)])
    raw = bytearray(open(path, 'rb').read())
    for pos in (3, 9, 40, len(raw) - 2):                               # length, length CRC, payload, payload CRC
        bad = bytearray(raw)
        bad[pos] ^= 0x10
        p = str(tmp_path / ('bad%d.tfrecord' % pos))
        open(p, 'wb').write(bytes(bad))
        with pytest.raises(IOError):
            list(tf_record_iterator(p))
    p = str(tmp_path / 'short.tfrecord')
    open(p, 'wb').write(bytes(raw[:-7]))
    with pytest.raises(IOError):
        list(tf_record_iterator(p))


def test_cache_paths(tmp_path):
    from src.evaluation.prediction import get_eval_path_name, get_pred_path_name, get_result_path_name
    pred_dir = str(tmp_path / 'cache')
    tf = '/data/tf/3dpw/test/downtown_walking_00.tfrecord'
    p, name = get_pred_path_name('/m/run/model.ckpt-1000', tf, 2, pred_dir=pred_dir)
    assert name == '3dpw-downtown_walking_00-P2.pkl' and p == os.path.join(pred_dir, 'model.ckpt-1000', name)
    assert os.path.isdir(os.path.dirname(p))
    assert get_pred_path_name('/m/run/model.ckpt-1000', tf, 0, pred_dir=pred_dir, incl_verts=True)[1] == '3dpw-downtown_walking_00-P0-verts.pkl'
    assert get_eval_path_name('/m/model.ckpt-5', 'pred', tf, 3, pred_dir='pd', min_visible=6) == \
        os.path.join('pd', 'model.ckpt-5', 'results_pred_downtown_walking_00_P3_min-vis6.pkl')
    assert get_eval_path_name('/m/model.ckpt-5', 'hal', tf, 0, pred_dir='pd') == os.path.join('pd', 'model.ckpt-5', 'results_hal_downtown_walking_00_P0.pkl')
    assert get_result_path_name('test', '/m/model.ckpt-5', 'pred', ['3dpw', 'h36m'], pred_dir='pd') == \
        os.path.join('pd', 'model.ckpt-5', 'results_test_pred_3dpw-h36m.json')


def test_aggregation_and_summary_table():
    from src.evaluation.eval import print_summary
    from src.evaluation.eval_util import extend_dict_entries, mean_of_dict_values, update_dict_entries
    ds = {}
    for tubes in ([{'kp': [1.0, np.nan], 'accel': np.array([0.5])}, {'kp': [3.0], 'accel': np.array([])}],
                  [{'kp': [np.nan], 'accel': np.array([1.5, 2.5])}]):
        path = {}
        for t in tubes:
            extend_dict_entries(path, t)
        update_dict_entries(ds, path)
    with np.errstate(all='ignore'), pytest.warns(RuntimeWarning):
        mean_of_dict_values(ds)
    assert ds['kp'] == 2.0 and ds['accel'] == round((0.5 + 2.0) / 2, 5)
    buf = io.StringIO()
    with redirect_stdout(buf):
        print_summary({'3dpw': {'kp': 2.0, 'accel': 1.25, 'joints': 0.0812345}, 'h36m': {'kp_pck': 0.5}})
    want = ('{:>15}'.format('Data') + ''.join('{:>11}'.format(k) for k in
                                             ('accel', 'kp', 'kp_pa', 'kp_pck', 'joints', 'joints_pa', 'mesh_posed', 'mesh_tpose')) + '\n' +
            '           3dpw    1.25000    2.00000   -1.00000   -1.00000    0.08123   -1.00000   -1.00000   -1.00000\n' +
            '           h36m   -1.00000   -1.00000   -1.00000    0.50000   -1.00000   -1.00000   -1.00000   -1.00000\n')
    assert buf.getvalue() == want


def test_oracle_edge_cases():
    """The float64 oracle on the generator's edge-case frames: no visible keypoint -> NaN, exactly min_visible -> a value, 3-D
    visibility at the threshold excluded and one above included, the mirrored frame aligned by a proper rotation, coinciding
    joints -> NaN PA-MPJPE."""
    from oracle import eval_ref
    t = eval_ref.make_eval_tubes([7], seed=3)[0]
    with np.errstate(all='ignore'):
        e = eval_ref.compute_errors_batched(has_3d=True, **t)
    assert np.isnan(e['kp'][0]) and np.isfinite(e['kp'][1])
    vis = np.sum(t['kps_gt'][:, :14, 2], axis=1) > 6
    assert not vis[2] and vis[3] and len(e['joints']) == vis.sum()
    row = {i: j for j, i in enumerate(np.nonzero(vis)[0])}
    assert e['joints_pa'][row[4]] > 1e-3                          # a reflection is not a rotation: the mirror is not undone
    assert np.isnan(e['joints_pa'][row[5]]) and np.isfinite(e['joints'][row[5]])
    assert len(e['accel']) == 5 and len(e['accel_error']) == sum(vis[i] and vis[i + 1] and vis[i + 2] for i in range(5))


def test_eval_abi_argument_checks_without_device():
    from human_dynamics_b200 import _lib
    a = _lib.EvalFramesArgs()
    assert _lib.lib.hd_eval_frames(None, None) == 1
    assert _lib.lib.hd_eval_frames(ctypes.byref(a), None) == 1
    assert b'null' in _lib.lib.hd_last_error()
    buf = ctypes.create_string_buffer(64)
    for f in ('seq_start', 'kps_gt', 'kps_pred', 'joints_pred', 'out'):
        setattr(a, f, ctypes.addressof(buf))
    a.N, a.n_seq, a.K, a.J, a.img_size, a.min_visible = 5, 1, 25, 14, 224.0, 6
    a.kps_gt_ld, a.kps_pred_ld, a.joints_pred_ld = 75, 50, 42
    for field, bad in (('n_seq', 0), ('N', -1), ('K', 0), ('K', 33), ('J', 3), ('kps_gt_ld', 74), ('kps_pred_ld', 49),
                       ('img_size', 0.0), ('min_visible', -1)):
        old = getattr(a, field)
        setattr(a, field, bad)
        assert _lib.lib.hd_eval_frames(ctypes.byref(a), None) == 1, field
        setattr(a, field, old)
    a.joints_gt, a.joints_gt_ld = ctypes.addressof(buf), 41
    assert _lib.lib.hd_eval_frames(ctypes.byref(a), None) == 1
    assert _lib.lib.hd_eval_verts_error(None, 3, None, 3, 1, 1, None, None) == 1
    p = ctypes.addressof(buf)
    assert _lib.lib.hd_eval_verts_error(p, 8, p, 9, 1, 3, p, None) == 1             # a_ld < 3V
    assert _lib.lib.hd_eval_verts_error(p, 9, p, 9, 1, 0, p, None) == 1             # V = 0
    assert _lib.lib.hd_eval_mesh_tpose(None, p, 10, p, 10, 1, p, None) == 1
    c = _lib.SmplConsts()
    assert _lib.lib.hd_eval_mesh_tpose(ctypes.byref(c), p, 10, p, 10, 1, p, None) == 1   # null dirs / lbs_w
    c.dirs, c.lbs_w, c.num_verts, c.lbs_nnz = p, p, 10, 4
    assert _lib.lib.hd_eval_mesh_tpose(ctypes.byref(c), p, 9, p, 10, 1, p, None) == 1    # beta stride < 10


# ------------------------------------------------------------------------------------- against the reference's own eval.py / common.py
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'eval_v1.npz')
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'eval_v1.tfrecord')
from oracle.eval_cases import assert_errors_close, golden_errors, golden_tubes, near_pi  # noqa: E402


def golden():
    return np.load(GOLDEN)


def test_oracle_matches_reference_float64_run():
    """The float64 oracle against the reference's compute_errors_batched on float64 inputs (with and without 3-D): 1e-9."""
    from oracle import eval_ref
    g = golden()
    for i, t in enumerate(golden_tubes(g, 'f64')):
        for mode, has_3d in (('2d', False), ('3d', True)):
            with np.errstate(all='ignore'):
                got = eval_ref.compute_errors_batched(img_size=224, has_3d=has_3d, min_visible=6, **t)
            assert_errors_close(got, golden_errors(g, 'f64/t%d/%s' % (i, mode)), 1e-9, 1e-12)


def test_oracle_matches_reference_natural_run(smpl_model):
    """The oracle against the reference as eval.py feeds it (float32 predictions, float64 ground truth, float32 SMPL), meshes included.
    The reference computes the prediction's accelerations and Procrustes means in float32 there, hence 1e-5 relative; PCK and NaN
    positions exact; meshes 1e-6 m, and 5e-5 m for the frame whose rotations lie within 1e-3 rad of pi (the reference's float32
    Rodrigues there differs from float64 by 1.9e-5 m of mesh distance)."""
    from oracle import eval_ref
    g = golden()
    for i, t in enumerate(golden_tubes(g, 'nat')):
        vis = np.sum(t['kps_gt'][:, :14, 2], axis=1) > 6
        tol = {'mesh_posed': (0, np.where(near_pi(t['poses_pred']), 5e-5, 1e-6)[vis]), 'mesh_tpose': (0, 1e-6)}
        for mode, has_3d, mesh in (('2d', False, False), ('3d', True, False), ('mesh', True, True)):
            with np.errstate(all='ignore'):
                got = eval_ref.compute_errors_batched(img_size=224, has_3d=has_3d, min_visible=6, compute_mesh=mesh,
                                                      smpl_model=smpl_model, **t)
            assert_errors_close(got, golden_errors(g, 'nat/t%d/%s' % (i, mode)), 1e-5, 1e-9, tol)


def test_golden_covers_the_edge_cases():
    """The reference's own values on the edge-case frames: no visible keypoint -> NaN, a mirrored prediction not undone by the
    rotation, coinciding joints -> NaN PA-MPJPE, tubes of 1 and 2 frames -> no acceleration."""
    g = golden()
    assert np.isnan(g['f64/t0/2d/kp'][0]) and g['f64/t0/2d/accel'].size == 0 and g['f64/t1/2d/accel'].size == 0
    assert np.isfinite(g['f64/t1/2d/kp'][0])                    # exactly min_visible keypoints
    pa = g['f64/t2/3d/joints_pa']
    assert np.isnan(pa).sum() == 1 and np.nanmin(pa) > 1e-3


def test_reader_matches_reference_read_from_example():
    """src/datasets/common.py on the fixture the reference's convert_to_example_temporal wrote, against the reference's
    read_from_example: every array exact, every decoded frame bit for bit."""
    import hashlib
    import json
    g = golden()
    recs = list(tf_record_iterator(FIXTURE))
    assert len(recs) == 4
    for p_id, rec in enumerate(recs):
        d = read_from_example(rec)
        for k in ('centers', 'kps', 'gt3ds', 'im_shapes', 'poses', 'scales', 'shape', 'start_pts'):
            want = g['fx/%d/%s' % (p_id, k)]
            assert np.asarray(d[k]).dtype.kind == want.dtype.kind and np.array_equal(np.asarray(d[k]), want), k
        assert d['N'] == int(g['fx/%d/N' % p_id]) and d['time_pts'] == g['fx/%d/time_pts' % p_id].tolist()
        assert [p.decode() for p in d['im_paths']] == json.loads(str(g['fx/%d/im_paths' % p_id]))
        assert [im.shape for im in d['images']] == [tuple(s) for s in g['fx/%d/images_shape' % p_id]]
        assert [hashlib.sha256(np.ascontiguousarray(im).tobytes()).hexdigest() for im in d['images']] == \
            json.loads(str(g['fx/%d/images_sha256' % p_id]))


def test_bookkeeping_matches_reference():
    """Cache paths, mean_of_dict_values and the print_summary text against the reference's prediction.py / eval_util.py / eval.py."""
    import json
    import warnings
    from src.evaluation.eval import print_summary
    from src.evaluation.eval_util import mean_of_dict_values
    from src.evaluation.prediction import get_eval_path_name, get_pred_path_name, get_result_path_name
    g = golden()
    agg = json.loads(str(g['agg_in']))
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        mean_of_dict_values(agg)
    want = json.loads(str(g['agg_out']))
    assert sorted(agg) == sorted(want) and all(agg[k] == want[k] or (np.isnan(agg[k]) and np.isnan(want[k])) for k in want)
    buf = io.StringIO()
    with redirect_stdout(buf):
        print_summary(json.loads(str(g['summary_in'])))
    assert buf.getvalue() == str(g['summary_text'])
    cwd = os.getcwd()
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        os.chdir(td)
        try:
            tf_path = os.path.join('tf', '3dpw', 'test', 'downtown_walking_00.tfrecord')
            got = [get_pred_path_name('logs/run/model.ckpt-1000', tf_path, 2, pred_dir='pd')[0],
                   get_pred_path_name('logs/run/model.ckpt-1000', tf_path, 0, pred_dir='pd', incl_verts=True)[0],
                   get_eval_path_name('logs/run/model.ckpt-1000', 'pred', tf_path, 3, pred_dir='pd', min_visible=6),
                   get_eval_path_name('logs/run/model.ckpt-1000', 'hal', tf_path, 0, pred_dir='pd'),
                   get_result_path_name('test', 'logs/run/model.ckpt-1000', 'pred', ['3dpw', 'h36m'], pred_dir='pd')]
        finally:
            os.chdir(cwd)
    assert got == json.loads(str(g['paths']))


def test_feature_merge_and_absent_features():
    """A list field repeated inside one Feature concatenates (protobuf merge); an absent feature reads as an empty list."""
    from src.datasets.common import _parse_feature
    from oracle.tfrecord_writer import _feature, _ld
    body = _feature('float', [1.0, 2.0]) + _feature('float', [3.0])                # two float_list fields in one Feature
    kind, vals = _parse_feature(memoryview(body))
    assert kind == 'float' and vals.tolist() == [1.0, 2.0, 3.0]
    imgs, kps, gt3ds, poses, shape = _tube(2)
    ex = make_test_example(imgs, kps, gt3ds, poses, shape)
    feats = parse_example(ex)
    del feats['meta/time_pts']
    ex2 = serialize_example(feats)
    assert read_from_example(ex2, decode_images=False)['time_pts'] == []
    assert _ld(1, b'') == b'\x0a\x00'
