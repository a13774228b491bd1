"""Generates tests/golden/eval_v1.npz and the fixture tests/golden/eval_v1.tfrecord by EXECUTING THE REFERENCE'S OWN SOURCE:

    src/evaluation/eval.py          compute_gpu_smpl, compute_errors_batched, test_sequence (pred and hal), test_sequence_const,
                                    print_summary
    src/evaluation/prediction.py    get_pred_path_name, get_eval_path_name, get_result_path_name
    src/evaluation/eval_util.py     every metric, rot_mat_to_axis_angle (cv2.Rodrigues), mean_of_dict_values
    src/datasets/common.py          convert_to_example_temporal + ImageCoder.encode_jpeg (writes the fixture), read_from_example

unmodified, over the numpy TensorFlow stand-in of oracle/ref_exec (see make_ref_exec_golden.py).  The evaluation needs a few more
stand-in pieces, added here at run time (test infrastructure only): tf.group and the two variable initialisers, tf.string, tf.image's
JPEG / PNG coders over OpenCV (RGB), tf.compat.as_bytes, tf.train.Example / Features / Feature / BytesList / FloatList / Int64List
as protobuf messages built from tensorflow/core/example's field numbers over google.protobuf, and tf.python_io's record writer and
iterator (framing and masked CRC32C from human_dynamics_b200/tf_checkpoint.py's CRC, not from the reader under test).

Inputs (oracle/eval_cases.py, seeded) and outputs are both stored.  Two runs of compute_errors_batched:
  nat  float32 predictions and float64 ground truth, as eval.py feeds them from read_from_example and Tester (the reference then
       computes parts of the metrics in float32);
  f64  the same cases in float64, with predicted keypoints on a 2^-12 grid so that the float32 pixel scaling of the port and the
       float64 one of this run agree exactly: everything the reference computes is float64 and pins the oracle to 1e-9.
The tubes have lengths 1, 2, 3, 6 and 12, and hold a frame with no visible keypoint, one with exactly min_visible, 3-D visibility at
and one above the threshold, a mirrored prediction, coinciding joints and rotations near pi.  Meshes use the synthetic SMPL model
(human_dynamics_b200.synthetic, seed 2) pickled like the official file.

Needs a checkout of the reference project, named by HD_REFERENCE_ROOT.  Run from the repo root:
    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_eval_golden.py
"""
import contextlib
import hashlib
import importlib.util
import io
import json
import os
import shutil
import struct
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'eval_v1.npz')
FIXTURE = os.path.join(HERE, 'eval_v1.tfrecord')
LENS = [1, 2, 3, 6, 12]
CONST_LEN, DELTA_T = 12, 2
MIN_VIS, IMG = 6, 224


def _by_path(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _example_classes():
    """tensorflow/core/example/{feature,example}.proto (field numbers and types as published), built over google.protobuf."""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fdp = descriptor_pb2.FileDescriptorProto(name='hd_standin_example.proto', package='tensorflow', syntax='proto3')

    def msg(name, fields, nested=None):
        m = fdp.message_type.add(name=name)
        for fname, num, typ, label, tname in fields:
            f = m.field.add(name=fname, number=num, type=typ, label=label)
            if tname:
                f.type_name = tname
        return m
    rep, opt = F.LABEL_REPEATED, F.LABEL_OPTIONAL
    msg('BytesList', [('value', 1, F.TYPE_BYTES, rep, None)])
    msg('FloatList', [('value', 1, F.TYPE_FLOAT, rep, None)])
    msg('Int64List', [('value', 1, F.TYPE_INT64, rep, None)])
    feat = msg('Feature', [('bytes_list', 1, F.TYPE_MESSAGE, opt, '.tensorflow.BytesList'),
                           ('float_list', 2, F.TYPE_MESSAGE, opt, '.tensorflow.FloatList'),
                           ('int64_list', 3, F.TYPE_MESSAGE, opt, '.tensorflow.Int64List')])
    feat.oneof_decl.add(name='kind')
    for f in feat.field:
        f.oneof_index = 0
    feats = msg('Features', [('feature', 1, F.TYPE_MESSAGE, rep, '.tensorflow.Features.FeatureEntry')])
    entry = feats.nested_type.add(name='FeatureEntry')
    entry.options.map_entry = True
    entry.field.add(name='key', number=1, type=F.TYPE_STRING, label=opt)
    entry.field.add(name='value', number=2, type=F.TYPE_MESSAGE, label=opt, type_name='.tensorflow.Feature')
    msg('Example', [('features', 1, F.TYPE_MESSAGE, opt, '.tensorflow.Features')])
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return {n: message_factory.GetMessageClass(pool.FindMessageTypeByName('tensorflow.' + n))
            for n in ('BytesList', 'FloatList', 'Int64List', 'Feature', 'Features', 'Example')}


def extend_standin(tf, ckpt):
    import cv2
    noop = lambda *ops, **kw: tf._op(lambda *a: np.zeros((), np.int32), [o for o in ops if isinstance(o, tf.Tensor)], 'noop')
    tf.group = noop
    tf.global_variables_initializer = lambda: noop()
    tf.local_variables_initializer = lambda: noop()
    tf.string, tf.uint8 = object, np.uint8
    # ImageCoder's placeholders have no static shape: any fed shape is accepted (the stand-in checks fed shapes against a probe)
    placeholder, run = tf.placeholder, tf.Session.run

    def any_shape_placeholder(dtype, shape=None, name=None):
        t = placeholder(dtype, () if shape is None else shape, name)
        t.any_shape = shape is None
        return t

    def run_any_shape(self, fetches, feed_dict=None):
        for k, v in (feed_dict or {}).items():
            if getattr(k, 'any_shape', False):
                k.probe = np.asarray(v, dtype=k.probe.dtype)
        return run(self, fetches, feed_dict)
    tf.placeholder, tf.Session.run = any_shape_placeholder, run_any_shape

    def as_bytes(s):
        s = s.item() if isinstance(s, np.ndarray) else s         # session results are 0-d object arrays
        return s if isinstance(s, bytes) else s.encode('utf-8')
    tf.compat = types.SimpleNamespace(as_bytes=as_bytes)

    def _item(a):
        a = np.asarray(a)
        return a.item() if a.dtype == object else a

    def decode(data):
        data = _item(data)
        if not isinstance(data, (bytes, bytearray)):
            return np.zeros((1, 1, 3), np.uint8)                 # graph-construction probe
        return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)[:, :, ::-1].copy()

    def encoder(ext, params):
        def enc(img):
            img = np.asarray(img)
            if img.ndim != 3:
                return np.asarray(b'', dtype=object)
            ok, buf = cv2.imencode(ext, np.ascontiguousarray(img[:, :, ::-1]), params)
            assert ok
            return np.asarray(buf.tobytes(), dtype=object)
        return enc
    tf.image = types.SimpleNamespace(
        decode_jpeg=lambda x, channels=3, **kw: tf._op(decode, [x], 'decode_jpeg'),
        decode_png=lambda x, channels=3, **kw: tf._op(decode, [x], 'decode_png'),
        encode_jpeg=lambda x, format='rgb', quality=95, **kw: tf._op(encoder('.jpg', [cv2.IMWRITE_JPEG_QUALITY, quality]), [x], 'encode_jpeg'),
        encode_png=lambda x, **kw: tf._op(encoder('.png', []), [x], 'encode_png'))
    for n, cls in _example_classes().items():
        setattr(tf.train, n, cls)

    def masked(b):
        return ckpt.mask_crc(ckpt.crc32c(b))

    class TFRecordWriter(object):
        def __init__(self, path):
            self.f = open(path, 'wb')

        def write(self, rec):
            head = struct.pack('<Q', len(rec))
            self.f.write(head + struct.pack('<I', masked(head)) + rec + struct.pack('<I', masked(rec)))

        def close(self):
            self.f.close()

    def tf_record_iterator(path):
        with open(path, 'rb') as f:
            while True:
                head = f.read(12)
                if not head:
                    return
                n, crc = struct.unpack('<QI', head)
                assert masked(head[:8]) == crc
                rec = f.read(n)
                assert masked(rec) == struct.unpack('<I', f.read(4))[0]
                yield rec
    tf.python_io = types.SimpleNamespace(TFRecordWriter=TFRecordWriter, tf_record_iterator=tf_record_iterator)


def _tubes(cases, special_seed, quantize):
    tubes = cases.make_eval_tubes(LENS, K=25, seed=special_seed, img_size=IMG, min_visible=MIN_VIS)
    for t in tubes:
        if quantize:
            t['kps_pred'] = (np.round(t['kps_pred'].astype(np.float64) * 4096) / 4096).astype(np.float32)
    return tubes


def _feed(t, f64):
    """The arguments test_sequence passes: ground truth float64 (read_from_example), predictions float32 (Tester) or all float64."""
    pd = np.float64 if f64 else np.float32
    n = len(t['kps_gt'])
    return dict(kps_gt=t['kps_gt'].astype(np.float64), kps_pred=t['kps_pred'].astype(pd), joints_gt=t['joints_gt'].astype(np.float64),
                joints_pred=t['joints_pred'].astype(pd), poses_gt=t['poses_gt'].astype(np.float64).reshape(n, 24, 3),
                poses_pred=t['poses_pred'].astype(pd), shape_gt=t['shape_gt'].astype(np.float64), shapes_pred=t['shapes_pred'].astype(pd))


def _store(out, prefix, errors):
    for k, v in errors.items():
        out['%s/%s' % (prefix, k)] = np.asarray(v, np.float64)


def run_reference(REF, tmp):
    gen = _by_path('_make_ref_exec_golden', os.path.join(HERE, 'make_ref_exec_golden.py'))
    gen.REF = REF
    syn, ckpt = gen.setup_paths()
    cases = _by_path('_hd_eval_cases', os.path.join(ROOT, 'oracle', 'eval_cases.py'))
    import tensorflow as tf
    extend_standin(tf, ckpt)
    os.chdir(tmp)
    os.makedirs('models')
    gen.write_smpl_pickle(syn.make_synthetic_smpl(seed=2), os.path.join('models', 'neutral_smpl_with_cocoplustoesankles_reg.pkl'))
    # src/config.py stops (ipdb) when the checkout has no models/ directory; eval.py only calls its get_config under __main__
    sys.modules['src.config'] = types.SimpleNamespace(get_config=None)
    from src.evaluation import eval as E
    from src.evaluation import prediction as P
    from src.evaluation import eval_util as U
    from src.datasets import common as CM
    out = {}

    # ---- compute_errors_batched: natural dtypes (with / without 3-D, with / without meshes) and the float64 run
    for name, quant, f64 in (('nat', False, False), ('f64', True, True)):
        tubes = _tubes(cases, 11, quant)
        for i, t in enumerate(tubes):
            for k, v in t.items():
                out['in_%s/t%d/%s' % (name, i, k)] = v
            a = _feed(t, f64)
            modes = (('2d', False, False), ('3d', True, False)) + ((('mesh', True, True),) if name == 'nat' else ())
            for mode, has_3d, mesh in modes:
                e = E.compute_errors_batched(img_size=IMG, has_3d=has_3d, min_visible=MIN_VIS, compute_mesh=mesh, **a)
                _store(out, '%s/t%d/%s' % (name, i, mode), e)

    # ---- test_sequence_const (delta_t, a flag no module defines, is given through the module's `config`) and test_sequence 'hal'
    rng = np.random.RandomState(5)
    base = cases.make_eval_tubes([CONST_LEN], seed=12, special=False)[0]
    n = CONST_LEN
    hal = {'kps_hal': np.stack([base['kps_pred'] + rng.normal(0, 0.02, (n, 25, 2)).astype(np.float32) for _ in range(3)], 1),
           'joints_hal': np.stack([np.concatenate([base['joints_pred'], rng.normal(0, .3, (n, 11, 3)).astype(np.float32)], 1)
                                   + rng.normal(0, 0.01, (n, 25, 3)).astype(np.float32) for _ in range(3)], 1),
           'poses_hal': np.stack([base['poses_pred']] * 3, 1), 'shapes_hal': np.stack([base['shapes_pred']] * 3, 1)}
    for k, v in hal.items():
        out['const_in/' + k] = v
    for k in ('kps_gt', 'joints_gt', 'poses_gt', 'shape_gt'):
        out['const_in/' + k] = base[k]
    data = {'kps': base['kps_gt'].astype(np.float64), 'gt3ds': base['joints_gt'].astype(np.float64),
            'poses': base['poses_gt'].astype(np.float64).reshape(n, 24, 3), 'shape': base['shape_gt'].astype(np.float64),
            'images': np.zeros((n, IMG, IMG, 3), np.uint8)}
    E.config = types.SimpleNamespace(delta_t=DELTA_T)
    const = E.test_sequence_const(data, hal, os.path.join(tmp, 'const.pkl'), has_3d=True, min_visible=MIN_VIS)
    for group, e in const.items():
        _store(out, 'const/' + group, e)
    e = E.test_sequence(data, hal, os.path.join(tmp, 'hal.pkl'), pred_mode='hal', has_3d=True, min_visible=MIN_VIS)
    _store(out, 'hal', e)

    # ---- bookkeeping: aggregation, the summary table, the cache paths
    agg_in = {'kp': [[1.0, float('nan'), 2.5], [float('nan')], [4.0]], 'accel': [[0.5], [], [1.5, 2.25]], 'mesh_posed': [[-1], [-1]]}
    agg = {k: [list(v) for v in vs] for k, vs in agg_in.items()}
    with np.errstate(all='ignore'):
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            U.mean_of_dict_values(agg)
    out['agg_in'] = np.asarray(json.dumps(agg_in))
    out['agg_out'] = np.asarray(json.dumps(agg))
    table = {'3dpw': {'accel': 0.0123456, 'kp': 10.5, 'kp_pa': 7.25, 'kp_pck': 0.9, 'joints': 0.081234, 'joints_pa': 0.05,
                      'mesh_posed': 0.1, 'mesh_tpose': 0.02, 'pose': -1, 'shape': -1},
             'penn_action': {'accel': 0.5, 'kp': 12.0, 'kp_pa': 9.0, 'kp_pck': 0.75}}
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        E.print_summary(table)
    out['summary_in'] = np.asarray(json.dumps(table))
    out['summary_text'] = np.asarray(buf.getvalue())
    tf_path = os.path.join('tf', '3dpw', 'test', 'downtown_walking_00.tfrecord')
    paths = [P.get_pred_path_name('logs/run/model.ckpt-1000', tf_path, 2, pred_dir='pd')[0],
             P.get_pred_path_name('logs/run/model.ckpt-1000', tf_path, 0, pred_dir='pd', incl_verts=True)[0],
             P.get_eval_path_name('logs/run/model.ckpt-1000', 'pred', tf_path, 3, pred_dir='pd', min_visible=6),
             P.get_eval_path_name('logs/run/model.ckpt-1000', 'hal', tf_path, 0, pred_dir='pd'),
             P.get_result_path_name('test', 'logs/run/model.ckpt-1000', 'pred', ['3dpw', 'h36m'], pred_dir='pd')]
    out['paths'] = np.asarray(json.dumps(paths))

    # ---- the fixture: 4 tubes written by the reference's convert_to_example_temporal, read back by its read_from_example
    coder = CM.ImageCoder()
    writer = tf.python_io.TFRecordWriter(os.path.join(tmp, 'fixture.tfrecord'))
    yy, xx = np.mgrid[0:IMG, 0:IMG]
    for j, m in enumerate([1, 2, 3, 4]):
        t = cases.make_eval_tubes([m], seed=30 + j, special=False)[0]
        imgs = [np.stack([(xx * (f + 1) + 3 * j) % 256, (yy * 2 + 17 * f) % 256, (xx + yy + 40 * j) % 256], -1).astype(np.uint8)
                for f in range(m)]
        labels = t['kps_gt'].transpose(0, 2, 1).astype(np.float64)               # N x 3 x 25
        ex = CM.convert_to_example_temporal(
            image_datas=[coder.encode_jpeg(im) for im in imgs], image_paths=['vid%d/frame%05d.jpg' % (j, f) for f in range(m)],
            image_shapes=[[IMG, IMG]] * m, labels=labels, centers=np.full((m, 2), IMG // 2 + j), gt3ds=t['joints_gt'],
            scale_factors=np.linspace(0.9, 1.1, m), start_pts=np.tile([[j, 2 * j]], (m, 1)), cams=np.ones((m, 3)),
            poses=t['poses_gt'], shape=t['shape_gt'], time_pts=[5 * j, 5 * j + m])
        writer.write(ex.SerializeToString())
    writer.close()
    for p_id, s_ex in enumerate(tf.python_io.tf_record_iterator(os.path.join(tmp, 'fixture.tfrecord'))):
        d = CM.read_from_example(s_ex)
        for k in ('centers', 'kps', 'gt3ds', 'im_shapes', 'poses', 'scales', 'shape', 'start_pts'):
            out['fx/%d/%s' % (p_id, k)] = np.asarray(d[k])
        out['fx/%d/N' % p_id] = np.asarray(d['N'])
        out['fx/%d/time_pts' % p_id] = np.asarray(list(d['time_pts']))
        out['fx/%d/images_sha256' % p_id] = np.asarray(json.dumps([hashlib.sha256(np.ascontiguousarray(im).tobytes()).hexdigest()
                                                                   for im in d['images']]))
        out['fx/%d/images_shape' % p_id] = np.asarray([im.shape for im in d['images']])
        out['fx/%d/im_paths' % p_id] = np.asarray(json.dumps([p.decode() for p in d['im_paths']]))
    return out


def main():
    REF = os.environ.get('HD_REFERENCE_ROOT', '')
    tmp = tempfile.mkdtemp()
    try:
        out = run_reference(REF, tmp)
        shutil.copyfile(os.path.join(tmp, 'fixture.tfrecord'), FIXTURE)
    finally:
        os.chdir(ROOT)
        shutil.rmtree(tmp, ignore_errors=True)
    np.savez_compressed(OUT, **out)
    print('wrote %s (%d arrays) and %s' % (OUT, len(out), FIXTURE))


if __name__ == '__main__':
    sys.exit(main())
