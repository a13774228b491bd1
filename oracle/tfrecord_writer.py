"""Test infrastructure: writes test tfrecords the way the reference's converters do (src/datasets/common.py feature helpers and
make_test_tfrecords.py's key set), so that the reader in src/datasets/common.py and the evaluation entry point can be exercised
without TensorFlow.  Floats and int64s are written packed, as TF does; `packed=False` writes the unpacked form protobuf also accepts.
"""
import struct

import numpy as np

from src.datasets.common import masked_crc32c


def _varint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _ld(num, payload):
    return _varint(num << 3 | 2) + _varint(len(payload)) + payload


def _feature(kind, values, packed=True):
    if kind == 'bytes':
        body = b''.join(_ld(1, bytes(v)) for v in values)
        return _ld(1, body)
    if kind == 'float':
        vals = np.asarray(values, np.float32).ravel()
        body = _ld(1, vals.astype('<f4').tobytes()) if packed else \
            b''.join(_varint(1 << 3 | 5) + struct.pack('<f', v) for v in vals)
        return _ld(2, body)
    vals = [int(v) for v in np.asarray(values, np.int64).ravel()]
    body = _ld(1, b''.join(_varint(v) for v in vals)) if packed else b''.join(_varint(1 << 3 | 0) + _varint(v) for v in vals)
    return _ld(3, body)


def serialize_example(features, packed=True):
    """{name: (kind, values)} -> serialized tf.train.Example (entries in sorted key order)."""
    entries = b''.join(_ld(1, _ld(1, k.encode('utf-8')) + _ld(2, _feature(kind, v, packed))) for k, (kind, v) in sorted(features.items()))
    return _ld(1, entries)


def write_tfrecord(path, records):
    with open(path, 'wb') as f:
        for r in records:
            head = struct.pack('<Q', len(r))
            f.write(head + struct.pack('<I', masked_crc32c(head)) + r + struct.pack('<I', masked_crc32c(r)))


def encode_jpeg(rgb, quality=95):
    import cv2
    ok, buf = cv2.imencode('.jpg', np.ascontiguousarray(rgb[:, :, ::-1]), [cv2.IMWRITE_JPEG_QUALITY, quality])
    assert ok
    return buf.tobytes()


def make_test_example(images, kps, gt3ds, poses, shape, packed=True):
    """One tube in the test-tfrecord layout: images N x S x S x 3 uint8 RGB, kps N x 25 x 3 (14 LSP points + vis, 5 face, 6 toe
    points), gt3ds N x J x 3, poses N x 72 axis-angle, shape 10."""
    N = len(images)
    kps = np.asarray(kps, np.float32)
    S = images[0].shape[0]
    feats = {
        'meta/N': ('int64', [N]),
        'image/encoded': ('bytes', [encode_jpeg(im) for im in images]),
        'image/centers': ('int64', np.full((N, 2), S // 2)),
        'image/xys': ('float', kps[:, :14, :2].transpose(0, 2, 1)),
        'image/visibilities': ('int64', kps[:, :14, 2].astype(np.int64)),
        'image/face_pts': ('float', kps[:, 14:19].transpose(0, 2, 1)),
        'image/toe_pts': ('float', kps[:, 19:25].transpose(0, 2, 1)),
        'image/scale_factors': ('float', np.ones(N)),
        'mosh/gt3ds': ('float', gt3ds),
        'mosh/poses': ('float', poses),
        'mosh/shape': ('float', shape),
        'meta/time_pts': ('int64', [0, N]),
        'image/crop_pts': ('int64', np.zeros((N, 2))),
        'image/heightwidths': ('int64', np.tile([S, S], (N, 1))),
        'image/filenames': ('bytes', [('frame%05d.jpg' % i).encode() for i in range(N)]),
    }
    return serialize_example(feats, packed=packed)
