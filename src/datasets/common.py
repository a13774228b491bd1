"""Reading the test tfrecords without TensorFlow -- drop-in for read_from_example of the reference's src/datasets/common.py (:86-163),
plus the `tf.python_io.tf_record_iterator` it is fed from.

A tfrecord file is a sequence of records: uint64 length (little endian), uint32 masked CRC32C of those 8 bytes, the payload, uint32
masked CRC32C of the payload.  Both checksums are verified; a short or corrupt record raises IOError.  The payload is a serialized
`tf.train.Example` (a Features map of name -> BytesList / FloatList / Int64List), decoded here from the protobuf wire format in pure
Python (packed and unpacked repeated fields both accepted).  JPEG frames are decoded with OpenCV, as RGB.  Writing records is not part
of this module.

The checksums are computed in Python (slicing-by-8 tables): about 15 MB/s on one host core, so a test record of a few hundred 224^2
JPEGs (a few MB) costs a fraction of a second to verify; tools/bench_eval.py times reading a record of that size.
"""
import struct

import numpy as np

# ----------------------------------------------------------------------------------------------------------- CRC32C (Castagnoli)
_POLY = 0x82F63B78


def _make_tables():
    t0 = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ _POLY if c & 1 else c >> 1
        t0.append(c)
    tables = [t0]
    for _ in range(7):                         # slicing-by-8: table k advances a byte through k further zero bytes
        prev = tables[-1]
        tables.append([(prev[i] >> 8) ^ t0[prev[i] & 0xFF] for i in range(256)])
    return tables


_T = _make_tables()


def crc32c(data, crc=0):
    """CRC-32C of `data` (bytes-like), continuing from `crc`."""
    t0, t1, t2, t3, t4, t5, t6, t7 = _T
    mv = memoryview(data).cast('B')
    c = crc ^ 0xFFFFFFFF
    n8 = len(mv) // 8 * 8
    for (w,) in struct.iter_unpack('<Q', mv[:n8]):
        x = c ^ (w & 0xFFFFFFFF)
        h = w >> 32
        c = (t7[x & 0xFF] ^ t6[(x >> 8) & 0xFF] ^ t5[(x >> 16) & 0xFF] ^ t4[x >> 24] ^
             t3[h & 0xFF] ^ t2[(h >> 8) & 0xFF] ^ t1[(h >> 16) & 0xFF] ^ t0[h >> 24])
    for b in mv[n8:]:
        c = (c >> 8) ^ t0[(c ^ b) & 0xFF]
    return c ^ 0xFFFFFFFF


def masked_crc32c(data):
    """The checksum tfrecord files store: the CRC rotated right by 15 bits plus 0xa282ead8."""
    c = crc32c(data)
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


def tf_record_iterator(path):
    """Yields the payload (bytes) of every record of a tfrecord file, like tf.python_io.tf_record_iterator (no compression)."""
    with open(path, 'rb') as f:
        while True:
            head = f.read(12)
            if not head:
                return
            if len(head) < 12:
                raise IOError('%s: truncated record header' % path)
            length, length_crc = struct.unpack('<QI', head)
            if masked_crc32c(head[:8]) != length_crc:
                raise IOError('%s: corrupt record length (CRC mismatch)' % path)
            data = f.read(length)
            foot = f.read(4)
            if len(data) < length or len(foot) < 4:
                raise IOError('%s: truncated record' % path)
            if masked_crc32c(data) != struct.unpack('<I', foot)[0]:
                raise IOError('%s: corrupt record payload (CRC mismatch)' % path)
            yield data


# ----------------------------------------------------------------------------------------------------------- tf.train.Example
def _varint(buf, pos):
    result, shift = 0, 0
    while True:
        if pos >= len(buf):
            raise ValueError('truncated varint')
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7
        if shift > 63:
            raise ValueError('varint too long')


def _fields(buf):
    """(field number, wire type, value) of a protobuf message: ints for varints / fixed, memoryviews for length-delimited fields."""
    pos, n = 0, len(buf)
    while pos < n:
        key, pos = _varint(buf, pos)
        num, wt = key >> 3, key & 7
        if wt == 0:
            val, pos = _varint(buf, pos)
        elif wt == 1:
            val, pos = buf[pos:pos + 8], pos + 8
        elif wt == 2:
            ln, pos = _varint(buf, pos)
            if pos + ln > n:
                raise ValueError('truncated length-delimited field')
            val, pos = buf[pos:pos + ln], pos + ln
        elif wt == 5:
            val, pos = buf[pos:pos + 4], pos + 4
        else:
            raise ValueError('unsupported wire type %d' % wt)
        yield num, wt, val


def _to_int64(v):
    return v - (1 << 64) if v >= (1 << 63) else v


def _parse_feature(buf):
    """Feature -> ('bytes', [bytes]) | ('float', float32 array) | ('int64', int64 array).  Repeated occurrences of the list field
    concatenate, as protobuf's merge does (TF's writers emit one)."""
    kind, out = None, []
    for num, _, lst in _fields(buf):
        k = {1: 'bytes', 2: 'float', 3: 'int64'}.get(num)
        if k is None:
            continue
        if k != kind:                               # a oneof: the last kind set wins
            kind, out = k, []
        for vnum, wt, v in _fields(lst):
            if vnum != 1:
                continue
            if kind == 'bytes':
                out.append(bytes(v))
            elif kind == 'float':
                out.extend(np.frombuffer(bytes(v), '<f4'))    # packed run or one fixed32 value
            elif wt == 2:                           # packed varints
                p = 0
                while p < len(v):
                    x, p = _varint(v, p)
                    out.append(_to_int64(x))
            else:
                out.append(_to_int64(v))
    if kind == 'float':
        return kind, np.asarray(out, np.float32)
    if kind == 'int64':
        return kind, np.asarray(out, np.int64)
    return kind or 'bytes', out


def parse_example(serialized):
    """A serialized tf.train.Example -> {feature name: (kind, values)}."""
    buf = memoryview(serialized).cast('B')
    feats = {}
    for num, _, features in _fields(buf):
        if num != 1:
            continue
        for fnum, _, entry in _fields(features):
            if fnum != 1:
                continue
            key, value = '', b''
            for enum, _, v in _fields(entry):
                if enum == 1:
                    key = bytes(v).decode('utf-8')
                elif enum == 2:
                    value = v
            feats[key] = _parse_feature(value)
    return feats


def decode_jpeg(data):
    """JPEG bytes -> H x W x 3 uint8 RGB."""
    import cv2
    img = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
    if img is None or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError('not a 3-channel JPEG')
    return img[:, :, ::-1].copy()


def read_from_example(serialized_ex, decode_images=True):
    """Returns data from an entry in a test tfrecord (common.py:86-163): N, centers (Nx2), kps (Nx25x3: the 14 LSP points with their
    visibilities, then 5 face and 6 toe points), gt3ds (Nx14x3), images (N decoded RGB frames), im_shapes (Nx2), im_paths (N),
    poses (Nx24x3), scales (N), shape (10), start_pts (Nx2), time_pts (2).  Float features come back as float64 like the reference's
    np.array over TF's Python floats.  decode_images=False leaves `images` as the list of JPEG strings (decode_jpeg decodes one)."""
    feats = parse_example(serialized_ex)

    def get(name):                                  # an absent feature reads as an empty list, like TF's feature map
        return feats[name][1] if name in feats else []

    N = int(get('meta/N')[0])
    im_datas = get('image/encoded')
    xys = np.asarray(get('image/xys'), np.float64).reshape((N, 2, 14))
    vis = np.asarray(get('image/visibilities'), np.float64).reshape((N, 1, 14))
    face_pts = np.asarray(get('image/face_pts'), np.float64).reshape((N, 3, 5))
    toe_pts = np.asarray(get('image/toe_pts'), np.float64).reshape((N, 3, 6))
    kps = np.transpose(np.dstack((np.hstack((xys, vis)), face_pts, toe_pts)), axes=[0, 2, 1])
    return {
        'N': N,
        'centers': np.asarray(get('image/centers')).reshape((N, 2)),
        'kps': kps,
        'gt3ds': np.asarray(get('mosh/gt3ds'), np.float64).reshape((N, -1, 3))[:, :14],
        'images': [decode_jpeg(d) for d in im_datas] if decode_images else list(im_datas),
        'im_shapes': np.asarray(get('image/heightwidths')).reshape((N, 2)),
        'im_paths': list(get('image/filenames')),
        'poses': np.asarray(get('mosh/poses'), np.float64).reshape((N, 24, 3)),
        'scales': np.asarray(get('image/scale_factors'), np.float64),
        'shape': np.asarray(get('mosh/shape'), np.float64),
        'start_pts': np.asarray(get('image/crop_pts')).reshape((N, 2)),
        'time_pts': list(int(t) for t in get('meta/time_pts')),
    }
