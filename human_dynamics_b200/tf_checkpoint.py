"""Pure-Python reader (and writer) of TensorFlow V2 checkpoints ("tensor bundles") -- no TensorFlow needed.

The reference restores its weights with `tf.train.Saver.restore(sess, load_path)` after checking that
`load_path + '.index'` exists (src/evaluation/tester.py:35-38, 92-116); the published HMMR / HMR models ship only in that
form (`model.ckpt-NNNN.index` + `model.ckpt-NNNN.data-00000-of-00001`).  TensorFlow 1.8 cannot be installed next to
this package, so the bundle is parsed directly and turned into the TF-named dict of numpy arrays the engine consumes
(SURVEY.md A.6).

Format (tensorflow/core/util/tensor_bundle + core/lib/io/table, stable since TF 0.12):
  <prefix>.index   an SSTable in the LevelDB table format: data blocks of prefix-compressed (key, value) entries, an
                   index block, and a 48-byte footer ending in the magic 0xdb4775248b80fb57.  Key "" holds a
                   BundleHeaderProto, every other key is a variable name whose value is a BundleEntryProto
                   {dtype, shape, shard_id, offset, size, crc32c}.
  <prefix>.data-SSSSS-of-NNNNN   raw little-endian tensor bytes, addressed by (shard_id, offset, size).
Block trailer: 1 byte compression type (0 = none; TF writes bundles uncompressed) + 4 bytes masked CRC-32C.

PARITY NOTE: no TensorFlow-written checkpoint exists in this container, so the reader is verified against the writer in
this file and against hand-assembled bytes (tests/test_assets.py) -- written from the format description above.
"""
from __future__ import annotations

import os
import struct

import numpy as np

TABLE_MAGIC = 0xdb4775248b80fb57
FOOTER_LEN = 48
BLOCK_TRAILER = 5

# tensorflow/core/framework/types.proto
_DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 5: np.int16, 6: np.int8, 9: np.int64, 10: np.bool_,
           14: None, 17: np.uint16, 19: np.float16, 22: np.uint32, 23: np.uint64}
_DTYPE_IDS = {np.dtype(v): k for k, v in _DTYPES.items() if v is not None}


# ------------------------------------------------------------------------------------------------ CRC-32C
def _crc_table():
    poly = 0x82F63B78
    t = np.zeros(256, np.uint32)
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ poly if c & 1 else c >> 1
        t[i] = c
    return t


_CRC = _crc_table()


def _crc_bytewise(data, c):
    tab = _CRC
    for b in data:
        c = int(tab[(c ^ b) & 0xFF]) ^ (c >> 8)
    return c


def _zeros_op(n):
    """The 32 x 32 GF(2) map that n zero bytes apply to a CRC register, as its 32 column images (column j = the register 1 << j)."""
    cols = np.array([1 << j for j in range(32)], np.uint64)
    sq = np.array([_crc_bytewise(b'\x00', 1 << j) for j in range(32)], np.uint64)     # one zero byte
    while n:
        if n & 1:
            cols = _apply(sq, cols)
        sq = _apply(sq, sq)
        n >>= 1
    return cols


def _apply(op, x):
    """op (32 column images) applied to every register of x."""
    x = np.asarray(x, np.uint64)
    out = np.zeros_like(x)
    for j in range(32):
        out ^= ((x >> np.uint64(j)) & np.uint64(1)) * op[j]
    return out


def crc32c(data: bytes, crc: int = 0) -> int:
    """CRC-32C (Castagnoli, reflected), as TF's tensor bundles checksum their blocks and tensors.  Long inputs run as many chunks in
    parallel, combined through the zero-byte operator (a CRC from register 0 ignores leading zero bytes, so the data is padded in
    front): a checkpoint holding optimizer slots is gigabytes, which a byte loop in Python takes minutes over."""
    n = len(data)
    if n < 1 << 16:
        return _crc_bytewise(data, crc ^ 0xFFFFFFFF) ^ 0xFFFFFFFF
    L = 4096
    k = -(-n // L)
    buf = np.zeros(k * L, np.uint8)
    buf[k * L - n:] = np.frombuffer(data, np.uint8)
    rows = buf.reshape(k, L)
    tab = _CRC.astype(np.uint32)
    c = np.zeros(k, np.uint32)
    for i in range(L):                               # every chunk's CRC from register 0, one byte position at a time
        c = tab[(c ^ rows[:, i]) & 0xFF] ^ (c >> 8)
    c = c.astype(np.uint64)
    span = L
    while len(c) > 1:                                # pairwise: crc(a || b) = zeros(len b)(crc a) ^ crc b
        if len(c) & 1:
            c = np.concatenate([np.zeros(1, np.uint64), c])     # a leading all-zero chunk changes nothing
        c = _apply(_zeros_op(span), c[0::2]) ^ c[1::2]
        span *= 2
    init = int(_apply(_zeros_op(n), np.array([crc ^ 0xFFFFFFFF], np.uint64))[0])
    return (init ^ int(c[0])) ^ 0xFFFFFFFF


def mask_crc(crc: int) -> int:
    return (((crc >> 15) | (crc << 17)) + 0xa282ead8) & 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------ varints / protobuf
def _get_varint(buf, pos):
    out, shift = 0, 0
    while True:
        b = buf[pos]
        pos += 1
        out |= (b & 0x7F) << shift
        if not b & 0x80:
            return out, pos
        shift += 7
        if shift > 70:
            raise ValueError('malformed varint')


def _put_varint(v):
    out = bytearray()
    v &= (1 << 64) - 1
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _parse_proto(buf):
    """Wire-format walk: yields (field_number, wire_type, value) with bytes for length-delimited fields."""
    pos, n = 0, len(buf)
    while pos < n:
        tag, pos = _get_varint(buf, pos)
        field, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = _get_varint(buf, pos)
        elif wt == 1:
            v = struct.unpack_from('<Q', buf, pos)[0]; pos += 8
        elif wt == 2:
            ln, pos = _get_varint(buf, pos)
            v = bytes(buf[pos:pos + ln]); pos += ln
        elif wt == 5:
            v = struct.unpack_from('<I', buf, pos)[0]; pos += 4
        else:
            raise ValueError('unsupported protobuf wire type %d' % wt)
        yield field, wt, v


def _signed64(v):
    return v - (1 << 64) if v >= (1 << 63) else v


def _parse_shape(buf):
    dims = []
    for f, wt, v in _parse_proto(buf):
        if f == 2 and wt == 2:                       # repeated Dim dim = 2
            size = 0
            for g, wt2, u in _parse_proto(v):
                if g == 1 and wt2 == 0:              # int64 size = 1
                    size = _signed64(u)
            dims.append(size)
        elif f == 3 and wt == 0 and v:               # unknown_rank
            raise ValueError('tensor of unknown rank in checkpoint')
    return tuple(dims)


class BundleEntry(object):
    __slots__ = ('dtype', 'shape', 'shard_id', 'offset', 'size', 'crc32c', 'sliced')

    def __init__(self):
        self.dtype, self.shape, self.shard_id, self.offset, self.size, self.crc32c, self.sliced = 0, (), 0, 0, 0, None, False


def _parse_entry(buf):
    e = BundleEntry()
    for f, wt, v in _parse_proto(buf):
        if f == 1 and wt == 0:
            e.dtype = v
        elif f == 2 and wt == 2:
            e.shape = _parse_shape(v)
        elif f == 3 and wt == 0:
            e.shard_id = v
        elif f == 4 and wt == 0:
            e.offset = _signed64(v)
        elif f == 5 and wt == 0:
            e.size = _signed64(v)
        elif f == 6 and wt == 5:
            e.crc32c = v
        elif f == 7:
            e.sliced = True                          # partitioned variable: not used by this model family
    return e


def _parse_header(buf):
    num_shards, endian = 1, 0
    for f, wt, v in _parse_proto(buf):
        if f == 1 and wt == 0:
            num_shards = v
        elif f == 2 and wt == 0:
            endian = v
    return num_shards, endian


# ------------------------------------------------------------------------------------------------ table
def _read_block(data, offset, size, verify):
    end = offset + size
    if end + BLOCK_TRAILER > len(data):
        raise ValueError('block handle points past the end of the index file')
    body = data[offset:end]
    ctype = data[end]
    if verify:
        want = struct.unpack_from('<I', data, end + 1)[0]
        got = mask_crc(crc32c(data[offset:end + 1]))
        if want != got:
            raise ValueError('index block checksum mismatch (offset %d)' % offset)
    if ctype != 0:
        raise ValueError('compressed index block (type %d): TensorFlow writes tensor bundles uncompressed; '
                         'snappy blocks are not supported' % ctype)
    return body


def _block_entries(block):
    """(key, value) pairs of one block (prefix-compressed keys, restart array at the end)."""
    if len(block) < 4:
        raise ValueError('block too small')
    num_restarts = struct.unpack_from('<I', block, len(block) - 4)[0]
    limit = len(block) - 4 - 4 * num_restarts
    if limit < 0:
        raise ValueError('bad restart array')
    pos, key = 0, b''
    while pos < limit:
        shared, pos = _get_varint(block, pos)
        non_shared, pos = _get_varint(block, pos)
        vlen, pos = _get_varint(block, pos)
        if shared > len(key):
            raise ValueError('corrupt key prefix')
        key = key[:shared] + bytes(block[pos:pos + non_shared])
        pos += non_shared
        yield key, bytes(block[pos:pos + vlen])
        pos += vlen


def read_index(index_path, verify=True):
    """-> (num_shards, {name: BundleEntry}) of `<prefix>.index`."""
    with open(index_path, 'rb') as f:
        data = f.read()
    if len(data) < FOOTER_LEN:
        raise ValueError('%s: too small to be a checkpoint index' % index_path)
    footer = data[-FOOTER_LEN:]
    if struct.unpack_from('<Q', footer, FOOTER_LEN - 8)[0] != TABLE_MAGIC:
        raise ValueError('%s: not a TensorFlow V2 checkpoint index (bad table magic)' % index_path)
    pos = 0
    _mi_off, pos = _get_varint(footer, pos)
    _mi_size, pos = _get_varint(footer, pos)
    idx_off, pos = _get_varint(footer, pos)
    idx_size, pos = _get_varint(footer, pos)
    entries, num_shards, saw_header = {}, 1, False
    for _, handle in _block_entries(_read_block(data, idx_off, idx_size, verify)):
        boff, p = _get_varint(handle, 0)
        bsize, p = _get_varint(handle, p)
        for key, value in _block_entries(_read_block(data, boff, bsize, verify)):
            if key == b'':
                num_shards, endian = _parse_header(value)
                saw_header = True
                if endian != 0:
                    raise ValueError('big-endian checkpoint: not supported')
            else:
                entries[key.decode('utf-8')] = _parse_entry(value)
    if not saw_header:
        raise ValueError('%s: bundle header missing' % index_path)
    return num_shards, entries


def is_checkpoint(prefix):
    """The reference's test for a V2 checkpoint: `load_path + '.index'` exists (tester.py:35)."""
    return isinstance(prefix, str) and os.path.exists(prefix + '.index')


def load_checkpoint(prefix, names=None, skip=None, verify_data=False):
    """{variable name: ndarray} of the V2 checkpoint `prefix` (`prefix.index` + `prefix.data-*`).

    names: optional predicate / collection restricting what is read; skip: predicate for names to leave out (default:
    optimizer slots, discriminator `D_*` variables -- tester.py:163-167 -- and step counters).  verify_data checks every
    tensor's CRC-32C (pure Python, slow: meant for tests and small files).
    """
    num_shards, entries = read_index(prefix + '.index')
    if skip is None:
        def skip(n):
            leaf = n.rsplit('/', 1)[-1]
            return (n.startswith('D_') or leaf in ('Adam', 'Adam_1', 'Momentum', 'ExponentialMovingAverage') or
                    n in ('global_step', 'beta1_power', 'beta2_power', 'beta1_power_1', 'beta2_power_1') or
                    n.startswith('_CHECKPOINTABLE') or n.startswith('save_counter'))
    if names is not None and not callable(names):
        wanted = set(names)
        names = wanted.__contains__
    shards, out = {}, {}
    for name in sorted(entries):
        e = entries[name]
        if (names is not None and not names(name)) or (names is None and skip(name)):
            continue
        if e.sliced:
            raise ValueError('%s is a partitioned variable (tensor slices): not supported' % name)
        dt = _DTYPES.get(e.dtype, None)
        if dt is None:
            if names is not None:
                raise ValueError('%s has unsupported dtype enum %d' % (name, e.dtype))
            continue                                 # strings etc. (e.g. object-graph metadata)
        if e.size == 0:                              # zero-size tensor: nothing to read (its shard may even be an empty file)
            raw = np.zeros(0, np.uint8)
        else:
            if e.shard_id not in shards:
                path = '%s.data-%05d-of-%05d' % (prefix, e.shard_id, num_shards)
                shards[e.shard_id] = np.memmap(path, dtype=np.uint8, mode='r')
            raw = shards[e.shard_id][e.offset:e.offset + e.size]
        count = int(np.prod(e.shape)) if e.shape else 1
        if raw.size != e.size or count * np.dtype(dt).itemsize != e.size:
            raise ValueError('%s: entry size %d does not match shape %s / data file' % (name, e.size, e.shape))
        if verify_data and e.crc32c is not None and mask_crc(crc32c(raw.tobytes())) != e.crc32c:
            raise ValueError('%s: tensor checksum mismatch' % name)
        out[name] = np.frombuffer(raw.tobytes(), dtype=np.dtype(dt).newbyteorder('<')).astype(dt).reshape(e.shape)
    return out


# ------------------------------------------------------------------------------------------------ writer (tests / tooling)
def _proto_field(field, wt, payload):
    return _put_varint((field << 3) | wt) + payload


def _entry_bytes(dtype_id, shape, offset, size, crc):
    dims = b''.join(_proto_field(2, 2, (lambda d: _put_varint(len(d)) + d)(_proto_field(1, 0, _put_varint(int(s))))) for s in shape)
    out = _proto_field(1, 0, _put_varint(dtype_id))
    out += _proto_field(2, 2, _put_varint(len(dims)) + dims)
    if offset:
        out += _proto_field(4, 0, _put_varint(offset))
    out += _proto_field(5, 0, _put_varint(size))
    out += _proto_field(6, 5, struct.pack('<I', crc))
    return out


def _build_block(items, restart_interval=16):
    buf, restarts, last = bytearray(), [], b''
    for i, (k, v) in enumerate(items):
        shared = 0
        if i % restart_interval == 0:
            restarts.append(len(buf))
        else:
            while shared < min(len(k), len(last)) and k[shared] == last[shared]:
                shared += 1
        buf += _put_varint(shared) + _put_varint(len(k) - shared) + _put_varint(len(v)) + k[shared:] + v
        last = k
    if not restarts:
        restarts = [0]
    for r in restarts:
        buf += struct.pack('<I', r)
    buf += struct.pack('<I', len(restarts))
    return bytes(buf)


def save_checkpoint(prefix, tensors, block_size=4096):
    """Write {name: ndarray} as a single-shard V2 checkpoint (the layout tf.train.Saver produces)."""
    names = sorted(tensors, key=lambda s: s.encode('utf-8'))
    data_path = '%s.data-00000-of-00001' % prefix
    records, offset = [], 0
    with open(data_path, 'wb') as f:
        for n in names:
            a = np.asarray(tensors[n], order='C')          # (np.ascontiguousarray would turn a scalar into shape (1,))
            if a.dtype not in _DTYPE_IDS:
                raise ValueError('%s: dtype %s not supported' % (n, a.dtype))
            raw = a.astype(a.dtype.newbyteorder('<')).tobytes()
            f.write(raw)
            records.append((n.encode('utf-8'), _entry_bytes(_DTYPE_IDS[a.dtype], a.shape, offset, len(raw), mask_crc(crc32c(raw)))))
            offset += len(raw)
    header = _proto_field(1, 0, _put_varint(1)) + _proto_field(3, 2, (lambda v: _put_varint(len(v)) + v)(_proto_field(1, 0, _put_varint(1))))
    items = [(b'', header)] + records
    out = bytearray()

    def emit(block):
        off = len(out)
        out.extend(block)
        out.append(0)
        out.extend(struct.pack('<I', mask_crc(crc32c(block + b'\x00'))))
        return _put_varint(off) + _put_varint(len(block))

    index_items, cur, cur_bytes = [], [], 0
    for k, v in items:
        cur.append((k, v))
        cur_bytes += len(k) + len(v) + 3
        if cur_bytes >= block_size:
            index_items.append((cur[-1][0], emit(_build_block(cur))))
            cur, cur_bytes = [], 0
    if cur:
        index_items.append((cur[-1][0], emit(_build_block(cur))))
    meta_handle = emit(_build_block([]))
    index_handle = emit(_build_block(index_items, restart_interval=1))
    footer = meta_handle + index_handle
    footer += b'\x00' * (FOOTER_LEN - 8 - len(footer)) + struct.pack('<Q', TABLE_MAGIC)
    out.extend(footer)
    with open(prefix + '.index', 'wb') as f:
        f.write(bytes(out))
    return prefix
