"""JPEG decoding on the GPU, bit for bit what libjpeg's default decompression gives (`cv2.imdecode`, `tf.image.decode_jpeg`).

`decode(jpegs)` takes a list of JPEG byte strings of one size and returns a uint8 CUDA tensor (N, H, W, 3) in RGB, the layout
`hd_process_image` and `hd_tube_augment` take.  Supported: baseline (SOF0 / SOF1) Huffman-coded 8-bit YCbCr with 4:4:4, 4:2:2 or
4:2:0 sampling, with or without restart intervals -- what OpenCV, PIL and TF's encoders write by default.  The markers are parsed on
the host by `hd_jpeg_parse` (C); the compressed bytes go up in one pinned host-to-device copy (about a sixth of the decoded frames'
bytes); then `hd_jpeg_decode` runs four launches per chunk of frames, the chunks bounding the coefficient workspace.

An unsupported or malformed stream, or a batch of mixed sizes or samplings, raises UnsupportedJPEG before anything is launched.
Corrupt entropy-coded data (a bad Huffman code, data that runs out, a marker out of place) is found on the device: `decode`
synchronises once and raises CorruptJPEG naming the images; `decode_with_status` returns the status words instead.  Both are HDErrors;
any other HDError (a failed launch, no CUDA device) is a fault of the call, not of the data.  There is no CPU fallback.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import HDError, lib

WORKSPACE_BUDGET = 1 << 30      # bytes of decoder workspace per chunk (a 224^2 4:2:0 frame needs 0.24 MB, a 300^2 one 0.42 MB)
_HDR = C.sizeof(_lib.JpegHeader)
_HUFF = C.sizeof(_lib.JpegHuffman)
_STATUS_BITS = ((_lib.HD_JPEG_BAD_CODE, 'bad Huffman code'), (_lib.HD_JPEG_OVERRUN, 'data overrun'),
                (_lib.HD_JPEG_MARKER, 'marker out of place'), (_lib.HD_JPEG_BAD_HEADER, 'bad header'))


class UnsupportedJPEG(HDError):
    """Input the GPU decoder does not take: a stream hd_jpeg_parse refuses (unsupported or malformed), or a batch of mixed sizes or
    samplings.  Nothing was launched."""


class CorruptJPEG(HDError):
    """Corrupt entropy-coded data in the images `indices` (their status words in `status`)."""

    def __init__(self, indices, status):
        self.indices, self.status = list(indices), list(status)
        why = ['%d (%s)' % (i, ', '.join(n for b, n in _STATUS_BITS if s & b)) for i, s in zip(self.indices, self.status)]
        super(CorruptJPEG, self).__init__('corrupt JPEG data in image(s) %s' % ', '.join(why))


def parse(data):
    """hd_jpeg_parse on one JPEG: (JpegHeader, JpegTables); UnsupportedJPEG if it is unsupported or malformed."""
    hdr, tab = _lib.JpegHeader(), _lib.JpegTables()
    _parse_into(bytes(data), hdr, tab, 0)
    return hdr, tab


def _parse_into(data, hdr, tab, index):
    rc = lib.hd_jpeg_parse(data, len(data), C.byref(hdr), C.byref(tab))
    if rc != 0:
        raise UnsupportedJPEG('JPEG %d: %s [%s]' % (index, lib.hd_status_string(rc).decode(), lib.hd_last_error().decode()))


def _intern(table, key, blob):
    i = table.get(key)
    if i is None:
        i = table[key] = len(table)
        blob.append(key)
    return i


def workspace_bytes(n, H, W, h_samp, v_samp):
    return int(lib.hd_jpeg_workspace_bytes(n, H, W, h_samp, v_samp))


def decode_with_status(jpegs, device=None, chunk=None, out=None):
    """(uint8 CUDA tensor (N, H, W, 3), int32 CUDA tensor (N,) of status words) without synchronising.  `chunk` caps the frames per
    launch group (default: as many as WORKSPACE_BUDGET allows); the result does not depend on it.  `out`: a contiguous uint8 CUDA tensor
    (N, H, W, 3) on the device to decode into (its device is then the device), instead of a new one."""
    jpegs = [bytes(j) for j in jpegs]
    N = len(jpegs)
    if N == 0:
        raise UnsupportedJPEG('jpeg.decode: no images')
    if out is not None:
        device = out.device
    if not torch.cuda.is_available():
        raise HDError('jpeg.decode: no CUDA device (there is no CPU fallback; src.datasets.common.decode_jpeg decodes on the host)')
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    if dev.type != 'cuda':
        raise HDError('jpeg.decode: expected a CUDA device (no CPU fallback exists), got %s' % dev)

    # ---- host: parse every image, intern its tables, lay out one upload
    hdrs = (_lib.JpegHeader * N)()
    tab = _lib.JpegTables()
    keys = []                                   # per image: the bytes of its 3 quant, 3 DC and 3 AC tables
    offsets = np.zeros(N + 1, np.int64)
    for i, d in enumerate(jpegs):
        h = hdrs[i]
        _parse_into(d, h, tab, i)
        keys.append([bytes(tab.quant[h.qt[c]]) for c in range(3)] + [bytes(tab.dc[h.dc[c]]) for c in range(3)] +
                    [bytes(tab.ac[h.ac[c]]) for c in range(3)])
        h.data_offset += int(offsets[i])
        offsets[i + 1] = offsets[i] + len(d)
    h0 = hdrs[0]
    H, W, hs, vs = h0.height, h0.width, h0.h_samp, h0.v_samp
    for i in range(1, N):
        h = hdrs[i]
        if (h.height, h.width, h.h_samp, h.v_samp) != (H, W, hs, vs):
            raise UnsupportedJPEG('jpeg.decode: image %d is %dx%d with %dx%d luma sampling, image 0 is %dx%d with %dx%d: one batch '
                                  'has one size and sampling' % (i, h.height, h.width, h.h_samp, h.v_samp, H, W, hs, vs))
    per_image = workspace_bytes(1, H, W, hs, vs)
    if per_image == 0:
        raise UnsupportedJPEG('jpeg.decode: %dx%d frames are outside hd_jpeg_decode\'s size contract' % (H, W))
    step = max(1, min(N, chunk or N, WORKSPACE_BUDGET // per_image))
    while workspace_bytes(step, H, W, hs, vs) == 0:          # keep every launch's grid within its limit
        step = (step + 1) // 2

    chunks = []                                 # (start, count, quant bytes, huffman bytes, n_quant, n_huff)
    for s in range(0, N, step):
        qt_ids, hf_ids, qt_blob, hf_blob = {}, {}, [], []
        for i in range(s, min(N, s + step)):
            k, h = keys[i], hdrs[i]
            for c in range(3):
                h.qt[c] = _intern(qt_ids, k[c], qt_blob)
                h.dc[c] = _intern(hf_ids, k[3 + c], hf_blob)
                h.ac[c] = _intern(hf_ids, k[6 + c], hf_blob)
        chunks.append((s, min(step, N - s), b''.join(qt_blob), b''.join(hf_blob), len(qt_blob), len(hf_blob)))

    def up(n):
        return (n + 255) // 256 * 256
    data_bytes = int(offsets[N])
    pos = up(data_bytes)
    hdr_at = pos
    pos += up(N * _HDR)
    table_at = []
    for c in chunks:
        table_at.append((pos, pos + up(len(c[2]))))
        pos += up(len(c[2])) + up(len(c[3]))
    host = torch.empty(pos, dtype=torch.uint8, pin_memory=True)
    buf = host.numpy()
    for i, d in enumerate(jpegs):
        buf[offsets[i]:offsets[i + 1]] = np.frombuffer(d, np.uint8)
    buf[hdr_at:hdr_at + N * _HDR] = np.frombuffer(hdrs, np.uint8)
    for (q_at, h_at), c in zip(table_at, chunks):
        buf[q_at:q_at + len(c[2])] = np.frombuffer(c[2], np.uint8)
        buf[h_at:h_at + len(c[3])] = np.frombuffer(c[3], np.uint8)

    # ---- device: one upload, then four launches per chunk
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev)
        blob = host.to(dev, non_blocking=True)
        if out is None:
            out = torch.empty((N, H, W, 3), dtype=torch.uint8, device=dev)
        elif out.dtype != torch.uint8 or tuple(out.shape) != (N, H, W, 3) or not out.is_contiguous():
            raise HDError('jpeg.decode: out must be a contiguous uint8 tensor (%d, %d, %d, 3)' % (N, H, W))
        status = torch.empty(N, dtype=torch.int32, device=dev)
        ws_bytes = workspace_bytes(step, H, W, hs, vs)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        base = blob.data_ptr()
        for (q_at, h_at), (s, n, _, _, nq, nh) in zip(table_at, chunks):
            _lib.check(lib.hd_jpeg_decode(C.c_void_p(base), data_bytes, C.c_void_p(base + hdr_at + s * _HDR), n, H, W, hs, vs,
                                          C.c_void_p(base + q_at), nq, C.c_void_p(base + h_at), nh,
                                          C.c_void_p(out.data_ptr() + s * H * W * 3), C.c_void_p(status.data_ptr() + 4 * s),
                                          C.c_void_p(ws.data_ptr()), ws_bytes, C.c_void_p(stream.cuda_stream)), 'hd_jpeg_decode')
    return out, status


def decode(jpegs, device=None, check=True, chunk=None, out=None):
    """JPEG byte strings of one size -> uint8 CUDA tensor (N, H, W, 3), RGB (`out` if given).  With `check` (default) it synchronises
    once and raises CorruptJPEG if the device flagged any image; without, a corrupt image's pixels are unspecified and nothing is
    reported."""
    out, status = decode_with_status(jpegs, device=device, chunk=chunk, out=out)
    if check:
        st = status.cpu().numpy()
        bad = np.nonzero(st)[0]
        if len(bad):
            raise CorruptJPEG(bad.tolist(), st[bad].tolist())
    return out
