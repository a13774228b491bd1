"""Baseline JPEG decoding restated in numpy: the specification `hd_jpeg_decode` (csrc/jpeg.cu) is written against.

It restates what libjpeg's default decompression computes for a baseline (SOF0 / SOF1), Huffman-coded, 8-bit, 3-component YCbCr
stream with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1 -- what `tf.image.decode_jpeg` (TF 1.8, default dct_method,
fancy_upscaling=True) and `cv2.imdecode` both run:

- markers and tables as ITU-T T.81 B.2 defines them; quantisation tables are transmitted in zig-zag order (T.81 A.3.6);
- sequential Huffman decoding (T.81 F.2.2): byte unstuffing of `FF 00`, the DC difference and the AC run/size symbols with EXTEND
  (F.2.2.1), restart markers resetting the DC predictors and byte-aligning the bit stream (F.2.2.5 / E.2.4);
- dequantisation, then libjpeg's `jpeg_idct_islow` (jidctint.c): CONST_BITS = 13, PASS1_BITS = 2, columns then rows, the final
  descale by CONST_BITS + PASS1_BITS + 3 and the range-limit table indexed with `& RANGE_MASK` (jdmaster.c prepare_range_limit_table),
  which wraps far overshoots instead of clamping them;
- libjpeg's "fancy" (triangle) chroma upsampling (jdsample.c): h2v1 as 3/4 * nearer + 1/4 * further with +1 / +2 biases and >> 2;
  h2v2 as column sums 3 * nearer + further, then the same horizontally with +8 / +7 biases and >> 4.  Edges replicate the last real
  sample row or column of the downsampled component (ceil(W / 2) columns, ceil(H / 2) rows), never the MCU padding; a downsampled
  width <= 2 uses plain replication (box) instead;
- the YCbCr -> RGB tables of jdcolor.c build_ycc_rgb_table (SCALEBITS = 16, ONE_HALF rounding) and a clamp to [0, 255].

Test infrastructure only: the Huffman decoding is pure Python, about 0.3 s for a 224^2 video frame at quality 95.
"""
import numpy as np

# T.81 Figure A.6: zig-zag index -> natural (row-major) index
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
                   61, 54, 47, 55, 62, 63], np.int64)
# libjpeg's jpeg_natural_order carries 16 extra entries so that a corrupt run past k = 63 lands on coefficient 63
NATURAL = np.concatenate([ZIGZAG, np.full(16, 63, np.int64)])


class Unsupported(ValueError):
    """A well-formed JPEG outside the supported set (progressive, arithmetic, 12-bit, not 3 components, other sampling)."""


class Invalid(ValueError):
    """Malformed or truncated input."""


def parse(data):
    """Markers of one JPEG -> dict: width, height, h_samp, v_samp (luma), qt / dc / ac (table slot per component), restart_interval,
    data_offset / data_bytes (the entropy-coded data up to the marker that ends the scan), quant {slot: 64 natural-order values},
    dc_tables / ac_tables {slot: (bits[16], vals)}."""
    d = bytes(data)
    n = len(d)
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise Invalid('no SOI')
    pos = 2
    quant, dct, act = {}, {}, {}
    frame = None
    ri = 0
    adobe_transform = None
    while True:
        while pos < n and d[pos] == 0xFF and pos + 1 < n and d[pos + 1] == 0xFF:     # fill bytes
            pos += 1
        if pos + 4 > n or d[pos] != 0xFF:
            raise Invalid('bad marker at %d' % pos)
        m = d[pos + 1]
        seg_len = (d[pos + 2] << 8) | d[pos + 3]
        body, end = pos + 4, pos + 2 + seg_len
        if seg_len < 2 or end > n:
            raise Invalid('truncated segment')
        seg = d[body:end]
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise Invalid('second SOF')
            if len(seg) < 6:
                raise Invalid('short SOF')
            prec, H, W, nc = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if len(seg) < 6 + 3 * nc:
                raise Invalid('short SOF')
            if prec != 8 or nc != 3:
                raise Unsupported('precision %d, %d components' % (prec, nc))
            if H == 0 or W == 0:
                raise Unsupported('DNL-defined height or zero width')
            if H * W > 2 ** 31 - 1:
                raise Unsupported('more than 2^31 - 1 pixels')
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(3)]
            hs, vs = comps[0][1], comps[0][2]
            if (hs, vs) not in ((1, 1), (2, 1), (2, 2)) or any((c[1], c[2]) != (1, 1) for c in comps[1:]):
                raise Unsupported('sampling')
            if any(c[3] > 3 for c in comps):
                raise Invalid('quant table id')
            if [c[0] for c in comps] == [82, 71, 66]:
                raise Unsupported('RGB component ids')
            frame = dict(width=W, height=H, h_samp=hs, v_samp=vs, ids=[c[0] for c in comps], qt=[c[3] for c in comps])
        elif m in (0xC2, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF):
            raise Unsupported('SOF%d' % (m - 0xC0))
        elif m == 0xC4:
            p = 0
            while p < len(seg):
                if p + 17 > len(seg):
                    raise Invalid('short DHT')
                tc, th = seg[p] >> 4, seg[p] & 15
                bits = list(seg[p + 1:p + 17])
                cnt = sum(bits)
                if tc > 1 or th > 3 or cnt > 256 or p + 17 + cnt > len(seg):
                    raise Invalid('bad DHT')
                vals = list(seg[p + 17:p + 17 + cnt])
                _check_huffman(bits, vals, tc == 0)
                (dct if tc == 0 else act)[th] = (bits, vals)
                p += 17 + cnt
        elif m == 0xDB:
            p = 0
            while p < len(seg):
                pq, tq = seg[p] >> 4, seg[p] & 15
                size = 64 * (pq + 1)
                if pq > 1 or tq > 3 or p + 1 + size > len(seg):
                    raise Invalid('bad DQT')
                raw = np.frombuffer(seg[p + 1:p + 1 + size], np.uint8 if pq == 0 else '>u2').astype(np.int64)
                q = np.zeros(64, np.int64)
                q[ZIGZAG] = raw
                quant[tq] = q
                p += 1 + size
        elif m == 0xDD:
            if len(seg) < 2:
                raise Invalid('short DRI')
            ri = (seg[0] << 8) | seg[1]
        elif m == 0xEE and len(seg) >= 12 and seg[:5] == b'Adobe':
            adobe_transform = seg[11]
        elif m == 0xDA:
            if frame is None:
                raise Invalid('SOS before SOF')
            ns = seg[0] if seg else 0
            if ns != 3 or len(seg) < 1 + 2 * ns + 3:
                raise Unsupported('scan with %d components' % ns)
            sel = [seg[1 + 2 * i] for i in range(3)]
            if sel != frame['ids']:
                raise Unsupported('scan component order')
            dc = [seg[2 + 2 * i] >> 4 for i in range(3)]
            ac = [seg[2 + 2 * i] & 15 for i in range(3)]
            ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if ss != 0 or se != 63 or ahal != 0:
                raise Invalid('spectral selection in a sequential scan')
            if adobe_transform == 0:
                raise Unsupported('Adobe RGB')
            for c in range(3):
                if frame['qt'][c] not in quant or dc[c] not in dct or ac[c] not in act:
                    raise Invalid('scan uses an undefined table')
            start = end
            q = start
            while True:                                   # the scan ends at the first marker other than RSTn
                q = d.find(b'\xff', q)
                if q < 0 or q + 1 >= n:
                    raise Invalid('entropy-coded data runs to the end of the stream')
                nxt = d[q + 1]
                if nxt == 0x00 or 0xD0 <= nxt <= 0xD7:
                    q += 2
                elif nxt == 0xFF:
                    q += 1
                else:
                    break
            if d[q + 1] != 0xD9:
                raise Unsupported('more than one scan')
            while q > start and d[q - 1] == 0xFF:      # fill bytes before EOI (T.81 B.1.1.2); a data FF is always stuffed
                q -= 1
            return dict(width=frame['width'], height=frame['height'], h_samp=frame['h_samp'], v_samp=frame['v_samp'],
                        qt=frame['qt'], dc=dc, ac=ac, restart_interval=ri, data_offset=start, data_bytes=q - start,
                        quant={k: quant[k] for k in set(frame['qt'])}, dc_tables={k: dct[k] for k in set(dc)},
                        ac_tables={k: act[k] for k in set(ac)})
        elif m == 0xD9:
            raise Invalid('EOI before SOS')
        elif 0xD0 <= m <= 0xD7 or m == 0x01:
            raise Invalid('stray marker')
        pos = end


def _check_huffman(bits, vals, is_dc):
    """jdhuff.c jpeg_make_d_derived_tbl's checks: the code lengths must fit (no code of length l reaches 2^l), DC symbols <= 15."""
    code = 0
    for ln in range(1, 17):
        code += bits[ln - 1]
        if code > (1 << ln):
            raise Invalid('bad Huffman table')
        code <<= 1
    if is_dc and any(v > 15 for v in vals):
        raise Invalid('DC symbol > 15')


def _derive(table):
    """Canonical codes (T.81 C.2) as a table over the next 16 bits of the stream: entry = (code length << 8) | symbol, or -1 for a
    bit pattern that starts no code."""
    bits, vals = table
    lut = [-1] * 65536
    code, k = 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            lo = code << (16 - ln)
            lut[lo:lo + (1 << (16 - ln))] = [(ln << 8) | vals[k]] * (1 << (16 - ln))
            k += 1
            code += 1
        code <<= 1
    return lut


class _Bits(object):
    """MSB-first bit reader over one entropy-coded segment with FF 00 unstuffed; past the end it reads zeros and records it."""

    def __init__(self, seg):
        out = bytearray()
        i, n = 0, len(seg)
        self.marker = False
        while i < n:
            b = seg[i]
            if b == 0xFF:
                if i + 1 < n and seg[i + 1] == 0x00:
                    i += 2
                else:
                    self.marker = True                   # a marker inside the segment: the data stops here
                    break
            else:
                i += 1
            out.append(b)
        self.nbits = 8 * len(out)
        self.val = int.from_bytes(bytes(out), 'big') if out else 0
        self.pos = 0

    def get(self, k):
        if k == 0:
            return 0
        p = self.pos
        self.pos += k
        if self.pos <= self.nbits:
            return (self.val >> (self.nbits - self.pos)) & ((1 << k) - 1)
        # partly or wholly past the end: zeros
        have = max(self.nbits - p, 0)
        head = (self.val & ((1 << have) - 1)) if have else 0
        return head << (k - have)

    def peek16(self):
        p = self.pos + 16
        if p <= self.nbits:
            return (self.val >> (self.nbits - p)) & 0xFFFF
        have = max(self.nbits - self.pos, 0)
        return ((self.val & ((1 << have) - 1)) << (16 - have)) if have else 0

    def overrun(self):
        return self.pos > self.nbits


def _decode_symbol(br, lut):
    e = lut[br.peek16()]
    if e < 0:
        return None
    br.pos += e >> 8
    return e & 255


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def _segments(d, start, length, n_seg):
    """Split the entropy-coded data at its RSTn markers into n_seg segments; returns (segments, corrupt)."""
    data = d[start:start + length]
    segs, cur, i, n, expect = [], 0, 0, len(data), 0
    corrupt = False
    while i + 1 < n:
        if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7:
            if data[i + 1] != 0xD0 + (expect & 7):
                corrupt = True
            expect += 1
            segs.append(data[cur:i].rstrip(b'\xff'))      # without the fill bytes before the marker
            cur = i + 2
            i += 2
        else:
            i += 1
    segs.append(data[cur:])
    if len(segs) != n_seg:
        corrupt = True
    return segs, corrupt


def block_grid(h, v, H, W):
    """(MCU columns, MCU rows) and the per-component block grid [(bw, bh)] of an interleaved scan."""
    mx, my = -(-W // (8 * h)), -(-H // (8 * v))
    return mx, my, [(mx * h, my * v), (mx, my), (mx, my)]


def entropy_decode(data, hdr):
    """Quantised coefficients [(bh, bw, 64) int64 natural order per component] and a corrupt flag (bad code, overrun, marker out of
    place).  Corrupt data leaves the rest of its segment's blocks zero."""
    h, v, H, W = hdr['h_samp'], hdr['v_samp'], hdr['height'], hdr['width']
    mx, my, grid = block_grid(h, v, H, W)
    coef = [np.zeros((bh, bw, 64), np.int64) for bw, bh in grid]
    n_mcu = mx * my
    ri = hdr['restart_interval'] or n_mcu
    n_seg = -(-n_mcu // ri)
    segs, corrupt = _segments(bytes(data), hdr['data_offset'], hdr['data_bytes'], n_seg)
    dcl = [_derive(hdr['dc_tables'][t]) for t in hdr['dc']]
    acl = [_derive(hdr['ac_tables'][t]) for t in hdr['ac']]
    layout = [(0, yy, xx) for yy in range(v) for xx in range(h)] + [(1, 0, 0), (2, 0, 0)]
    for s in range(n_seg):
        if s >= len(segs):
            break
        br = _Bits(segs[s])
        corrupt |= br.marker
        pred = [0, 0, 0]
        bad = False
        for m in range(s * ri, min((s + 1) * ri, n_mcu)):
            my_, mx_ = divmod(m, mx)
            for c, yy, xx in layout:
                t = _decode_symbol(br, dcl[c])
                if t is None:
                    bad = True
                    break
                diff = _extend(br.get(t), t)
                pred[c] += diff
                blk = np.zeros(64, np.int64)
                blk[0] = np.int16(np.int64(pred[c]).astype(np.int16))
                k = 1
                while k < 64:
                    rs = _decode_symbol(br, acl[c])
                    if rs is None:
                        bad = True
                        break
                    r, sz = rs >> 4, rs & 15
                    if sz:
                        k += r
                        blk[NATURAL[k]] = _extend(br.get(sz), sz)
                    else:
                        if r != 15:
                            break
                        k += 15
                    k += 1
                if bad:
                    break
                bh_, bw_ = (my_ * v + yy, mx_ * h + xx) if c == 0 else (my_, mx_)
                coef[c][bh_, bw_] = blk
            if bad:
                break
        corrupt |= bad or br.overrun()
    return coef, corrupt


# --------------------------------------------------------------------------------------------------------- jidctint.c islow
CONST_BITS, PASS1_BITS = 13, 2
FIX_0_298631336, FIX_0_390180644, FIX_0_541196100, FIX_0_765366865 = 2446, 3196, 4433, 6270
FIX_0_899976223, FIX_1_175875602, FIX_1_501321110, FIX_1_847759065 = 7373, 9633, 12299, 15137
FIX_1_961570560, FIX_2_053119869, FIX_2_562915447, FIX_3_072711026 = 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(s0, s1, s2, s3, s4, s5, s6, s7):
    """The even / odd butterflies shared by both passes of jpeg_idct_islow; returns the eight outputs before descaling."""
    z1 = (s2 + s6) * FIX_0_541196100
    tmp2 = z1 + s6 * -FIX_1_847759065
    tmp3 = z1 + s2 * FIX_0_765366865
    tmp0 = (s0 + s4) << CONST_BITS
    tmp1 = (s0 - s4) << CONST_BITS
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = s7, s5, s3, s1
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * FIX_1_175875602
    t0, t1, t2, t3 = t0 * FIX_0_298631336, t1 * FIX_2_053119869, t2 * FIX_3_072711026, t3 * FIX_1_501321110
    z1, z2 = z1 * -FIX_0_899976223, z2 * -FIX_2_562915447
    z3, z4 = z3 * -FIX_1_961570560 + z5, z4 * -FIX_0_390180644 + z5
    t0 += z1 + z3
    t1 += z2 + z4
    t2 += z2 + z3
    t3 += z1 + z4
    return [tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0, tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3]


def idct_range_limit(x):
    """range_limit[x & RANGE_MASK] of jpeg_idct_islow (IDCT_range_limit = sample_range_limit + CENTERJSAMPLE): x centred on 0;
    [-128, 127] -> x + 128, [128, 511] -> 255, [512, 895] -> 0, and the pattern repeats modulo 1024."""
    u = (np.asarray(x, np.int64) + 128) & 1023
    return np.where(u < 256, u, np.where(u < 640, 255, 0)).astype(np.uint8)


def idct_islow(coef, q):
    """coef [..., 64] quantised (natural order), q [64] -> [..., 8, 8] uint8 samples."""
    x = np.asarray(coef, np.int64) * np.asarray(q, np.int64)
    x = x.reshape(x.shape[:-1] + (8, 8))                   # [..., row (v), col (u)]
    cols = _idct_1d(*[x[..., r, :] for r in range(8)])      # pass 1: each column, from rows 0..7
    ws = np.stack([_descale(c, CONST_BITS - PASS1_BITS) for c in cols], axis=-2)
    rows = _idct_1d(*[ws[..., :, c] for c in range(8)])     # pass 2: each row
    out = np.stack([_descale(r, CONST_BITS + PASS1_BITS + 3) for r in rows], axis=-1)
    return idct_range_limit(out)


def planes(coef, hdr):
    """Sample planes [(bh*8, bw*8) uint8] of the three components (MCU padding included)."""
    out = []
    for c, blocks in enumerate(coef):
        s = idct_islow(blocks, hdr['quant'][hdr['qt'][c]])       # [bh, bw, 8, 8]
        bh, bw = blocks.shape[:2]
        out.append(s.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8))
    return out


# --------------------------------------------------------------------------------------------------------- jdsample.c fancy
def upsample(plane, h, v, H, W):
    """One chroma plane -> [H, W] int64, libjpeg's fancy upsampling for (h, v) = (1, 1), (2, 1), (2, 2) luma sampling."""
    if (h, v) == (1, 1):
        return plane[:H, :W].astype(np.int64)
    dw = -(-W // 2)
    dh = -(-H // v)
    p = plane[:dh, :dw].astype(np.int64)
    if dw <= 2:                                             # plain replication
        return np.repeat(np.repeat(p, 2, axis=1), v, axis=0)[:H, :W]
    left = np.concatenate([p[:, :1], p[:, :-1]], axis=1)
    right = np.concatenate([p[:, 1:], p[:, -1:]], axis=1)
    out = np.empty((p.shape[0], 2 * dw), np.int64)
    if v == 1:                                              # h2v1
        out[:, 0::2] = (3 * p + left + 1) >> 2
        out[:, 1::2] = (3 * p + right + 2) >> 2
        return out[:H, :W]
    up = np.concatenate([p[:1], p[:-1]], axis=0)
    down = np.concatenate([p[1:], p[-1:]], axis=0)
    rows = np.empty((2 * dh, dw), np.int64)
    rows[0::2] = 3 * p + up                                 # output row 2r: nearer row r, further row r - 1
    rows[1::2] = 3 * p + down                               # output row 2r + 1: further row r + 1
    left = np.concatenate([rows[:, :1], rows[:, :-1]], axis=1)
    right = np.concatenate([rows[:, 1:], rows[:, -1:]], axis=1)
    out = np.empty((2 * dh, 2 * dw), np.int64)
    out[:, 0::2] = (3 * rows + left + 8) >> 4
    out[:, 1::2] = (3 * rows + right + 7) >> 4
    return out[:H, :W]


# --------------------------------------------------------------------------------------------------------- jdcolor.c
SCALEBITS = 16
ONE_HALF = 1 << (SCALEBITS - 1)


def _fix(x):
    return int(x * (1 << SCALEBITS) + 0.5)


_X = np.arange(256, dtype=np.int64) - 128
CR_R = (_fix(1.40200) * _X + ONE_HALF) >> SCALEBITS
CB_B = (_fix(1.77200) * _X + ONE_HALF) >> SCALEBITS
CR_G = -_fix(0.71414) * _X
CB_G = -_fix(0.34414) * _X + ONE_HALF


def ycc_to_rgb(y, cb, cr):
    y = np.asarray(y, np.int64)
    r = y + CR_R[cr]
    g = y + ((CB_G[cb] + CR_G[cr]) >> SCALEBITS)
    b = y + CB_B[cb]
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def decode(data, return_corrupt=False):
    """JPEG bytes -> H x W x 3 uint8 RGB (and, with return_corrupt, whether the entropy-coded data was corrupt)."""
    hdr = parse(data)
    coef, corrupt = entropy_decode(data, hdr)
    y, cb, cr = planes(coef, hdr)
    H, W, h, v = hdr['height'], hdr['width'], hdr['h_samp'], hdr['v_samp']
    rgb = ycc_to_rgb(y[:H, :W], upsample(cb, h, v, H, W), upsample(cr, h, v, H, W))
    return (rgb, corrupt) if return_corrupt else rgb


# --------------------------------------------------------------------------------------------------------- test cases
SAMPLINGS = ('444', '422', '420')


def make_image(H, W, seed, kind='photo'):
    """A seeded H x W x 3 uint8 BGR image: 'photo' (smooth gradients, blobs and mild noise, like a video frame), 'noise' (uniform) or
    'saturated' (random 0 / 255 pixels, grey: at quality 100 the IDCT then overshoots [0, 255] and the range-limit table decides)."""
    rs = np.random.RandomState(seed)
    if kind == 'noise':
        return rs.randint(0, 256, size=(H, W, 3)).astype(np.uint8)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    if kind == 'saturated':
        return np.repeat(((rs.rand(H, W) > 0.5) * 255)[..., None], 3, axis=2).astype(np.uint8)
    img = np.zeros((H, W, 3))
    for c in range(3):
        a, b, ph = rs.uniform(0.02, 0.3, size=3)
        img[..., c] = 128 + 80 * np.sin(a * xx + b * yy + 6 * ph)
        for _ in range(3):
            cy, cx, r = rs.uniform(0, H), rs.uniform(0, W), rs.uniform(2, max(3, min(H, W) / 3))
            img[..., c] += rs.uniform(-90, 90) * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r))
    img += rs.normal(0, 6, size=img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def encode(img, quality=95, sampling='420', optimize=False, rst=0, progressive=False):
    """cv2.imencode of a BGR (or grayscale) image with the given quality, chroma sampling ('444', '422', '420', '411', '440'),
    optimised Huffman tables, restart interval (MCUs) and progressive coding."""
    import cv2
    sf = {'444': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, '422': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
          '420': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, '411': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411,
          '440': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440}[sampling]
    params = [cv2.IMWRITE_JPEG_QUALITY, int(quality), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sf,
              cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize), cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)]
    if rst:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, int(rst)]
    ok, buf = cv2.imencode('.jpg', img, params)
    assert ok
    return buf.tobytes()


def cv2_decode(data):
    """The live reference: cv2.imdecode (libjpeg-turbo), BGR -> RGB."""
    import cv2
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)[:, :, ::-1]


def add_fill_bytes(data, n=2):
    """The same JPEG with n fill bytes (FF, T.81 B.1.1.2) before every restart marker and before EOI: a valid stream libjpeg skips them in."""
    h = parse(data)
    a, b = h['data_offset'], h['data_offset'] + h['data_bytes']
    seg = data[a:b]
    for m in range(0xD0, 0xD8):
        seg = seg.replace(bytes([0xFF, m]), b'\xff' * (n + 1) + bytes([m]))
    return data[:a] + seg + b'\xff' * n + data[b:]
