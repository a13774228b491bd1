"""CPU: the JPEG restatement (oracle/jpeg_ref.py) against cv2.imdecode (libjpeg-turbo) bit for bit, and hd_jpeg_parse (host C in
libhd_b200.so) against the restatement's parse, its refusals and its behaviour on damaged streams."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import jpeg_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cv2 = pytest.importorskip('cv2')

HD_ERR_INVALID, HD_ERR_UNSUPPORTED = 1, 4             # hd_status
SIZES = [(1, 1), (2, 9), (9, 2), (7, 13), (17, 33), (64, 48)]


def _same(data):
    got, want = jpeg_ref.decode(data), jpeg_ref.cv2_decode(data)
    assert got.shape == want.shape and np.array_equal(got, want), \
        ('%d of %d bytes differ' % ((got != want).sum(), got.size)) if got.shape == want.shape else (got.shape, want.shape)


@pytest.mark.parametrize('sampling', jpeg_ref.SAMPLINGS)
@pytest.mark.parametrize('quality', [50, 95, 100])
def test_oracle_equals_cv2_matrix(sampling, quality):
    """Every size, with standard and optimised Huffman tables, without and with restart intervals (1 and 2 MCUs)."""
    for i, (H, W) in enumerate(SIZES):
        img = jpeg_ref.make_image(H, W, seed=31 * i + quality, kind='photo' if i % 2 else 'noise')
        for optimize, rst in ((False, 0), (True, 0), (False, 1), (True, 2)):
            _same(jpeg_ref.encode(img, quality, sampling, optimize=optimize, rst=rst))


@pytest.mark.parametrize('sampling', jpeg_ref.SAMPLINGS)
def test_oracle_equals_cv2_saturated_quality_100(sampling):
    """Random 0 / 255 pixels at quality 100: the IDCT overshoots [0, 255] (checked), so the range-limit table decides the output."""
    for H, W in ((17, 33), (64, 48)):
        data = jpeg_ref.encode(jpeg_ref.make_image(H, W, seed=H, kind='saturated'), 100, sampling)
        hdr = jpeg_ref.parse(data)
        coef, corrupt = jpeg_ref.entropy_decode(data, hdr)
        assert not corrupt
        x = (coef[0] * hdr['quant'][hdr['qt'][0]]).reshape(-1, 8, 8)
        ws = np.stack([jpeg_ref._descale(c, 11) for c in jpeg_ref._idct_1d(*[x[:, r, :] for r in range(8)])], axis=-2)
        pre = np.stack([jpeg_ref._descale(r, 18) for r in jpeg_ref._idct_1d(*[ws[:, :, c] for c in range(8)])], axis=-1)
        assert pre.min() < -128 and pre.max() > 127
        _same(data)


def test_oracle_equals_cv2_224():
    for sampling in jpeg_ref.SAMPLINGS:
        _same(jpeg_ref.encode(jpeg_ref.make_image(224, 224, seed=5), 95, sampling))


def test_range_limit_table():
    """jdmaster.c's post-IDCT table: identity on [-128, 127] (+128), 255 up to 511, 0 from 512 to 895, periodic in 1024."""
    x = np.arange(-2048, 2048)
    got = jpeg_ref.idct_range_limit(x).astype(np.int64)
    u = x & 1023
    want = np.where(u < 128, u + 128, np.where(u < 512, 255, np.where(u < 896, 0, u - 896)))
    assert np.array_equal(got, want)


def test_oracle_equals_cv2_on_eval_fixture():
    from src.datasets.common import read_from_example, tf_record_iterator
    n = 0
    for rec in tf_record_iterator(os.path.join(ROOT, 'tests', 'golden', 'eval_v1.tfrecord')):
        for data in read_from_example(rec, decode_images=False)['images']:
            hdr = jpeg_ref.parse(data)
            assert (hdr['height'], hdr['width'], hdr['h_samp'], hdr['v_samp'], hdr['restart_interval']) == (224, 224, 2, 2, 0)
            _same(data)
            n += 1
    assert n == 10


# ------------------------------------------------------------------------------------------------------------------ hd_jpeg_parse
def _parse(data):
    from human_dynamics_b200 import _lib
    hdr, tab = _lib.JpegHeader(), _lib.JpegTables()
    buf = C.create_string_buffer(bytes(data), len(data))      # exactly len(data) bytes: the parser must stay inside them
    rc = _lib.lib.hd_jpeg_parse(buf, len(data), C.byref(hdr), C.byref(tab))
    return rc, hdr, tab


@pytest.mark.parametrize('sampling', jpeg_ref.SAMPLINGS)
def test_parse_agrees_with_oracle(sampling):
    for i, (H, W) in enumerate(SIZES + [(224, 224), (300, 300)]):
        for optimize, rst, q in ((False, 0, 95), (True, 3, 50), (False, 1, 100)):
            data = jpeg_ref.encode(jpeg_ref.make_image(H, W, seed=i), q, sampling, optimize=optimize, rst=rst)
            rc, h, t = _parse(data)
            r = jpeg_ref.parse(data)
            assert rc == 0
            assert (h.width, h.height, h.h_samp, h.v_samp, h.restart_interval, h.data_offset, h.data_bytes) == \
                (r['width'], r['height'], r['h_samp'], r['v_samp'], r['restart_interval'], r['data_offset'], r['data_bytes'])
            assert list(h.qt) == r['qt'] and list(h.dc) == r['dc'] and list(h.ac) == r['ac']
            for s, qv in r['quant'].items():
                assert t.quant_defined >> s & 1 and list(t.quant[s]) == list(qv)
            for mine, theirs, mask in ((t.dc, r['dc_tables'], t.dc_defined), (t.ac, r['ac_tables'], t.ac_defined)):
                for s, (bits, vals) in theirs.items():
                    assert mask >> s & 1 and list(mine[s].bits) == bits and list(mine[s].vals)[:len(vals)] == vals


def test_parse_refuses_unsupported():
    img = jpeg_ref.make_image(32, 48, seed=3)
    cases = {
        'progressive': jpeg_ref.encode(img, 90, '420', progressive=True),
        'grayscale': jpeg_ref.encode(img[:, :, 0], 90),
        '4:1:1': jpeg_ref.encode(img, 90, '411'),
        '4:4:0': jpeg_ref.encode(img, 90, '440'),
    }
    for name, data in cases.items():
        rc, _, _ = _parse(data)
        assert rc == HD_ERR_UNSUPPORTED, name
        with pytest.raises(jpeg_ref.Unsupported):
            jpeg_ref.parse(data)


def test_parse_damaged_streams_return_a_status():
    """Every truncation, and random byte flips, give a status (never a crash or a read outside the buffer); a stream the parser
    accepts is one the oracle's parse accepts with the same header."""
    data = jpeg_ref.encode(jpeg_ref.make_image(40, 56, seed=9), 90, '420', rst=2)
    for n in range(len(data)):
        rc, _, _ = _parse(data[:n])
        assert rc == HD_ERR_INVALID, n
    rs = np.random.RandomState(0)
    seen = set()
    for trial in range(3000):
        b = bytearray(data)
        for _ in range(1 + trial % 3):
            b[rs.randint(len(b))] = rs.randint(256)
        rc, h, _ = _parse(b)
        seen.add(rc)
        assert rc in (0, HD_ERR_INVALID, HD_ERR_UNSUPPORTED)
        if rc == 0:
            r = jpeg_ref.parse(bytes(b))
            assert (h.width, h.height, h.data_offset, h.data_bytes) == (r['width'], r['height'], r['data_offset'], r['data_bytes'])
    assert seen >= {0, HD_ERR_INVALID}


def test_workspace_bytes():
    from human_dynamics_b200 import _lib
    ws = _lib.lib.hd_jpeg_workspace_bytes
    assert ws(0, 224, 224, 2, 2) == 0 and ws(1, 224, 224, 1, 2) == 0 and ws(1, 0, 224, 2, 2) == 0
    blocks = 14 * 14 * 6                                     # 4:2:0 224^2: 196 MCUs of 6 blocks
    assert ws(1, 224, 224, 2, 2) >= blocks * 64 * 3          # int16 coefficients + uint8 samples
    assert ws(160, 224, 224, 2, 2) >= 160 * blocks * 64 * 3


@pytest.mark.parametrize('sampling', jpeg_ref.SAMPLINGS)
def test_fill_bytes_before_markers(sampling):
    """Fill bytes before RSTn and EOI are not data: the oracle equals cv2 on such streams, and hd_jpeg_parse leaves them out of
    data_bytes exactly as the oracle's parse does."""
    for rst in (0, 1, 3):
        plain = jpeg_ref.encode(jpeg_ref.make_image(40, 56, seed=rst), 90, sampling, rst=rst)
        data = jpeg_ref.add_fill_bytes(plain, n=3)
        assert len(data) > len(plain)
        _same(data)
        rc, h, _ = _parse(data)
        r = jpeg_ref.parse(data)
        assert rc == 0 and (h.data_offset, h.data_bytes) == (r['data_offset'], r['data_bytes'])
        assert data[h.data_offset + h.data_bytes - 1] != 0xFF


def _with_size(data, H, W):
    """The same stream with its SOF0 height and width fields rewritten."""
    b = bytearray(data)
    at = bytes(b).index(b'\xff\xc0')
    b[at + 5:at + 9] = bytes([H >> 8, H & 255, W >> 8, W & 255])
    return bytes(b)


def test_size_contract():
    """H * W <= 2^31 - 1 pixels per image, and each launch's grid within 2^31 - 1 blocks: the parser refuses larger frames
    (HD_ERR_UNSUPPORTED), hd_jpeg_workspace_bytes returns 0 and hd_jpeg_decode refuses the call before touching a device."""
    from human_dynamics_b200 import _lib
    lib = _lib.lib
    data = jpeg_ref.encode(jpeg_ref.make_image(16, 16, seed=1), 90, '420')
    assert _parse(_with_size(data, 46340, 46340))[0] == 0                     # 2 147 395 600 pixels
    assert _parse(_with_size(data, 46341, 46341))[0] == HD_ERR_UNSUPPORTED    # 2 147 488 281 pixels
    assert _parse(_with_size(data, 65535, 65535))[0] == HD_ERR_UNSUPPORTED
    assert lib.hd_jpeg_workspace_bytes(1, 46340, 46340, 2, 2) > 0
    assert lib.hd_jpeg_workspace_bytes(1, 46341, 46341, 2, 2) == 0
    assert lib.hd_jpeg_workspace_bytes(1, 65535, 32768, 1, 1) > 0 and lib.hd_jpeg_workspace_bytes(1, 65535, 32769, 1, 1) == 0
    n_max = (2 ** 31 - 1) * 256 // (224 * 224)                                # the colour kernel's grid bounds N at 224^2
    assert lib.hd_jpeg_workspace_bytes(n_max, 224, 224, 2, 2) > 0
    assert lib.hd_jpeg_workspace_bytes(n_max + 1, 224, 224, 2, 2) == 0
    p = C.c_void_p(256)                                                        # never dereferenced: the checks come first

    def call(N, H, W):
        return lib.hd_jpeg_decode(p, 1, p, N, H, W, 2, 2, p, 1, p, 1, p, p, p, 1 << 62, None)
    assert call(1, 46341, 46341) == HD_ERR_INVALID and b'2^31' in lib.hd_last_error()
    assert call(n_max + 1, 224, 224) == HD_ERR_INVALID and b'grid' in lib.hd_last_error()
    assert call(1, 0, 224) == HD_ERR_INVALID


def test_image_size_from_header_without_decoding():
    """eval's per-tube image size comes from the SOF marker: no decode, no device."""
    from human_dynamics_b200 import _lib
    from src.evaluation.eval import _img_size
    jpegs = [jpeg_ref.encode(jpeg_ref.make_image(48, 64, seed=i), 90, '420') for i in range(3)]
    _lib.lib.hd_launch_count_reset()
    assert _img_size(jpegs) == 48
    assert _lib.lib.hd_launch_count() == 0
    assert _img_size(np.zeros((2, 32, 40, 3), np.uint8)) == 32


def test_decode_jpegs_without_a_device_raises():
    """Only input the GPU decoder does not take goes to OpenCV; no CUDA device is an error, not a quiet host fallback."""
    torch = pytest.importorskip('torch')
    if torch.cuda.is_available():
        pytest.skip('checks the behaviour without a CUDA device')
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200 import jpeg
    from src.datasets.common import decode_jpegs
    jpegs = [jpeg_ref.encode(jpeg_ref.make_image(16, 16, seed=1), 90, '420')]
    with pytest.raises(HDError) as e:
        decode_jpegs(jpegs)
    assert not isinstance(e.value, (jpeg.UnsupportedJPEG, jpeg.CorruptJPEG)) and 'no CUDA device' in str(e.value)
