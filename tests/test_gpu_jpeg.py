"""GPU: hd_jpeg_decode (csrc/jpeg.cu) through human_dynamics_b200.jpeg against cv2.imdecode bit for bit, its batching, chunking,
streams and corrupt-data reporting, and the evaluation's device decode path (get_predictions) against the cv2 host path."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
cv2 = pytest.importorskip('cv2')
if not torch.cuda.is_available():
    pytest.skip('needs a CUDA device', allow_module_level=True)

from human_dynamics_b200 import jpeg, _lib                # noqa: E402
from oracle import jpeg_ref                               # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check(jpegs, **kw):
    """Decode into output buffers filled with 0x00, 0xFF and 0x5A in turn: every pattern must be overwritten with cv2's bytes, so a byte
    the decoder never writes fails at least two of the three runs.  Returns the decoded tensor."""
    want = np.stack([jpeg_ref.cv2_decode(d) for d in jpegs])
    out = torch.empty(want.shape, dtype=torch.uint8, device='cuda')
    for v in (0x00, 0xFF, 0x5A):
        out.fill_(v)
        got = jpeg.decode(jpegs, out=out, **kw)
        assert got.data_ptr() == out.data_ptr() and got.dtype == torch.uint8 and tuple(got.shape) == want.shape
        g = got.cpu().numpy()
        assert np.array_equal(g, want), 'pattern 0x%02X: %d of %d bytes differ' % (v, (g != want).sum(), g.size)
    fresh = jpeg.decode(jpegs, **kw)
    assert fresh.is_cuda and np.array_equal(fresh.cpu().numpy(), want)
    return fresh


def _batch(n, H, W, sampling, quality, optimize=False, rst=0, seed=0, kind='photo'):
    return [jpeg_ref.encode(jpeg_ref.make_image(H, W, seed=seed + i, kind=kind), quality, sampling, optimize=optimize, rst=rst)
            for i in range(n)]


@pytest.mark.parametrize('sampling', jpeg_ref.SAMPLINGS)
@pytest.mark.parametrize('quality', [50, 95, 100])
@pytest.mark.parametrize('size', [(224, 224), (300, 300), (37, 53), (1, 1), (2, 9), (9, 2), (7, 13), (17, 33), (64, 48)])
def test_decode_matches_cv2(size, sampling, quality):
    """Standard and optimised Huffman tables, with restart intervals of 1 and 5 MCUs; noise and saturated images at quality 100."""
    H, W = size
    for optimize, rst in ((False, 0), (True, 0), (False, 1), (True, 5)):
        _check(_batch(3, H, W, sampling, quality, optimize, rst, seed=H * 7 + W + quality))
    if quality == 100:
        _check(_batch(2, H, W, sampling, 100, kind='saturated', seed=H))
        _check(_batch(2, H, W, sampling, 100, kind='noise', seed=W))


@pytest.mark.parametrize('N', [1, 7, 160, 640])
def test_batches_with_mixed_tables(N):
    """One batch whose images carry different quantisation and Huffman tables (qualities 40..100, standard and optimised tables,
    restart intervals or not): every image exact, at 224^2 and 300^2."""
    for H in (224, 300):
        rs = np.random.RandomState(N + H)
        jpegs = []
        for i in range(N):
            img = jpeg_ref.make_image(H, H, seed=1000 * H + i, kind='noise' if i % 11 == 3 else 'photo')
            jpegs.append(jpeg_ref.encode(img, int(rs.randint(40, 101)), '420', optimize=bool(rs.randint(2)),
                                         rst=int(rs.choice([0, 0, 1, 4]))))
        _check(jpegs)


def test_repeats_and_chunks_bit_identical():
    jpegs = _batch(40, 224, 224, '420', 95, seed=77)
    ref = _check(jpegs).cpu()
    for chunk in (1, 3, 7, 40, None):
        for _ in range(2):
            assert torch.equal(jpeg.decode(jpegs, chunk=chunk).cpu(), ref), chunk


def test_corrupt_image_is_flagged_alone():
    """Image 3's entropy data cut short (EOI halfway), image 5's restart markers out of sequence: exactly those indices are reported,
    every other image is exact.  src.datasets.common.decode_jpegs then falls back to cv2 for the whole tube."""
    jpegs = _batch(8, 64, 96, '420', 90, rst=2, seed=5)
    h = jpeg_ref.parse(jpegs[3])
    cut = h['data_offset'] + h['data_bytes'] // 2
    jpegs[3] = jpegs[3][:cut] + (b'\x00' if jpegs[3][cut - 1] == 0xFF else b'') + b'\xff\xd9'
    b = bytearray(jpegs[5])
    h = jpeg_ref.parse(bytes(b))
    seg = b[h['data_offset']:h['data_offset'] + h['data_bytes']]
    at = next(i for i in range(len(seg) - 1) if seg[i] == 0xFF and seg[i + 1] == 0xD1)
    b[h['data_offset'] + at + 1] = 0xD4
    jpegs[5] = bytes(b)
    out, status = jpeg.decode_with_status(jpegs)
    st = status.cpu().numpy()
    assert np.nonzero(st)[0].tolist() == [3, 5], st
    assert st[3] & (_lib.HD_JPEG_OVERRUN | _lib.HD_JPEG_BAD_CODE) and st[5] & _lib.HD_JPEG_MARKER
    got = out.cpu().numpy()
    for i in (0, 1, 2, 4, 6, 7):
        assert np.array_equal(got[i], jpeg_ref.cv2_decode(jpegs[i])), i
    with pytest.raises(jpeg.CorruptJPEG) as e:
        jpeg.decode(jpegs)
    assert e.value.indices == [3, 5]
    from src.datasets.common import decode_jpeg, decode_jpegs
    fb = decode_jpegs(jpegs)
    assert isinstance(fb, np.ndarray) and np.array_equal(fb, np.stack([decode_jpeg(d) for d in jpegs]))


@pytest.mark.parametrize('sampling', jpeg_ref.SAMPLINGS)
def test_fill_bytes_before_markers(sampling):
    """Fill bytes before the restart markers and EOI are skipped: valid streams, status 0, bit for bit cv2."""
    jpegs = [jpeg_ref.add_fill_bytes(d, n=1 + i % 3) for i, d in enumerate(_batch(6, 64, 96, sampling, 90, rst=2, seed=11))]
    jpegs += [jpeg_ref.add_fill_bytes(d, n=2) for d in _batch(2, 64, 96, sampling, 90, seed=13)]
    _, status = jpeg.decode_with_status(jpegs)
    assert not status.cpu().numpy().any()
    _check(jpegs)


def test_refusals_raise_before_launch():
    ok = _batch(2, 32, 32, '420', 90)
    with pytest.raises(jpeg.UnsupportedJPEG):
        jpeg.decode(ok + _batch(1, 32, 40, '420', 90))                       # mixed sizes
    with pytest.raises(jpeg.UnsupportedJPEG):
        jpeg.decode(ok + _batch(1, 32, 32, '444', 90))                       # mixed sampling
    with pytest.raises(jpeg.UnsupportedJPEG):
        jpeg.decode(ok + [jpeg_ref.encode(jpeg_ref.make_image(32, 32, 1), 90, '420', progressive=True)])
    from src.datasets.common import decode_jpegs
    gray = [jpeg_ref.encode(jpeg_ref.make_image(32, 32, 1)[:, :, 0], 90)] * 2
    fb = decode_jpegs(gray)                                                   # grayscale: the cv2 path, as before
    assert isinstance(fb, np.ndarray) and fb.shape == (2, 32, 32, 3)
    dev = decode_jpegs(ok)
    assert isinstance(dev, torch.Tensor) and dev.is_cuda


def test_non_default_stream():
    jpegs = _batch(16, 224, 224, '420', 95, seed=3)
    want = np.stack([jpeg_ref.cv2_decode(d) for d in jpegs])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = jpeg.decode(jpegs)
        host = got.to('cpu', non_blocking=True)
        s.synchronize()
    assert np.array_equal(host.numpy(), want)


def test_launch_count_fixed():
    for n in (1, 50):
        jpegs = _batch(n, 48, 48, '420', 90)
        torch.cuda.synchronize()
        _lib.lib.hd_launch_count_reset()
        jpeg.decode(jpegs)
        assert _lib.lib.hd_launch_count() == 4


def test_get_predictions_device_decode_equals_host_path(tmp_path, weights, smpl_model):
    """get_predictions on eval_v1.tfrecord's JPEG strings (decoded on the device) returns the arrays the cv2-decoded host frames give."""
    from human_dynamics_b200.config import HMMRConfig
    from src.datasets.common import decode_jpeg, decode_jpegs, read_from_example, tf_record_iterator
    from src.evaluation.prediction import get_predictions
    from src.evaluation.tester import Tester
    model = Tester(HMMRConfig(batch_size=1, sequence_length=20, weights=weights, smpl_model=smpl_model, pred_mode='pred'))
    path = os.path.join(ROOT, 'tests', 'golden', 'eval_v1.tfrecord')
    for p_id, rec in enumerate(tf_record_iterator(path)):
        jpegs = read_from_example(rec, decode_images=False)['images']
        assert isinstance(decode_jpegs(jpegs), torch.Tensor)                  # the device path, not the cv2 fallback
        dev = get_predictions(model, jpegs, 'm', path, p_id, pred_dir=str(tmp_path / 'dev'))
        host = get_predictions(model, [decode_jpeg(d) for d in jpegs], 'm', path, p_id, pred_dir=str(tmp_path / 'host'))
        assert sorted(dev) == sorted(host)
        for k in host:
            if isinstance(host[k], np.ndarray):
                assert dev[k].dtype == host[k].dtype and np.array_equal(dev[k], host[k]), k
            else:
                assert dev[k] == host[k], k


def test_unit_range_table_matches_numpy():
    from src.evaluation.prediction import to_unit_range
    x = np.arange(256, dtype=np.uint8).reshape(1, 16, 16, 1).repeat(3, axis=3)
    got = to_unit_range(torch.from_numpy(x).cuda()).cpu().numpy()
    want = np.asarray((np.array(x) / 255) * 2 - 1, dtype=np.float32)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    dark = torch.ones((2, 4, 4, 3), dtype=torch.uint8, device='cuda')       # max <= 1.1: left as is, like the host path
    assert torch.equal(to_unit_range(dark), dark.float())
