"""CPU: the float32 oracle of the tube augmentation (oracle/tube_ref.py) against the fixture made by executing the reference's own
tube_augmentation.py / data_utils.py (tests/golden/tube_aug_v1.npz), known answers, the torch walk formula on recorded draws, and
the C-ABI's argument checks of hd_tube_augment (no device needed)."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from oracle import tube_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEN = os.path.join(ROOT, 'tests', 'golden', 'make_tube_golden.py')
GOLD = os.path.join(ROOT, 'tests', 'golden', 'tube_aug_v1.npz')


def tubes():
    """[(inputs, cfg, S, draws, reference outputs)] per fixture tube."""
    return tube_ref.load_fixture(GOLD)


def oracle_tube(x, cfg, S, draws):
    T = len(x['frames'])
    trans, scale, rot, flip = tube_ref.tube_walks(T, cfg, draws)
    res = tube_ref.augment_tube(x['frames'], x['labels'], x['centers'], x['poses'], x['gt3ds'], trans, scale, rot, flip, S,
                                cfg['trans_max'], cfg['rotate_max'] != 0)
    res.update(trans_walk=trans, scale_walk=scale, rot_walk=rot, flip=flip)
    return res


@pytest.mark.parametrize('i', [0, 1, 2])
def test_oracle_matches_reference_fixture(i):
    x, cfg, S, draws, ref = tubes()[i]
    o = oracle_tube(x, cfg, S, draws)
    assert np.array_equal(o['trans_walk'], ref['trans_walk'])
    assert np.array_equal(o['scale_walk'], ref['scale_walk'])
    assert np.array_equal(o['rot_walk'], ref['rot_walk'])
    assert np.array_equal(o['center'], ref['centers'][..., 0])
    assert np.abs(o['images'] - ref['images']).max() <= 1e-6
    for k in ('labels', 'gt3ds', 'poses'):
        assert np.abs(o[k[:-1] if k != 'labels' else 'label'] - ref[k]).max() <= 1e-6, k


def test_fixture_covers_the_cases():
    t = tubes()
    assert t[0][3]['flip_u'] < 0.5 and 'trans_start_u' not in t[0][3]                      # iid branch, flipped
    assert t[1][3]['flip_u'] >= 0.5 and 'trans_start_u' in t[1][3] and t[1][0]['frames'].shape[1:3] == (72, 100)
    assert t[2][1]['rotate_max'] != 0 and t[2][3]['flip_u'] < 0.5 and 'rot_u' in t[2][3]
    assert os.path.getsize(GOLD) < 1 << 20


def test_u8_conversion_is_the_converters_division():
    """float32(u8 / 255.) (float64 division, as the converters do) == float32 u8 / float32 255 (the kernel's)."""
    u = np.arange(256)
    assert np.array_equal((u / 255.).astype(np.float32), u.astype(np.float32) / np.float32(255))


def test_torch_walks_from_recorded_draws():
    """human_dynamics_b200.augment.random_walks on the fixture's draws == the reference's walks (CPU torch, sequential cumsum)."""
    from human_dynamics_b200.augment import random_walks
    for x, cfg, S, draws, ref in tubes():
        T = len(x['frames'])
        w = random_walks([T], cfg, draws=[draws])
        assert np.array_equal(w['trans'].numpy(), ref['trans_walk'])
        assert np.array_equal(w['scale'].numpy(), ref['scale_walk'][:, 0])
        assert np.array_equal(w['rot'].numpy(), ref['rot_walk'][:, 0])
        assert bool(w['tube_flip'][0]) == bool(draws['flip_u'] < 0.5)
        assert (w['flip'].numpy() == int(draws['flip_u'] < 0.5)).all()


def test_walk_branches_and_bounds():
    rng = np.random.RandomState(0)
    assert tube_ref.walk_branch(-20, 21, -20, 21) == 'iid' and tube_ref.walk_branch(-20, 21, -3, 4) == 'walk'
    assert tube_ref.walk_branch(0, 0, 0, 0) == 'zeros'
    for lo, hi, dlo, dhi, dt in ((-20, 21, -3, 4, np.int32), (-0.3, 0.3, -0.05, 0.05, np.float32)):
        w = tube_ref.bounded_random_walk(lo, hi, dlo, dhi, 200, dt, 2, rng.random_sample((1, 2)), rng.random_sample((200, 2)))
        assert w.dtype == dt and (w >= np.asarray(lo, dt)).all() and (w <= np.asarray(hi, dt)).all()
    # the reflected walk is the walk itself while it stays inside (-tm, tm)
    w = tube_ref.bounded_random_walk(-20, 21, -3, 4, 5, np.int32, 1, np.array([[0.5]]), np.full((5, 1), 0.5))
    assert list(w[:, 0]) == [0, 0, 0, 0, 0]      # start 0 (floor(0.5 * 41) - 20), steps 0 (floor(0.5 * 7) - 3)


def _frame(H=90, W=110, seed=1):
    rng = np.random.RandomState(seed)
    img = rng.uniform(0, 1, size=(H, W, 3)).astype(np.float32)
    lab = np.stack([rng.uniform(0, W, 25), rng.uniform(0, H, 25), rng.choice([0., 1.], 25)]).astype(np.float32)
    return img, lab, np.array([W // 2, H // 2]), rng.normal(0, 0.4, 72).astype(np.float32), rng.normal(0, 0.4, (14, 3)).astype(np.float32)


def test_zero_walk_is_the_plain_centred_crop():
    img, lab, c, pose, g = _frame()
    S = 64
    o = tube_ref.preprocess_frame(img, lab, c, pose, g, [0, 0], np.float32(0), np.float32(0), False, S)
    y0, x0 = c[1] - S // 2, c[0] - S // 2
    assert np.array_equal(o['crop'], (img[y0:y0 + S, x0:x0 + S] - np.float32(0.5)) * np.float32(2))
    assert np.array_equal(o['pose'], pose) and np.array_equal(o['gt3d'], g)
    assert list(o['geom']) == [90, 110, c[0], c[1], x0, y0]
    v = lab[2] > 0
    assert np.allclose(o['label'][0][v], 2 * (lab[0][v] - x0) / S - 1, atol=1e-6)
    assert (o['label'][:, ~v] == 0).all()


def test_flipping_twice_is_the_identity_on_labels():
    img, lab, c, pose, g = _frame()
    g = g - g.mean(0)                         # reflect_joints3d assumes mean-subtracted joints
    S = 64
    once = tube_ref.preprocess_frame(img, lab, c, pose, g, [0, 0], np.float32(0), np.float32(0), True, S)
    # back to crop pixels, then flip again through the same frame-free path
    kx = (once['label'][0] + 1) / 2 * S
    kx2 = (np.float32(S) - kx) - 1
    lab2 = np.stack([kx2[tube_ref.KP_SWAP], ((once['label'][1] + 1) / 2 * S)[tube_ref.KP_SWAP], once['label'][2][tube_ref.KP_SWAP]])
    vis = lab[2] > 0
    before = 2 * ((lab[0] - (c[0] - S // 2)) / S) - 1
    assert np.allclose(((2 * (lab2[0] / S) - 1))[vis], before[vis], atol=1e-5)
    assert np.array_equal(once['pose'][tube_ref.POSE_SWAP] * tube_ref.POSE_SIGN, pose)
    j = once['gt3d'][tube_ref.J3D_SWAP] * np.array([-1, 1, 1], np.float32)
    assert np.allclose(j - j.mean(0), g, atol=1e-6)


def test_quarter_turn_of_a_symmetric_ramp():
    """rotate by pi/2 about the crop centre: (x, y) -> input (ox * 0 - oy * 1 + x_off, ox * 1 + oy * 0 + y_off) with x_off = S - 1,
    y_off = 0: out[y][x] = crop[x][S - 1 - y].  A ramp v = x / (S - 1) (constant over rows) turns into 1 - y / (S - 1)."""
    S = 32
    ramp = np.tile((np.arange(S, dtype=np.float32) / np.float32(S - 1))[None, :, None], (S, 1, 3))
    c, s, a = tube_ref.rotate_coeffs(np.pi / 2, S)
    assert abs(a[2] - (S - 1)) < 1e-5 and abs(a[5]) < 1e-5
    out = tube_ref.rotate_image(ramp, a)
    want = np.tile((1 - np.arange(S, dtype=np.float32) / np.float32(S - 1))[:, None, None], (1, S, 3))
    inner = slice(1, S - 1)           # the outermost rows / columns read the zero fill through the taps' rounding
    assert np.abs(out[inner, inner] - want[inner, inner]).max() < 1e-5


def test_struct_layout_matches_header():
    from human_dynamics_b200 import _lib
    if shutil.which('gcc') is None:
        pytest.skip('gcc not available')
    import tempfile
    fields = ['F', 'trans', 'labels', 'K', 'centers', 'S', 'trans_max', 'geom', 'crops', 'plane_lo', 'WP']
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "hd_b200.h"\nint main(){printf("%zu", sizeof(hd_tube_aug_args));\n'
    src += ''.join('printf(" %%zu", offsetof(hd_tube_aug_args, %s));\n' % f for f in fields) + 'return 0;}\n'
    with tempfile.TemporaryDirectory() as td:
        cfile, exe = os.path.join(td, 't.c'), os.path.join(td, 't')
        open(cfile, 'w').write(src)
        subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), cfile, '-o', exe])
        out = [int(v) for v in subprocess.check_output([exe]).split()]
    assert out[0] == ctypes.sizeof(_lib.TubeAugArgs)
    for f, off in zip(fields, out[1:]):
        assert getattr(_lib.TubeAugArgs, f).offset == off, f


def test_abi_argument_checks_without_device():
    from human_dynamics_b200 import _lib
    L = _lib.lib
    p = 4096                        # never dereferenced: every call below fails its argument check first

    def args(**kw):
        a = _lib.TubeAugArgs()
        for k in ('frames', 'trans', 'scale', 'rot', 'flip', 'labels', 'centers', 'poses', 'gt3ds', 'labels_out', 'centers_out',
                  'poses_out', 'gt3ds_out', 'crops'):
            setattr(a, k, p)
        a.geom = p
        a.F, a.H, a.W, a.K, a.S, a.trans_max, a.flags = 2, 30, 40, 25, 64, 20, _lib.HD_AUG_FLIP
        for k, v in kw.items():
            setattr(a, k, v)
        return a
    before = L.hd_launch_count()
    assert L.hd_tube_augment(None, None) == 1
    for bad in (dict(frames=None), dict(trans=None), dict(labels=None), dict(gt3ds_out=None), dict(geom=None),
                dict(crops=None), dict(S=63), dict(S=0), dict(F=0), dict(flags=8), dict(flags=_lib.HD_AUG_FLIP | 16),
                dict(K=19), dict(flags=_lib.HD_AUG_ROTATE | _lib.HD_AUG_FLIP, rot=None), dict(geom=p + 4),
                dict(plane_hi=p), dict(crops=None, plane_hi=p, plane_lo=p, WP=70), dict(trans_max=-1)):
        assert L.hd_tube_augment(ctypes.byref(args(**bad)), None) == 1, bad
    assert b'hd_tube_augment' in L.hd_last_error()
    assert L.hd_launch_count() == before
    assert L.hd_version() >= 105


@pytest.mark.skipif(not os.path.isdir(os.path.join(os.environ.get('HD_REFERENCE_ROOT', '/nonexistent'), 'src')),
                    reason='HD_REFERENCE_ROOT does not name a reference checkout')
def test_golden_generator_reproduces_the_fixture():
    r = subprocess.run([sys.executable, GEN, '--check'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
