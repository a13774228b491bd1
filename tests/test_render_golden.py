"""CPU: the VisRenderer drop-in's host code and the oracle's composite against tests/golden/render_v1.npz, which records what the
reference's own nmr_renderer.py hands the Neural Mesh Renderer and what it makes of NMR's output (tests/golden/make_render_golden.py).

Pinned here: projection and y flip (R1), image size and settings handed to NMR, the camera chain of visualize_img_orig above and
below max_img_size, make_square / remove_pads, the rotated() view, and the uint8 composite of every variant (R8), all exactly
(float32 where the reference computes in float32)."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import render_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'render_v1.npz')


def _gen():
    spec = importlib.util.spec_from_file_location('_render_golden', os.path.join(ROOT, 'tests', 'golden', 'make_render_golden.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _host():
    """The drop-in module; the helpers used here are pure host code (numpy, cv2) and touch no device."""
    pytest.importorskip('cv2')
    from src.util.render import nmr_renderer as M
    return M


@pytest.fixture(scope='module')
def z():
    with np.load(GOLD) as f:
        yield {k: f[k] for k in f.files}


def _proj32(v, cam):
    """R1 as the reference evaluates it in float32 (torch_utils.py:21-29 then nmr_renderer.py:143)."""
    v = np.asarray(v, np.float32)
    cam = np.asarray(cam, np.float32)
    xy = cam[..., 0, None, None] * (v[..., :2] + cam[..., None, 1:3])
    out = np.concatenate([xy, v[..., 2:3]], axis=-1)
    out[..., 1] *= -1
    return out


def test_settings_and_faces_handed_to_nmr(z):
    from human_dynamics_b200.render import COLORS, DEFAULT_LIGHT
    faces = np.load(os.path.join(ROOT, 'src', 'tf_smpl', 'smpl_faces.npy')).astype(np.int64)
    for i in range(int(z['num_calls'])):
        assert str(z['call%d_camera_mode' % i]) == 'look_at' and str(z['call%d_perspective' % i]) == 'False'
        assert z['call%d_faces_shape' % i][1:].tolist() == list(faces.shape)
        assert int(z['call%d_faces_sum' % i]) == int(faces.sum()) * int(z['call%d_faces_shape' % i][0])
        assert z['call%d_light' % i].tolist() == list(DEFAULT_LIGHT[0]) + [DEFAULT_LIGHT[1], DEFAULT_LIGHT[2]]
        assert z['call%d_bg' % i].tolist() == [1.0, 1.0, 1.0]
        if str(z['call%d_kind' % i]) == 'rgb':
            color = 'pink' if i in z['rotated_x30_calls'] else 'blue'
            assert np.array_equal(z['call%d_texture' % i], np.tile(np.float32(COLORS[color]), (len(z['call%d_texture' % i]), 1)))
            assert np.allclose(COLORS[color], R.COLORS[color])


def test_projection_and_flip_exact(z):
    ids = z['vert_ids']
    v = z['verts'][:, ids]
    cams = z['cams']
    single = {'cam0': (0, cams[0]), 'cam1': (0, cams[1]), 'cam2': (0, cams[2]), 'default_cam': (0, np.float32([0.9, 0, 0])),
              'img': (1, cams[1]), 'alpha': (1, cams[1]), 'mask': (1, cams[1])}
    for name, (k, cam) in single.items():
        for c in z[name + '_calls']:
            assert np.array_equal(z['call%d_verts' % c][0], _proj32(v[k], cam)), name
    for name in ('batch_img', 'batch_mask'):
        for c in z[name + '_calls']:
            assert np.array_equal(z['call%d_verts' % c], _proj32(v, cams)), name


def test_rotated_view_vertices(z):
    """rotated(): R (v - mean) + mean with the drop-in's rotation(); the reference does it in float32 torch, the oracle in float64."""
    from human_dynamics_b200.render import rotation
    v = z['verts'][2]
    for name, deg, axis, cam in (('rotated90', 90, 'y', z['cams'][2]), ('rotated_x30', 30, 'x', z['cams'][0])):
        want = _proj32(R.rotate_about_mean(v, rotation(deg, axis))[z['vert_ids']], cam)
        got = z['call%d_verts' % z[name + '_calls'][0]][0]
        assert np.abs(got - want).max() < 2e-6, name


def test_composites_of_every_variant_exact(z):
    gen = _gen()
    S = 32

    def stub(c, kind, B):
        return gen.stub_outputs(int(c), kind, B, S)

    for name in ('cam0', 'cam1', 'cam2', 'default_cam', 'rotated90', 'rotated_x30'):
        c, = z[name + '_calls']
        rgb = stub(c, 'rgb', 1)[0].transpose(1, 2, 0)
        assert np.array_equal(z[name + '_out'], R.composite(rgb, None)), name
    # img in [0, 255] (what visualize_img passes): img * (1 - mask) + rend * mask, float32
    c_rgb, c_a = z['img_calls']
    rend = np.clip(stub(c_rgb, 'rgb', 1)[0].transpose(1, 2, 0), 0, 1) * np.float32(255)
    m = np.repeat(stub(c_a, 'alpha', 1)[0][..., None], 3, axis=2)
    assert np.array_equal(z['img_out'], (z['img255'] * (1 - m) + rend * m).astype(np.uint8))
    # alpha=True: RGBA with alpha = uint8(mask * 255)
    c_rgb, c_a = z['alpha_calls']
    a = stub(c_a, 'alpha', 1)[0]
    want = np.dstack([R.composite(stub(c_rgb, 'rgb', 1)[0].transpose(1, 2, 0), None), (a * 255).astype(np.uint8)])
    assert np.array_equal(z['alpha_out'], want)
    # rend_mask: the silhouette as RGB; batched, the reference's [1, S, S, 3B] layout
    c, = z['mask_calls']
    assert np.array_equal(z['mask_out'], np.repeat((stub(c, 'alpha', 1)[0] * 255)[..., None], 3, axis=2).astype(np.uint8))
    c, = z['batch_mask_calls']
    sil = stub(c, 'alpha', 3)
    assert np.array_equal(z['batch_mask_out'], (np.tile(sil[None], (1, 3, 1, 1)).transpose(0, 2, 3, 1) * 255).astype(np.uint8))
    c_rgb, c_a = z['batch_img_calls']
    rend = np.clip(stub(c_rgb, 'rgb', 3).transpose(0, 2, 3, 1), 0, 1) * np.float32(255)
    m = np.repeat(stub(c_a, 'alpha', 3)[..., None], 3, axis=3)
    assert np.array_equal(z['batch_img_out'], (z['img255'][None] * (1 - m) + rend * m).astype(np.uint8))


def test_visualize_img_orig_camera_chain_square_and_composite(z):
    """Both frame sizes: the drop-in's orig_frame_size / orig_frame_cam give the image size and the vertices NMR was handed, exactly;
    make_square + the oracle's R8 composite + remove_pads reproduce the reference's overlay and rotated view exactly."""
    M = _host()
    from oracle import preproc_ref
    from human_dynamics_b200.render import rotation
    gen = _gen()
    for j in range(len(gen.ORIG_CASES)):
        H, W, mx, sx, sy, sc = z['orig%d_case' % j]
        H, W, mx = int(H), int(W), int(mx)
        scale_orig, Hs, Ws, S = M.orig_frame_size(H, W, mx)
        assert (scale_orig is None) == (max(H, W) <= mx)
        c_rgb, c_a, c_rot = z['orig%d_calls' % j]
        assert int(z['call%d_image_size' % c_rgb]) == S == int(z['call%d_image_size' % c_rot])
        cam = M.orig_frame_cam(z['cams'][1], np.array([sx, sy]), sc, [224, 224], S, scale_orig)
        v = z['verts'][1][z['vert_ids']]
        assert np.array_equal(z['call%d_verts' % c_rgb][0], _proj32(v, cam))
        assert np.abs(z['call%d_verts' % c_rot][0] - _proj32(R.rotate_about_mean(z['verts'][1], rotation(90))[z['vert_ids']], cam)).max() < 2e-6
        img = z['orig%d_img' % j]
        if scale_orig is not None:
            img, _ = preproc_ref.resize_img(img, scale_orig)
        sq, pads = M.make_square(img)
        assert sq.shape[:2] == (S, S) and list(pads) == [S - Hs, S - Ws]
        rgb = gen.stub_outputs(int(c_rgb), 'rgb', 1, S)[0].transpose(1, 2, 0)
        alpha = gen.stub_outputs(int(c_a), 'alpha', 1, S)[0]
        over = M.remove_pads(R.composite(rgb, alpha, sq), pads)
        assert over.shape == (Hs, Ws, 3)
        assert np.array_equal(z['orig%d_out1' % j], over / 255)
        rot = M.remove_pads(R.composite(gen.stub_outputs(int(c_rot), 'rgb', 1, S)[0].transpose(1, 2, 0), None), pads)
        assert np.array_equal(z['orig%d_out2' % j], rot / 255)
