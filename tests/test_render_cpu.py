"""CPU: the rendering model R1-R8 (oracle/render_ref.py) on hand-computed cases, and the C struct of hd_render_params.

R3-R6 are assumptions about the Neural Mesh Renderer's internals ([NMR-ext], unpinned): these tests check that the oracle states them,
not that NMR behaves so."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import render_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_render_params_matches_compiled_struct(tmp_path):
    """[R-ABI] hd_render_params: gcc sizeof/offsetof against the ctypes mirror."""
    from human_dynamics_b200 import _lib
    if shutil.which('gcc') is None:
        pytest.skip('gcc not available')
    fields = ['color', 'light_dir', 'ambient', 'directional', 'bg', 'near_z', 'far_z', 'eye_z', 'rot', 'use_rot']
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "hd_b200.h"\nint main(){printf("%zu", sizeof(hd_render_params));\n'
    src += ''.join('printf(" %%zu", offsetof(hd_render_params, %s));\n' % f for f in fields) + 'return 0;}\n'
    c = tmp_path / 't.c'
    c.write_text(src)
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(c), '-o', str(tmp_path / 't')])
    out = [int(x) for x in subprocess.check_output([str(tmp_path / 't')]).split()]
    assert out[0] == ctypes.sizeof(_lib.RenderParams) == 96
    for f, off in zip(fields, out[1:]):
        assert getattr(_lib.RenderParams, f).offset == off, f
    assert _lib.lib.hd_version() >= 101


def test_render_workspace_and_argument_checks_without_device():
    """Arguments are checked before any CUDA call: null pointers and bad sizes return HD_ERR_INVALID, a small workspace
    HD_ERR_WORKSPACE."""
    from human_dynamics_b200 import _lib
    L = _lib.lib
    assert L.hd_render_workspace_bytes(1, 224, 13776) >= 448 * 448 * 8 + 13776 * 16
    assert L.hd_render_workspace_bytes(0, 224, 10) == 0
    p = _lib.RenderParams()
    fake = ctypes.c_void_p(0x1000)            # never dereferenced: every call below fails its checks first
    args = lambda S=8, N=1, V=3, F=1, ws=1 << 20, verts=fake: (verts, 9, N, V, fake, F, fake, 3, ctypes.byref(p), None, S, fake, None,
                                                                  fake, ws, None)
    assert L.hd_render_mesh(*args(verts=None)) == 1
    assert b'null' in L.hd_last_error()
    assert L.hd_render_mesh(*args(S=0)) == 1 and L.hd_render_mesh(*args(S=2049)) == 1
    assert L.hd_render_mesh(*args(V=0)) == 1 and L.hd_render_mesh(*args(F=0)) == 1 and L.hd_render_mesh(*args(N=-1)) == 1
    assert L.hd_render_mesh(*args(ws=16)) == 2
    assert L.hd_render_mesh(*args(N=0)) == 0


def test_r3_r7_single_triangle_covers_exact_samples():
    """One triangle, legs on x = -1 and y = -1 (outside every sample centre), hypotenuse 1.5x + y = 0.1: the covered samples are
    exactly those with 1.5 x_c + y_r < 0.1, and pixel alpha = covered quarter."""
    S = 4
    cen = R.sample_centres(S)
    X0, Y0 = -1.0, -1.0
    tri_img = np.array([[X0, Y0], [(0.1 - Y0) / 1.5, Y0], [X0, 0.1 - 1.5 * X0]])
    verts = np.array([[x, y, 0.0] for x, y in tri_img])
    r = R.rasterize(verts, [1.0, 0.0, 0.0], np.array([[0, 1, 2]]), S)
    want = (1.5 * cen[None, :] + cen[:, None]) < 0.1                                   # [row, col]
    assert np.array_equal(r['face'] >= 0, want)
    alpha = want.reshape(S, 2, S, 2).mean(axis=(1, 3))
    assert np.array_equal(r['alpha'], alpha)
    assert set(np.unique(r['alpha']).tolist()) == {0.0, 0.25, 0.5, 0.75, 1.0}
    assert np.all(r['margin'][want] > 0)
    # R7: colour = mean of the 2x2 samples, white where empty
    fc = R.face_colors(R.project(verts, [1, 0, 0])[3], np.array([[0, 1, 2]]), R.COLORS['blue'])[0]
    exp = alpha[..., None] * fc + (1 - alpha[..., None]) * 1.0
    assert np.allclose(r['rgb'], exp, atol=1e-12)


def _quad(x0, x1, y0, y1, Z):
    v = np.array([[x0, y0, Z], [x1, y0, Z], [x1, y1, Z], [x0, y1, Z]], np.float64)
    return v, np.array([[0, 1, 2], [0, 2, 3]])


def test_r4_nearer_quad_wins_whatever_the_face_order():
    S = 8
    va, fa = _quad(-0.8, 0.45, -0.8, 0.4, 0.3)        # far
    vb, fb = _quad(-0.4, 0.85, -0.4, 0.8, -0.2)       # near (smaller z = nearer the eye at -z)
    verts = np.concatenate([va, vb])
    for order in (np.concatenate([fa, fb + 4]), np.concatenate([fb + 4, fa])):
        r = R.rasterize(verts, [1.0, 0.0, 0.0], order, S)
        cen = R.sample_centres(S)
        in_b = (cen[:, None] > -0.4) & (cen[:, None] < 0.8) & (cen[None, :] > -0.4) & (cen[None, :] < 0.85)
        in_a = (cen[:, None] > -0.8) & (cen[:, None] < 0.4) & (cen[None, :] > -0.8) & (cen[None, :] < 0.45)
        covered = r['face'] >= 0
        # the quads' diagonals pass through no sample centre, so they leave no hole
        assert np.array_equal(covered, in_a | in_b)
        near_faces = set((np.nonzero(np.all(order >= 4, axis=1))[0]).tolist())
        winner_is_b = np.isin(r['face'], list(near_faces))
        assert np.array_equal(winner_is_b, in_b)
        assert np.allclose(r['depth'][in_b], -0.2 + R.EYE_SHIFT)
        assert np.allclose(r['depth'][in_a & ~in_b], 0.3 + R.EYE_SHIFT)


def test_r4_exact_tie_goes_to_lower_face_index():
    v, f = _quad(-0.5, 0.5, -0.5, 0.5, 0.0)
    faces = np.concatenate([f, f[:, ::-1]])           # the same two triangles again, other winding, at indices 2, 3
    r = R.rasterize(v, [1.0, 0.0, 0.0], faces, 4)
    assert set(np.unique(r['face'][r['face'] >= 0]).tolist()) == {0, 1}


def test_r5_r6_back_facing_triangle_gets_the_eye_facing_normal():
    """fill_back: both windings of a triangle render the same colour, lit by the normal that points to -z.
    Triangle in the plane z = x (tilted 45 degrees about y): eye-facing unit normal n = (1, 0, -1)/sqrt2,
    n . d = (1 + 1)/sqrt2 = sqrt2 with d = [1, .5, -1] unnormalised, shade = 0.7 + 0.3 sqrt2."""
    verts = np.array([[-0.5, -0.5, -0.5], [0.5, -0.5, 0.5], [0.0, 0.5, 0.0]])
    r1 = R.project(verts, [1.0, 0.0, 0.0])[3]
    c = R.COLORS['pink']
    a = R.face_colors(r1, np.array([[0, 1, 2]]), c)[0]
    b = R.face_colors(r1, np.array([[2, 1, 0]]), c)[0]
    want = np.array(c) * (0.7 + 0.3 * np.sqrt(2.0))
    assert np.allclose(a, want, atol=1e-12) and np.allclose(b, want, atol=1e-12)
    assert (want > np.array(c)).all() and want[0] > 1.0                             # the colour may exceed 1 (clipped in R8)
    # a triangle facing away from the light: n . d < 0 -> ambient only
    flat = np.array([[0, 0, 0], [1, 0, -1], [0, 1, 0]], np.float64)                 # plane z = -x: n = (-1, 0, -1)/sqrt2 -> n.d = 0
    assert np.allclose(R.face_colors(R.project(flat, [1, 0, 0])[3], np.array([[0, 1, 2]]), c)[0], np.array(c) * 0.7)
    for S in (4, 6):
        ra = R.rasterize(verts, [1.0, 0.0, 0.0], np.array([[0, 1, 2]]), S)
        rb = R.rasterize(verts, [1.0, 0.0, 0.0], np.array([[2, 1, 0]]), S)
        assert np.array_equal(ra['face'], rb['face']) and np.allclose(ra['rgb'], rb['rgb'])


def test_r4_near_far_clipping():
    S = 4
    v, f = _quad(-0.9, 0.9, -0.9, 0.9, 0.0)
    shift = R.EYE_SHIFT
    for Z, drawn in ((0.1 - shift - 1e-3, False), (0.1 - shift + 1e-3, True), (100 - shift - 1e-3, True), (100 - shift + 1e-3, False)):
        vz = v.copy()
        vz[:, 2] = Z
        r = R.rasterize(vz, [1.0, 0.0, 0.0], f, S)
        assert (r['face'] >= 0).any() == drawn, Z


def test_r8_truncation_and_order():
    rgb = np.array([[[0.5, 1.2, -0.1]]])
    alpha = np.array([[0.75]])
    assert R.composite(rgb, alpha).tolist() == [[[127, 255, 0]]]                   # 127.5 truncates, clip to [0, 1]
    img = np.array([[[1.0, -1.0, 0.0]]], np.float32)
    out = R.composite(rgb, alpha, img)
    f = np.float32
    rend = np.clip(rgb.astype(f), 0, 1) * f(255)
    img255 = ((img + f(1)) * f(0.5)) * f(255)
    want = np.trunc(img255 * (f(1) - f(0.75)) + rend * f(0.75))
    assert out.tolist() == want.astype(np.uint8).tolist() == [[[159, 191, 31]]]
    # alpha 0: the image comes back truncated, alpha 1: the render
    assert R.composite(rgb, np.zeros((1, 1)), img).tolist() == [[[255, 0, 127]]]
    assert R.composite(rgb, np.ones((1, 1)), img).tolist() == [[[127, 255, 0]]]


def test_r1_r2_vertex_lands_on_its_keypoint_sample():
    """A point P whose keypoint s*(P_xy + t) is the centre of sample (r0, c0) -- kps convention, row from the top -- is covered
    there by a tiny triangle around it, and nowhere else: R1's y negation and NMR's vertical flip cancel."""
    S = 16
    cam = np.array([0.8, 0.1, -0.2])
    cen = R.sample_centres(S)
    r0, c0 = 5, 20
    X, Y = cen[c0] / cam[0] - cam[1], cen[r0] / cam[0] - cam[2]
    kp = cam[0] * (np.array([X, Y]) + cam[1:])
    assert np.allclose(kp, [cen[c0], cen[r0]])
    e = 0.3 / (2 * S) / cam[0]
    verts = np.array([[X - e, Y - e, 0], [X + 2 * e, Y - e, 0], [X - e, Y + 2 * e, 0]])
    r = R.rasterize(verts, cam, np.array([[0, 1, 2]]), S)
    assert np.argwhere(r['face'] >= 0).tolist() == [[r0, c0]]
