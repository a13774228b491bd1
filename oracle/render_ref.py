"""Float64 restatement of the mesh rendering the reference's visualiser gets from the Neural Mesh Renderer (NMR).

The reference draws its predictions with `VisRenderer` (src/util/render/nmr_renderer.py:43-240), a wrapper around the third-party
NMR (`neural_renderer`, pinned at commit 55a05a by src/external/install_external.sh:3-7), called as
`nr.Renderer(img_size, camera_mode='look_at', perspective=False)`, `set_light_dir([1, .5, -1], int_dir=0.3, int_amb=0.7)`,
`set_bgcolor([1, 1, 1])` and NMR's defaults otherwise (anti_aliasing=True, fill_back=True, near 0.1, far 100,
eye [0, 0, -(1/tan 30deg + 1)]).  NMR cannot be installed next to this project, so its behaviour under those settings is
restated here as assumptions R1-R8.  Each is marked [NMR-ext] and is *unpinned* in the sense of the [TF-ext] assumptions
(SURVEY App. A): what the reference itself authored around NMR (projection, y flip, camera chain, rotation, composite) is pinned
by tests/golden/render_v1.npz, which runs the reference's own nmr_renderer.py / torch_utils.py; R3-R6 are NMR's internals and
cannot be checked against NMR itself here.

  R1 projection [NMR-ext]  (torch_utils.orthographic_proj_withz_idrot + nmr_renderer.py:140-143):  x = s*(X + tx),
     y = -s*(Y + ty), z = Z.  NMR's look_at transform with that eye is the identity plus z += 1/tan 30deg + 1 = 2.7320508;
     there is no perspective divide.
  R2 pixel grid [NMR-ext]  the image is rasterised at 2S x 2S; after NMR's vertical flip, sample (r, c) has its centre at
     x_img = (2c + 1 - 2S) / 2S, y_img = (2r + 1 - 2S) / 2S, where y_img = -y of R1 -- the convention of `kps`: a vertex lands
     where its keypoint would.
  R3 coverage [NMR-ext]  a sample is inside a face when all three screen-space barycentric weights are > 0.
  R4 depth [NMR-ext]  sample depth is 1 / sum(w_i / z_i) (NMR's interpolation, used even without perspective); samples with
     depth <= near or >= far are dropped; the smallest depth wins and an exact tie goes to the lower face index.
  R5 fill_back [NMR-ext]  every face is drawn exactly once, in whichever of its two windings faces the eye; its lighting normal
     is normalize(cross(v0 - v1, v2 - v1)) of that winding in R1 coordinates, i.e. the sign that points toward the eye (-z).
  R6 lighting [NMR-ext]  face colour = c * (0.7 + 0.3 * relu(n . d)), d = [1, .5, -1] NOT normalised (so a colour can exceed 1);
     c from the `colors` table (nmr_renderer.py:25-36).
  R7 anti-aliasing [NMR-ext]  pixel colour = mean of its 2x2 samples, the background colour for empty samples; alpha = covered
     fraction, exactly 0, 1/4, 1/2, 3/4 or 1.
  R8 output [NMR-ext]  rend = clip(rgb, 0, 1) * 255; with a background image in [-1, 1], img255 = (img + 1) * 0.5 * 255 and
     the result is uint8(trunc(img255 * (1 - alpha) + rend * alpha)), evaluated in float32 in that order (nmr_renderer.py:154-168,
     visualize_img :305-306, with a float32 image); without one it is uint8(rend).

The rasteriser below is deliberately plain: every face, in index order, tests every sample of its bounding box with barycentric
weights solved directly in image coordinates, and keeps a per-sample (depth, face) z-buffer.  Besides the image it returns the
per-sample face id, the winner's barycentric margin (smallest weight) and depth, so a test can tell an edge or depth-tie
disagreement from a real one.  Only tests import this module.
"""
import numpy as np

COLORS = {
    'blue': [0.65098039, 0.74117647, 0.85882353],
    'pink': [.9, .7, .7],
    'mint': [166 / 255., 229 / 255., 204 / 255.],
    'mint2': [202 / 255., 229 / 255., 223 / 255.],
    'green': [153 / 255., 216 / 255., 201 / 255.],
    'green2': [171 / 255., 221 / 255., 164 / 255.],
    'red': [251 / 255., 128 / 255., 114 / 255.],
    'orange': [253 / 255., 174 / 255., 97 / 255.],
    'yellow': [250 / 255., 230 / 255., 154 / 255.],
}
EYE_SHIFT = 1.0 / np.tan(np.radians(30.0)) + 1.0
DEFAULTS = dict(light_dir=(1.0, 0.5, -1.0), ambient=0.7, directional=0.3, bg=(1.0, 1.0, 1.0), near=0.1, far=100.0,
                eye_shift=EYE_SHIFT)


def rotate_about_mean(verts, rot):
    """VisRenderer.rotated: R (v - mean) + mean with the vertex mean of the frame (nmr_renderer.py:213-216)."""
    v = np.asarray(verts, np.float64)
    m = v.mean(axis=0)
    return (v - m) @ np.asarray(rot, np.float64).T + m


def project(verts, cam, eye_shift=EYE_SHIFT):
    """R1 + R2: [V,3] -> image x, image y (= -y of R1), z after the look_at shift; and the R1 coordinates themselves."""
    v = np.asarray(verts, np.float64)
    s, tx, ty = (float(c) for c in cam)
    r1 = np.stack([s * (v[:, 0] + tx), -(s * (v[:, 1] + ty)), v[:, 2]], axis=1)
    return r1[:, 0], -r1[:, 1], r1[:, 2] + eye_shift, r1


def face_colors(r1, faces, color, light_dir=DEFAULTS['light_dir'], ambient=0.7, directional=0.3):
    """R5 + R6: per-face colour from the eye-facing normal."""
    p0, p1, p2 = r1[faces[:, 0]], r1[faces[:, 1]], r1[faces[:, 2]]
    n = np.cross(p0 - p1, p2 - p1)
    n = np.where(n[:, 2:3] > 0, -n, n)                        # the winding that faces the eye has its normal toward -z
    n = n / np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-12)
    shade = ambient + directional * np.maximum(n @ np.asarray(light_dir, np.float64), 0.0)
    return np.asarray(color, np.float64)[None, :] * shade[:, None]


def barycentric(xi, yi, tri_x, tri_y):
    """Barycentric weights of image points (xi, yi) in the triangle (tri_x, tri_y): [..., 3]."""
    x0, x1, x2 = tri_x
    y0, y1, y2 = tri_y
    det = (x1 - x0) * (y2 - y0) - (x2 - x0) * (y1 - y0)
    w1 = ((xi - x0) * (y2 - y0) - (x2 - x0) * (yi - y0)) / det
    w2 = ((x1 - x0) * (yi - y0) - (xi - x0) * (y1 - y0)) / det
    return np.stack([1.0 - w1 - w2, w1, w2], axis=-1)


def sample_centres(S):
    """R2: image coordinate of sample index k (rows and columns alike) on the 2S grid."""
    k = np.arange(2 * S, dtype=np.float64)
    return (2 * k + 1 - 2 * S) / (2 * S)


def face_at(verts, cam, faces, f, r, c, S, eye_shift=EYE_SHIFT):
    """(min barycentric weight, depth) of face f at sample (r, c): for classifying a disagreement."""
    xi, yi, z, _ = project(verts, cam, eye_shift)
    idx = np.asarray(faces[f])
    cen = sample_centres(S)
    w = barycentric(cen[c], cen[r], xi[idx], yi[idx])
    return float(w.min()), float(1.0 / np.sum(w / z[idx]))


def rasterize(verts, cam, faces, S, color=COLORS['blue'], light_dir=DEFAULTS['light_dir'], ambient=0.7, directional=0.3,
              bg=(1.0, 1.0, 1.0), near=0.1, far=100.0, eye_shift=EYE_SHIFT, rot=None):
    """One frame.  verts [V,3], cam [3], faces [F,3] int; faces with an index outside [0, V) are skipped.

    -> dict(face [2S,2S] int64 (-1 empty), margin, depth [2S,2S] float64 (nan empty), rgb [S,S,3] float64 (R7, unclipped),
            alpha [S,S] float64)."""
    v = np.asarray(verts, np.float64)
    if rot is not None:
        v = rotate_about_mean(v, rot)
    faces = np.asarray(faces, np.int64)
    V = v.shape[0]
    ok = np.all((faces >= 0) & (faces < V), axis=1)
    xi, yi, z, r1 = project(v, cam, eye_shift)
    safe = np.where(ok[:, None], faces, 0)
    fcol = face_colors(r1, safe, color, light_dir, ambient, directional)
    cen = sample_centres(S)
    S2 = 2 * S
    zbuf = np.full((S2, S2), np.inf)
    fid = np.full((S2, S2), -1, np.int64)
    marg = np.full((S2, S2), np.nan)
    for f in np.nonzero(ok)[0]:
        idx = faces[f]
        tx, ty, tz = xi[idx], yi[idx], z[idx]
        # bounding box in sample indices: centre (2k + 1 - 2S) / 2S  <=>  k = (x * 2S + 2S - 1) / 2
        c_lo = max(int(np.ceil((tx.min() * S2 + S2 - 1) / 2)), 0)
        c_hi = min(int(np.floor((tx.max() * S2 + S2 - 1) / 2)), S2 - 1)
        r_lo = max(int(np.ceil((ty.min() * S2 + S2 - 1) / 2)), 0)
        r_hi = min(int(np.floor((ty.max() * S2 + S2 - 1) / 2)), S2 - 1)
        if c_lo > c_hi or r_lo > r_hi:
            continue
        det = (tx[1] - tx[0]) * (ty[2] - ty[0]) - (tx[2] - tx[0]) * (ty[1] - ty[0])
        if det == 0:
            continue
        X, Y = np.meshgrid(cen[c_lo:c_hi + 1], cen[r_lo:r_hi + 1])
        w = barycentric(X, Y, tx, ty)
        inside = np.all(w > 0, axis=-1)                                                  # R3
        d = 1.0 / np.sum(w / tz, axis=-1)                                                # R4
        cur = zbuf[r_lo:r_hi + 1, c_lo:c_hi + 1]
        win = inside & (d > near) & (d < far) & (d < cur)                                # strict: earlier (lower) face keeps a tie
        if not win.any():
            continue
        cur[win] = d[win]
        fid[r_lo:r_hi + 1, c_lo:c_hi + 1][win] = f
        marg[r_lo:r_hi + 1, c_lo:c_hi + 1][win] = w.min(axis=-1)[win]
    covered = fid >= 0
    samp = np.where(covered[..., None], fcol[np.maximum(fid, 0)], np.asarray(bg, np.float64))
    rgb = samp.reshape(S, 2, S, 2, 3).mean(axis=(1, 3))                                  # R7
    alpha = covered.reshape(S, 2, S, 2).mean(axis=(1, 3))
    depth = np.where(covered, zbuf, np.nan)
    return {'face': fid, 'margin': marg, 'depth': depth, 'rgb': rgb, 'alpha': alpha}


def composite(rgb, alpha, img=None):
    """R8 in float32, in the reference's order: uint8(rend) or uint8(img255 * (1 - alpha) + rend * alpha)."""
    rend = np.clip(np.asarray(rgb, np.float32), 0, 1) * np.float32(255.0)
    if img is None:
        return rend.astype(np.uint8)
    img255 = ((np.asarray(img, np.float32) + np.float32(1)) * np.float32(0.5)) * np.float32(255.0)
    a = np.asarray(alpha, np.float32)[..., None]
    return (img255 * (np.float32(1) - a) + rend * a).astype(np.uint8)


def render(verts, cams, faces, S, background=None, **kw):
    """Batch of frames -> (uint8 [N,S,S,3], alpha [N,S,S], per-frame rasterize() dicts)."""
    outs, alphas, info = [], [], []
    for i in range(len(verts)):
        r = rasterize(verts[i], cams[i], faces, S, **kw)
        outs.append(composite(r['rgb'], r['alpha'], None if background is None else background[i]))
        alphas.append(r['alpha'])
        info.append(r)
    return np.stack(outs), np.stack(alphas), info
