"""float32 numpy restatement of the reference's training-time tube augmentation -- TEST INFRASTRUCTURE.

Restates, in the reference's op order:
  * src/util/tube_augmentation.py:36-186  TubePreprocessor.__call__ / preprocess_image (map over frames, flip per tube);
  * src/util/data_utils.py:512-548        jitter_center, jitter_scale;
                           :551-579        pad_image_edge (edge padding = clamping into the scaled image);
                           :601-699        flip_image, reflect_pose, reflect_joints3d;
                           :702-762        rotate_img;
                           :787-835        bounded_random_walk;
and the TensorFlow 1.x kernels they call, from the TF 1.x sources:
  * tf.image.resize_images (BILINEAR, align_corners=False): core/kernels/resize_bilinear_op.cc -- scale = in / out in float32,
    compute_interpolation_weights: in = i * scale, lower = (int64) in, upper = min(lower + 1, in_size - 1), lerp = in - lower;
    compute_lerp: top = tl + (tr - tl) * x_lerp, bottom likewise, top + (bottom - top) * y_lerp;
  * tf.contrib.image.rotate (BILINEAR): contrib/image/python/ops/image_ops.py angles_to_projective_transforms
    ([cos, -sin, x_off, sin, cos, y_off, 0, 0]) and contrib/image/kernels/image_ops.h ProjectiveGenerator: input_x =
    (a0 * x + a1 * y + a2) / projection, floor / floor + 1 taps, read_with_fill_value (0 outside the image), weights
    (x_ceil - x), (x - x_floor), then (y_ceil - y), (y - y_floor);
  * tf.floormod on floats: core/kernels/cwise_ops.h google_floor_fmod: r = fmod(x, y); (x < 0) == (y < 0) ? r : fmod(r + y, y);
    on ints: Python's floor modulo;
  * tf.random_uniform: float draws u in [0, 1) mapped as u * (max - min) + min in float32 (random_ops.py); the int32 op draws
    from raw bits, which is not reproduced: here min + floor(u * (max - min)) in float64.
cos / sin / 2^x are evaluated in float64 and rounded once (TF's float32 Eigen versions are not correctly rounded either; the
float32 results can differ in the last bit between the two).  These kernels are not pinned by a TensorFlow run (see
oracle/ref_exec/README.md).
"""
import numpy as np

f32 = np.float32

KP_SWAP = np.array([5, 4, 3, 2, 1, 0, 11, 10, 9, 8, 7, 6, 12, 13, 14, 16, 15, 18, 17, 20, 19, 22, 21, 24, 23])
POSE_SWAP = np.array([0, 1, 2, 6, 7, 8, 3, 4, 5, 9, 10, 11, 15, 16, 17, 12, 13, 14, 18, 19, 20, 24, 25, 26, 21, 22, 23, 27, 28,
                      29, 33, 34, 35, 30, 31, 32, 36, 37, 38, 42, 43, 44, 39, 40, 41, 45, 46, 47, 51, 52, 53, 48, 49, 50, 57, 58,
                      59, 54, 55, 56, 63, 64, 65, 60, 61, 62, 69, 70, 71, 66, 67, 68])
POSE_SIGN = np.tile(np.array([1, -1, -1], f32), 24)
J3D_SWAP = np.array([5, 4, 3, 2, 1, 0, 11, 10, 9, 8, 7, 6, 12, 13])


# ---- random walks -----------------------------------------------------------------------------------------------------------
def uniform_map(u, minval, maxval, dtype):
    """tf.random_uniform(minval, maxval, dtype) from draws u in [0, 1)."""
    if np.dtype(dtype).kind == 'i':
        r = int(maxval) - int(minval)
        return (int(minval) + np.minimum(np.floor(np.asarray(u, np.float64) * r), r - 1)).astype(np.int32)
    lo, hi = f32(minval), f32(maxval)
    return np.asarray(u, f32) * (hi - lo) + lo


def floormod(x, y):
    if np.asarray(x).dtype.kind == 'i':
        return np.mod(x, y)
    y = np.asarray(y, x.dtype)
    r = np.fmod(x, y)
    return np.where((x < 0) == (y < 0), r, np.fmod(r + y, y)).astype(x.dtype)


def walk_branch(minval, maxval, delta_min, delta_max):
    """'zeros', 'iid' (the 'old data augmentation') or 'walk' -- bounded_random_walk's branches, data_utils.py:808-821."""
    if maxval <= minval:
        return 'zeros'
    if minval == delta_min and maxval == delta_max:
        return 'iid'
    return 'walk'


def bounded_random_walk(minval, maxval, delta_min, delta_max, T, dtype=np.float32, dim=1, start_u=None, delta_u=None):
    """data_utils.py:787-835 from given draws: start_u (1, dim), delta_u (T, dim) (the iid branch uses delta_u only)."""
    br = walk_branch(minval, maxval, delta_min, delta_max)
    if br == 'zeros':
        return np.ones((T, dim), f32) * f32(minval)
    if br == 'iid':
        return uniform_map(delta_u, minval, maxval, dtype)
    start = uniform_map(start_u, minval, maxval, dtype)
    size = maxval - minval
    walk = np.cumsum(uniform_map(delta_u, delta_min, delta_max, dtype), axis=0, dtype=np.dtype(dtype))
    t = np.dtype(dtype).type
    x = ((walk + start) - t(minval)) + t(size)
    return (np.abs(floormod(x, t(2 * size)) - t(size)) + t(minval)).astype(dtype)


def tube_walks(T, cfg, draws):
    """TubePreprocessor.__call__'s walks (tube_augmentation.py:56-85) for one tube from its draws dict:
    flip_u (), trans_start_u (1,2), trans_u (T,2), scale_start_u (1,1), scale_u (T,1), rot_start_u (1,1), rot_u (T,1)."""
    flip = bool(f32(draws['flip_u']) < f32(0.5))
    trans = bounded_random_walk(-cfg['trans_max'], cfg['trans_max'] + 1, -cfg['delta_trans_max'], cfg['delta_trans_max'] + 1, T,
                                np.int32, 2, draws.get('trans_start_u'), draws.get('trans_u'))
    scale = bounded_random_walk(-cfg['scale_max'], cfg['scale_max'], -cfg['delta_scale_max'], cfg['delta_scale_max'], T,
                                np.float32, 1, draws.get('scale_start_u'), draws.get('scale_u'))
    rot = bounded_random_walk(-cfg['rotate_max'], cfg['rotate_max'], -cfg['delta_rotate_max'], cfg['delta_rotate_max'], T,
                              np.float32, 1, draws.get('rot_start_u'), draws.get('rot_u'))
    return trans, scale, rot, flip


# ---- TF kernels -------------------------------------------------------------------------------------------------------------
def resize_bilinear(img, Hs, Ws):
    H, W = img.shape[:2]
    img = np.asarray(img, f32)

    def weights(n_out, n_in):
        scale = f32(n_in) / f32(n_out)
        v = np.arange(n_out).astype(f32) * scale
        lo = v.astype(np.int64)
        hi = np.minimum(lo + 1, n_in - 1)
        return lo, hi, v - lo.astype(f32)
    ylo, yhi, yl = weights(Hs, H)
    xlo, xhi, xl = weights(Ws, W)
    xl = xl[None, :, None]
    tl, tr = img[ylo][:, xlo], img[ylo][:, xhi]
    bl, br = img[yhi][:, xlo], img[yhi][:, xhi]
    top = tl + (tr - tl) * xl
    bot = bl + (br - bl) * xl
    return top + (bot - top) * yl[:, None, None]


def rotate_coeffs(theta, S):
    c, s = f32(np.cos(np.float64(theta))), f32(np.sin(np.float64(theta)))
    w1 = h1 = f32(S) - f32(1)
    xo = (w1 - (c * w1 - s * h1)) / f32(2)
    yo = (h1 - (s * w1 + c * h1)) / f32(2)
    return c, s, np.array([c, -s, xo, s, c, yo], f32)


def rotate_image(img, a):
    """contrib.image.rotate's ImageProjectiveTransform, BILINEAR, fill 0, for an S x S x 3 image."""
    S = img.shape[0]
    oy, ox = np.meshgrid(np.arange(S).astype(f32), np.arange(S).astype(f32), indexing='ij')
    x = (a[0] * ox + a[1] * oy) + a[2]
    y = (a[3] * ox + a[4] * oy) + a[5]
    xf, yf = np.floor(x), np.floor(y)
    xc, yc = xf + f32(1), yf + f32(1)

    def rd(yy, xx):
        yi, xi = yy.astype(np.int64), xx.astype(np.int64)
        ok = (yi >= 0) & (yi < S) & (xi >= 0) & (xi < S)
        v = img[np.clip(yi, 0, S - 1), np.clip(xi, 0, S - 1)]
        return np.where(ok[..., None], v, f32(0))
    w = lambda t: t[..., None]
    vyf = w(xc - x) * rd(yf, xf) + w(x - xf) * rd(yf, xc)
    vyc = w(xc - x) * rd(yc, xf) + w(x - xf) * rd(yc, xc)
    return w(yc - y) * vyf + w(y - yf) * vyc


# ---- one frame --------------------------------------------------------------------------------------------------------------
def preprocess_frame(image, label, center, pose, gt3d, trans, scale, rot, flip, S=224, trans_max=20, rotate=False):
    """TubePreprocessor.preprocess_image for one frame.  image float32 [H,W,3] in [0,1]; label [3,K]; center int [2]; pose [72];
    gt3d [14,3]; trans int [2]; scale, rot float32 scalars; flip bool.  -> dict(crop, label, pose, gt3d, center, geom) where
    geom = [Hs, Ws, cx, cy, x0, y0] (the crop's top-left (x0, y0) in the scaled image)."""
    image = np.asarray(image, f32)
    H, W = image.shape[:2]
    label = np.asarray(label, f32)
    K = label.shape[1]
    vis, kp = label[2], label[:2]
    c = np.asarray(center, np.int32) + np.asarray(trans, np.int32)                        # jitter_center
    sf = f32(np.exp2(np.float64(f32(scale))))                                              # jitter_scale
    Hs, Ws = int(f32(H) * sf), int(f32(W) * sf)
    img = resize_bilinear(image, Hs, Ws)
    fy, fx = f32(Hs) / f32(H), f32(Ws) / f32(W)
    x, y = kp[0] * fx, kp[1] * fy
    cx, cy = int(f32(c[0]) * fx), int(f32(c[1]) * fy)
    margin = S // 2
    ms = margin + trans_max + 50
    sx0, sy0 = cx + ms - margin, cy + ms - margin
    rows = np.clip(np.arange(S) + sy0 - ms, 0, Hs - 1)                                     # pad_image_edge + tf.slice
    cols = np.clip(np.arange(S) + sx0 - ms, 0, Ws - 1)
    crop = img[rows][:, cols]
    kx = (x + f32(ms)) - f32(sx0)
    ky = (y + f32(ms)) - f32(sy0)
    pose = np.asarray(pose, f32).copy()
    gt3d = np.asarray(gt3d, f32).copy()
    if rotate:                                                                             # rotate_img
        cs, sn, a = rotate_coeffs(rot, S)
        crop = rotate_image(crop, a)
        cen = f32(S) * f32(0.5)
        x0, y0 = kx - cen, ky - cen
        kx, ky = (x0 * cs + y0 * sn) + cen, (x0 * (-sn) + y0 * cs) + cen
        R = np.array([[cs, -sn, 0], [sn, cs, 0], [0, 0, 1]], f32)
        mean = f32(np.sum(gt3d, dtype=f32) / f32(42))
        g0 = gt3d - mean
        gt3d = np.stack([((g0[:, 0] * R[0, j] + g0[:, 1] * R[1, j]) + g0[:, 2] * R[2, j]) for j in range(3)], 1) + mean
        from oracle import smpl_ref
        R0 = smpl_ref.batch_rodrigues(pose[None, :3])[0]
        Rn = np.array([[(R[0, i] * R0[0, j] + R[1, i] * R0[1, j]) + R[2, i] * R0[2, j] for j in range(3)] for i in range(3)], f32)
        pose[:3] = smpl_ref.batch_rot2aa(Rn[None])[0]
    if flip:                                                                               # flip_image
        crop = crop[:, ::-1]
        kx = (f32(S) - kx) - f32(1)
        if K != 25:
            raise ValueError('flip_image swaps the 25 keypoints of its name lists, got K=%d' % K)
        kx, ky, vis = kx[KP_SWAP], ky[KP_SWAP], vis[KP_SWAP]
        pose = pose[POSE_SWAP] * POSE_SIGN
        j = gt3d[J3D_SWAP] * np.array([-1, 1, 1], f32)
        gt3d = j - (np.sum(j, axis=0, dtype=f32) / f32(14))
    v = (vis > 0).astype(f32)
    lab = np.stack([f32(2) * (kx / f32(S)) - f32(1), f32(2) * (ky / f32(S)) - f32(1), v]) * v
    return {'crop': ((crop - f32(0.5)) * f32(2)).astype(f32), 'label': lab.astype(f32), 'pose': pose.astype(f32),
            'gt3d': gt3d.astype(f32), 'center': np.array([cx, cy], np.int32),
            'geom': np.array([Hs, Ws, cx, cy, sx0 - ms, sy0 - ms], np.int32)}


def augment_tube(images, labels, centers, poses, gt3ds, trans, scale, rot, flip, S=224, trans_max=20, rotate=False):
    """preprocess_frame over a tube; images [T,H,W,3] float in [0,1] (or uint8: / 255. as the converters do).  Returns stacked
    arrays under the keys of preprocess_frame plus 'images' (= 'crop')."""
    images = np.asarray(images)
    if images.dtype == np.uint8:
        images = (images / 255.).astype(f32)
    out = [preprocess_frame(images[t], labels[t], centers[t], poses[t], gt3ds[t], trans[t], np.asarray(scale).reshape(-1)[t],
                            np.asarray(rot).reshape(-1)[t], flip, S, trans_max, rotate) for t in range(len(images))]
    res = {k: np.stack([o[k] for o in out]) for k in out[0]}
    res['images'] = res['crop']
    return res


CFG_KEYS = ('trans_max', 'delta_trans_max', 'scale_max', 'delta_scale_max', 'rotate_max', 'delta_rotate_max')
DRAW_KEYS = ('flip_u', 'trans_start_u', 'trans_u', 'scale_start_u', 'scale_u', 'rot_start_u', 'rot_u')


def load_fixture(path):
    """tests/golden/tube_aug_v1.npz -> [(inputs, cfg, S, draws, reference outputs)] per tube (see make_tube_golden.py)."""
    z = np.load(path)
    out = []
    i = 0
    while 't%d_cfg' % i in z.files:
        p = 't%d_' % i
        c = z[p + 'cfg']
        cfg = dict(zip(CFG_KEYS, [int(c[0]), int(c[1])] + [float(v) for v in c[2:6]]))
        x = {k: z[p + k] for k in ('frames', 'image_sizes', 'labels', 'centers', 'poses', 'gt3ds')}
        draws = {k: z[p + k] for k in DRAW_KEYS if p + k in z.files}
        ref = {k[len(p) + 4:]: z[k] for k in z.files if k.startswith(p + 'out_')}
        out.append((x, cfg, int(c[6]), draws, ref))
        i += 1
    return out
