"""Generates tests/golden/tube_aug_v1.npz by EXECUTING THE REFERENCE'S OWN SOURCE: src/util/tube_augmentation.py
(TubePreprocessor.__call__ with return_walk=True, hence preprocess_image over every frame) and src/util/data_utils.py
(bounded_random_walk, jitter_center, jitter_scale, pad_image_edge, rotate_img, flip_image, reflect_pose, reflect_joints3d,
rescale_image), with src/tf_smpl/batch_lbs.py for rotate_img's pose.  It runs over the numpy TensorFlow stand-in in oracle/ref_exec,
set up as make_ref_exec_golden.py does; extend_standin() adds, in this process only, what these files need that the stand-in does not
have, each from its TF 1.x definition:
  - tf.random_uniform fed from recorded draws: u in [0, 1) (float32, seeded here) mapped as u * (max - min) + min in float32
    (random_ops.py); int32 as min + floor(u * (max - min)) in float64 (TF's raw-bit int draw is not reproduced);
  - tf.cumsum (sequential, in the input's dtype), Tensor % (floormod: Python's on ints, google_floor_fmod on floats), tf.less,
    tf.fill, tf.ones with a tensor dimension, tf.to_int32, tf.tile with tensor multiples, tf.slice (fails outside the input as TF
    does), tf.reverse, Tensor ** and 2 ** Tensor (tf.pow);
  - tf.map_fn and tf.cond, unrolled over the statically known number of frames / evaluated on both branches and selected;
  - tf.image.resize_images (resize_bilinear, align_corners=False: in = out * (in / out), lower = (int) in, upper = min(lower + 1,
    in - 1), top / bottom / vertical lerps) and tf.contrib.image.rotate (angles_to_projective_transforms, then the BILINEAR
    ImageProjectiveTransform with zero fill).
The inputs enter as constants, so that shapes that depend on the walks (the scaled image) are known when the graph is built.

Three tubes at S = 64 (TubePreprocessor's constructor arguments in brackets):
  0: 96 x 96 uint8 noise, T = 4, the 'old augmentation' branch (20 / 20, 0.3 / 0.3), flipped;
  1: 72 x 100 uint8 noise (non-square), T = 5, the walk branch (20 / 3, 0.3 / 0.05), not flipped;
  2: 80 x 80 float ramp, T = 3, rotate_max = 0.6, delta_rotate_max = 0.15 (walk), flipped.
The uint8 frames are fed as frames / 255. (float32), as the converters do.  Stored per tube (prefix t<i>_): the frames, the inputs,
the configuration, the recorded draws under the walk each feeds (flip_u, trans_start_u, trans_u, scale_start_u, scale_u, rot_start_u,
rot_u; no *_start_u in the iid branch, no rot_* where rotate_max = 0) and the reference's outputs (images, labels, poses, gt3ds,
centers, trans_walk, scale_walk, rot_walk).

Needs a checkout of the reference project, named by HD_REFERENCE_ROOT.  Run from the repo root:
    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_tube_golden.py            (writes tests/golden/tube_aug_v1.npz)
    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_tube_golden.py --check    (exit 0 when it reproduces the file)
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'tube_aug_v1.npz')
S = 64
TUBES = [
    dict(T=4, H=96, W=96, kind='u8', flip=True, cfg=(20, 20, 0.3, 0.3, 0, 0)),
    dict(T=5, H=72, W=100, kind='u8', flip=False, cfg=(20, 3, 0.3, 0.05, 0, 0)),
    dict(T=3, H=80, W=80, kind='ramp', flip=True, cfg=(20, 3, 0.3, 0.05, 0.6, 0.15)),
]
ONE_MINUS = np.nextafter(np.float32(1), np.float32(0))


def _by_path(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def draw_keys(cfg):
    """The order TubePreprocessor.__call__ consumes draws in (tube_augmentation.py:57-85, data_utils.py:808-833)."""
    tm, dtm, sm, dsm, rm, drm = cfg
    keys = ['flip_u']
    for name, lo, hi, dlo, dhi in (('trans', -tm, tm + 1, -dtm, dtm + 1), ('scale', -sm, sm, -dsm, dsm), ('rot', -rm, rm, -drm, drm)):
        if hi <= lo:
            continue
        if not (lo == dlo and hi == dhi):
            keys.append(name + '_start_u')
        keys.append(name + '_u')
    return keys


def inputs(i, tube):
    rng = np.random.RandomState(300 + i)
    T, H, W, K = tube['T'], tube['H'], tube['W'], 25
    if tube['kind'] == 'u8':
        frames = rng.randint(0, 256, size=(T, H, W, 3)).astype(np.uint8)
        images = (frames / 255.).astype(np.float32)
    else:
        yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing='ij')
        ramp = np.stack([xx / (W - 1.), yy / (H - 1.), (xx + yy) / (W + H - 2.)], -1)
        frames = np.repeat(ramp[None], T, 0).astype(np.float32)
        images = frames
    centers = np.stack([rng.randint(W // 3, 2 * W // 3, size=T), rng.randint(H // 3, 2 * H // 3, size=T)], 1).astype(np.int32)
    labels = np.zeros((T, 3, K), np.float32)
    labels[:, 0] = rng.uniform(0, W, size=(T, K))
    labels[:, 1] = rng.uniform(0, H, size=(T, K))
    labels[:, 2] = rng.choice([0., 1.], p=[0.3, 0.7], size=(T, K))
    poses = rng.normal(0, 0.4, size=(T, 72)).astype(np.float32)
    gt3ds = rng.normal(0, 0.4, size=(T, 14, 3)).astype(np.float32)
    sizes = np.tile(np.array([[H, W]], np.int32), (T, 1))
    return dict(frames=frames, images=images, image_sizes=sizes, labels=labels, centers=centers, poses=poses, gt3ds=gt3ds)


def extend_standin(tf, draw_source):
    """See the module docstring.  draw_source(shape) -> float32 draws in [0, 1)."""
    T_ = tf.Tensor

    def static(v):
        return int(np.asarray(v.probe)) if isinstance(v, T_) else int(v)

    def random_uniform(shape, minval=0, maxval=None, dtype=np.float32, seed=None, name=None):
        shp = [static(s) for s in (shape if isinstance(shape, (list, tuple)) else [shape])]
        u = draw_source(shp)
        if np.dtype(dtype).kind == 'i':
            r = int(maxval) - int(minval)
            return tf._const_tensor((int(minval) + np.minimum(np.floor(u.astype(np.float64) * r), r - 1)).astype(np.int32))
        lo = tf.convert_to_tensor(0. if minval is None else minval, np.float32)
        hi = tf.convert_to_tensor(1. if maxval is None else maxval, np.float32)
        return tf.add(tf._const_tensor(u) * (hi - lo), lo)
    tf.random_uniform = random_uniform

    def floormod(a, b):
        if a.dtype.kind in 'iu':
            return np.mod(a, b)
        r = np.fmod(a, b)
        return np.where((a < 0) == (b < 0), r, np.fmod(r + b, b)).astype(a.dtype)
    T_.__mod__ = lambda self, o: tf._binary(floormod, 'floormod')(self, o)
    T_.__pow__ = lambda self, o: tf._binary(lambda a, b: np.power(a, b), 'pow')(self, o)
    T_.__rpow__ = lambda self, o: tf._binary(lambda a, b: np.power(a, b), 'pow')(o, self)
    tf.less = lambda x, y, name=None: tf._binary(lambda a, b: a < b, 'less')(x, y)
    tf.to_int32 = lambda x, name=None: tf.cast(x, np.int32)
    tf.cumsum = lambda x, axis=0, **kw: tf._op(lambda a: np.cumsum(a, axis=axis, dtype=a.dtype), [tf.convert_to_tensor(x)], 'cumsum')

    def fill(dims, value, name=None):
        shp = [static(d) for d in dims]
        return tf._op(lambda v: np.full(shp, v, dtype=np.asarray(v).dtype), [tf.convert_to_tensor(value)], 'fill')
    tf.fill = fill
    _ones = tf.ones
    tf.ones = lambda shape, dtype=np.float32, name=None: _ones([static(s) for s in shape], dtype)

    def tile(x, multiples, name=None):
        m = tf.stack([tf.convert_to_tensor(v, np.int32) if not isinstance(v, T_) else v for v in multiples])
        return tf._op(lambda a, mm: np.tile(a, [int(v) for v in mm]), [tf.convert_to_tensor(x), m], 'tile')
    tf.tile = tile

    def slice_(x, begin, size, name=None):
        def fn(a, b, s):
            out = a[tuple(slice(int(bb), int(bb) + int(ss)) for bb, ss in zip(b, s))]
            if any(int(bb) < 0 for bb in b) or list(out.shape) != [int(ss) for ss in s]:
                raise ValueError('Expected begin and size arguments to be within the input: %s + %s vs %s' % (b, s, a.shape))
            return out
        return tf._op(fn, [tf.convert_to_tensor(x), tf.convert_to_tensor(begin, np.int32), tf.convert_to_tensor(size, np.int32)],
                      'slice')
    import builtins

    class _SliceMeta(type):
        """tf.slice becomes the stand-in module's global `slice`, which its own indexing code also reads as Python's slice type:
        the attribute answers as that type, and as tf.slice when called with a Tensor."""
        def __instancecheck__(cls, obj):
            return isinstance(obj, builtins.slice)

        def __call__(cls, *args, **kw):
            if args and isinstance(args[0], T_):
                return slice_(*args, **kw)
            return builtins.slice(*args)
    tf.slice = _SliceMeta('slice', (), {})
    tf.reverse = lambda x, axis, name=None: tf._op(lambda a: np.flip(a, axis=tuple(int(v) for v in axis)).copy(),
                                                     [tf.convert_to_tensor(x)], 'reverse')

    def map_fn(fn, elems, dtype=None, **kw):
        seq = isinstance(elems, (list, tuple))
        es = list(elems) if seq else [elems]
        n = es[0].probe.shape[0]
        outs = [fn(tuple(e[t] for e in es) if seq else es[0][t]) for t in range(n)]
        single = not isinstance(outs[0], (list, tuple))
        outs = [[o] if single else list(o) for o in outs]
        dts = list(dtype) if isinstance(dtype, (list, tuple)) else [dtype] * len(outs[0])
        res = [tf.cast(tf.stack([o[j] for o in outs]), dts[j]) for j in range(len(outs[0]))]
        return res[0] if single else tuple(res)
    tf.map_fn = map_fn

    def cond(pred, true_fn, false_fn, name=None):
        a, b = true_fn(), false_fn()
        pick = lambda x, y: tf._op(lambda p, u, v: u if bool(p) else v, [pred, tf.convert_to_tensor(x), tf.convert_to_tensor(y)], 'cond')
        if isinstance(a, (list, tuple)):
            return type(a)(pick(x, y) for x, y in zip(a, b))
        return pick(a, b)
    tf.cond = cond

    def resize_bilinear(img, size):
        H, W = img.shape[:2]
        Hs, Ws = int(size[0]), int(size[1])

        def weights(n_out, n_in):
            scale = np.float32(n_in) / np.float32(n_out)
            v = np.arange(n_out).astype(np.float32) * scale
            lo = v.astype(np.int64)
            return lo, np.minimum(lo + 1, n_in - 1), v - lo.astype(np.float32)
        ylo, yhi, yl = weights(Hs, H)
        xlo, xhi, xl = weights(Ws, W)
        img = img.astype(np.float32)
        top = img[ylo][:, xlo] + (img[ylo][:, xhi] - img[ylo][:, xlo]) * xl[None, :, None]
        bot = img[yhi][:, xlo] + (img[yhi][:, xhi] - img[yhi][:, xlo]) * xl[None, :, None]
        return top + (bot - top) * yl[:, None, None]
    tf.image = types.SimpleNamespace(
        resize_images=lambda images, size, method=0, align_corners=False: tf._op(resize_bilinear, [
            tf.convert_to_tensor(images), tf.convert_to_tensor(size, np.int32)], 'resize_bilinear'))

    def transform(img, a):
        Hh, Ww = img.shape[:2]
        oy, ox = np.meshgrid(np.arange(Hh).astype(np.float32), np.arange(Ww).astype(np.float32), indexing='ij')
        proj = a[6] * ox + a[7] * oy + np.float32(1)
        x = (a[0] * ox + a[1] * oy + a[2]) / proj
        y = (a[3] * ox + a[4] * oy + a[5]) / proj
        xf, yf = np.floor(x), np.floor(y)
        xc, yc = xf + np.float32(1), yf + np.float32(1)

        def rd(yy, xx):
            yi, xi = yy.astype(np.int64), xx.astype(np.int64)
            ok = (yi >= 0) & (yi < Hh) & (xi >= 0) & (xi < Ww)
            return np.where(ok[..., None], img[np.clip(yi, 0, Hh - 1), np.clip(xi, 0, Ww - 1)], np.float32(0))
        e = lambda t: t[..., None]
        vyf = e(xc - x) * rd(yf, xf) + e(x - xf) * rd(yf, xc)
        vyc = e(xc - x) * rd(yc, xf) + e(x - xf) * rd(yc, xc)
        return (e(yc - y) * vyf + e(y - yf) * vyc).astype(img.dtype)

    def rotate(images, angles, interpolation='NEAREST', name=None):
        assert interpolation == 'BILINEAR'
        images = tf.convert_to_tensor(images)
        h = tf.cast(tf.shape(images)[0], np.float32)
        w = tf.cast(tf.shape(images)[1], np.float32)
        ang = tf.convert_to_tensor(angles)
        x_off = ((w - 1) - (tf.cos(ang) * (w - 1) - tf.sin(ang) * (h - 1))) / 2.0
        y_off = ((h - 1) - (tf.sin(ang) * (w - 1) + tf.cos(ang) * (h - 1))) / 2.0
        xf = tf.concat([tf.cos(ang), -tf.sin(ang), x_off, tf.sin(ang), tf.cos(ang), y_off, tf.zeros((2,), np.float32)], 0)
        return tf._op(transform, [images, xf], 'image_projective_transform')
    import tensorflow.contrib as contrib
    contrib.image = types.SimpleNamespace(rotate=rotate)


def run_reference():
    gen = _by_path('_make_ref_exec_golden', os.path.join(HERE, 'make_ref_exec_golden.py'))
    gen.setup_paths()
    import tensorflow as tf
    rng = np.random.RandomState(2024)
    record = []

    def draw_source(shape):
        u = np.minimum(rng.random_sample(shape).astype(np.float32), ONE_MINUS)
        record.append(u)
        return u
    from src.util.tube_augmentation import TubePreprocessor
    res = {}
    for i, tube in enumerate(TUBES):
        x = inputs(i, tube)
        keys = draw_keys(tube['cfg'])
        del record[:]
        first = [np.float32(0.25 if tube['flip'] else 0.75)]

        def source(shape, _first=first):
            if _first:          # the tube's flip draw, chosen so that the three cases cover both flips
                u = np.full(shape, _first.pop(), np.float32)
                record.append(u)
                return u
            return draw_source(shape)
        extend_standin(tf, source)
        pre = TubePreprocessor(S, *tube['cfg'])
        out = pre(tf.convert_to_tensor(x['images']), tf.convert_to_tensor(x['image_sizes']), tf.convert_to_tensor(x['labels']),
                  tf.convert_to_tensor(x['centers']), tf.convert_to_tensor(x['poses']), tf.convert_to_tensor(x['gt3ds']),
                  return_walk=True)
        assert len(record) == len(keys), (len(record), keys)
        with tf.Session() as sess:
            got = sess.run(out)
        p = 't%d_' % i
        res[p + 'frames'] = x['frames']
        for k in ('image_sizes', 'labels', 'centers', 'poses', 'gt3ds'):
            res[p + k] = x[k]
        res[p + 'cfg'] = np.array(tube['cfg'] + (S,), np.float64)
        for k, u in zip(keys, record):
            res[p + k] = np.asarray(u, np.float32)
        for k, v in got.items():
            res[p + 'out_' + k] = np.asarray(v)
    return res


def main():
    res = run_reference()
    if '--check' in sys.argv:
        with np.load(OUT) as z:
            same = sorted(z.files) == sorted(res) and all(np.array_equal(z[k], res[k]) for k in z.files)
        print('reproduces %s: %s' % (OUT, same))
        raise SystemExit(0 if same else 1)
    np.savez_compressed(OUT, **res)
    print('wrote %s: %s' % (OUT, ', '.join('%s %s %s' % (k, np.shape(v), np.asarray(v).dtype) for k, v in res.items())))


if __name__ == '__main__':
    main()
