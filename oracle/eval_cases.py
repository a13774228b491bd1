"""Seeded inputs for the evaluation tests, golden generator and benchmark (numpy only: no import of `src`, so that the golden generator
can load it by path while `src` names the reference's package)."""
import numpy as np


def _rodrigues(aa):
    th = np.linalg.norm(aa, axis=-1, keepdims=True)
    k = aa / np.maximum(th, 1e-12)
    K = np.zeros(aa.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -k[..., 2], k[..., 1], -k[..., 0]
    K = K - np.swapaxes(K, -1, -2)
    s, c = np.sin(th)[..., None], np.cos(th)[..., None]
    return np.eye(3) + s * K + (1 - c) * (K @ K)


def make_eval_tubes(lens, K=25, seed=0, img_size=224, min_visible=6, special=True):
    """Seeded float32 tubes in the layout test_sequence feeds compute_errors_batched: kps_gt [n,K,3] (pixels, vis 0/1), kps_pred [n,K,2]
    in [-1, 1], joints_gt / joints_pred [n,14,3], poses_gt [n,72] axis-angle, poses_pred [n,24,3,3], shape_gt [10], shapes_pred
    [n,10].  With `special`, the first frames of the split carry the edge cases: no visible keypoint, exactly min_visible visible
    keypoints, 3-D visibility exactly at and one above the threshold, a mirrored prediction (the reflection branch of the
    similarity transform), a prediction whose joints all coincide (NaN PA-MPJPE), and pose rotations near pi."""
    rng = np.random.RandomState(seed)
    tubes = []
    for n in lens:
        base = rng.normal(0, 0.3, size=(1, 14, 3)) + np.linspace(-0.8, 0.8, 14)[None, :, None] * np.array([0.2, 1.0, 0.1])
        gt3 = base + rng.normal(0, 0.02, size=(n, 14, 3)) + np.cumsum(rng.normal(0, 0.01, size=(n, 1, 3)), axis=0)
        pred3 = gt3 * rng.uniform(0.8, 1.2) + rng.normal(0, 0.05, size=(n, 14, 3))
        kp_gt = np.empty((n, K, 3))
        kp_gt[..., :2] = rng.uniform(0, img_size, size=(n, K, 2))
        kp_gt[..., 2] = rng.rand(n, K) > 0.2
        kp_pred = (kp_gt[..., :2] / img_size * 2 - 1) * rng.uniform(0.9, 1.1) + rng.normal(0, 0.05, size=(n, K, 2))
        poses_gt = rng.normal(0, 0.3, size=(n, 72))
        aa_pred = poses_gt.reshape(n, 24, 3) + rng.normal(0, 0.1, size=(n, 24, 3))
        tubes.append(dict(kps_gt=kp_gt, kps_pred=kp_pred, joints_gt=gt3, joints_pred=pred3, poses_gt=poses_gt, poses_pred=aa_pred,
                          shape_gt=rng.normal(0, 1, size=10), shapes_pred=rng.normal(0, 1, size=(n, 10))))
    if special:
        flat = [(t, i) for t in tubes for i in range(len(t['kps_gt']))]
        edits = [
            lambda t, i: t['kps_gt'][i, :, 2].__setitem__(slice(None), 0),                            # nothing visible
            lambda t, i: (t['kps_gt'][i, :, 2].__setitem__(slice(None), 0),
                          t['kps_gt'][i, :min_visible, 2].__setitem__(slice(None), 1)),                # exactly min_visible
            lambda t, i: (t['kps_gt'][i, :14, 2].__setitem__(slice(None), 0),
                          t['kps_gt'][i, :min_visible, 2].__setitem__(slice(None), 1)),                # 3-D vis sum == threshold
            lambda t, i: (t['kps_gt'][i, :14, 2].__setitem__(slice(None), 0),
                          t['kps_gt'][i, :min_visible + 1, 2].__setitem__(slice(None), 1)),            # one above
            lambda t, i: t['joints_pred'].__setitem__(i, t['joints_gt'][i] * np.array([-1.0, 1.0, 1.0])),   # mirrored
            lambda t, i: t['joints_pred'].__setitem__(i, np.tile(t['joints_pred'][i, :1], (14, 1))),    # all joints coincide
            lambda t, i: t['poses_pred'][i].__setitem__(slice(None), _near_pi(rng)),                  # rotations near pi
        ]
        for e, (t, i) in zip(edits, flat):
            e(t, i)
    for t in tubes:
        t['poses_pred'] = _rodrigues(t['poses_pred'])
        for k in t:
            t[k] = np.ascontiguousarray(t[k], np.float32)
    return tubes


def _near_pi(rng):
    axis = rng.normal(size=(24, 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    return axis * (np.pi - rng.uniform(0, 1e-3, size=(24, 1)))


# ---------------------------------------------------------------------------------------------------------------- golden access
METRICS = ('accel', 'kp', 'kp_pa', 'kp_pck', 'accel_error', 'joints', 'joints_pa', 'mesh_posed', 'mesh_tpose', 'pose', 'shape')


def golden_tubes(g, run):
    """The stored input tubes of run 'nat' or 'f64' (float32 arrays, oracle/eval_cases.py layout)."""
    tubes, i = [], 0
    while 'in_%s/t%d/kps_gt' % (run, i) in g:
        tubes.append({k: g['in_%s/t%d/%s' % (run, i, k)] for k in
                      ('kps_gt', 'kps_pred', 'joints_gt', 'joints_pred', 'poses_gt', 'poses_pred', 'shape_gt', 'shapes_pred')})
        i += 1
    return tubes


def near_pi(Rs):
    """Frames of [n, 24, 3, 3] rotations with a rotation within 1e-2 rad of pi."""
    cos = (np.trace(np.asarray(Rs, np.float64), axis1=2, axis2=3) - 1) / 2
    return (cos < np.cos(np.pi - 1e-2)).any(axis=1)


def golden_errors(g, prefix):
    return {k: g['%s/%s' % (prefix, k)] for k in METRICS if '%s/%s' % (prefix, k) in g}


def assert_errors_close(got, want, rtol, atol, key_tol=None):
    assert sorted(got) == sorted(want)
    for k in want:
        a, b = np.asarray(got[k], np.float64), np.asarray(want[k], np.float64)
        assert a.shape == b.shape, (k, a.shape, b.shape)
        assert np.array_equal(np.isnan(a), np.isnan(b)), k
        ok = ~np.isnan(b)
        if k == 'kp_pck':
            assert np.array_equal(a[ok], b[ok]), k
            continue
        r, t = (key_tol or {}).get(k, (rtol, atol))
        t = np.broadcast_to(t, b.shape)[ok] if np.ndim(t) and np.ndim(b) else t
        assert np.all(np.abs(a[ok] - b[ok]) <= t + r * np.abs(b[ok])), (k, np.abs(a[ok] - b[ok]).max())
