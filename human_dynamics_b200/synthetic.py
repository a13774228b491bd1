"""Synthetic assets for the HMMR hot path (no real SMPL pkl / checkpoint exists offline).

Everything here is plain numpy and deterministic in its seed, so the GPU product
path, the CPU oracle and the tests all see identical constants.

Shapes, names and layouts follow the reference:
  * SMPL dict keys mirror the pickle consumed by `src/tf_smpl/batch_smpl.py:27-86`
    (v_template, shapedirs, J_regressor, posedirs, kintree_table, weights,
    cocoplus_regressor) -- dense ndarrays instead of chumpy / scipy-sparse.
  * weight dict keys are the TF-slim variable names a checkpoint loader would see
    (SURVEY.md Appendix A.6): conv weights HWIO, FC weights [in, out].
"""
from __future__ import annotations

import numpy as np

NUM_VERTS = 6890
NUM_JOINTS = 24
NUM_BETAS = 10
NUM_POSE_BASIS = 207

# Standard SMPL kinematic tree (kintree_table[0]); root stored as uint32(-1) in the pkl,
# batch_smpl.py:66 casts it with astype(np.int32) -> -1.
SMPL_PARENTS = np.array(
    [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21],
    dtype=np.int64)

# resnet_v2_50 blocks: (base_depth, num_units, stride) -- stride on the LAST unit.
RESNET_BLOCKS = ((64, 3, 2), (128, 4, 2), (256, 6, 2), (512, 3, 1))


def make_synthetic_smpl(seed: int = 2, num_kps: int = 25, dense_weights: bool = False,
                        num_verts: int = NUM_VERTS) -> dict:
    """A random but well-conditioned stand-in for the licensed SMPL pickle.

    `weights` is row-stochastic with <=4 non-zeros per vertex (like real SMPL) unless
    `dense_weights`; regressors are non-negative and column-stochastic over vertices.
    """
    rng = np.random.RandomState(seed)
    V = num_verts
    # capsule-ish figure ~1.7 m tall
    h = rng.uniform(-0.85, 0.85, size=V)
    ang = rng.uniform(0, 2 * np.pi, size=V)
    rad = 0.12 + 0.05 * rng.rand(V)
    v_template = np.stack([rad * np.cos(ang), h, rad * np.sin(ang)], axis=1)

    shapedirs = rng.normal(0, 0.01, size=(V, 3, NUM_BETAS))
    posedirs = rng.normal(0, 0.001, size=(V, 3, NUM_POSE_BASIS))

    def _regressor(cols, nnz_lo, nnz_hi):
        R = np.zeros((cols, V))
        for j in range(cols):
            nnz = rng.randint(nnz_lo, nnz_hi + 1)
            idx = rng.choice(V, size=nnz, replace=False)
            w = rng.rand(nnz) + 0.05
            R[j, idx] = w / w.sum()
        return R

    J_regressor = _regressor(NUM_JOINTS, 10, 30)           # (24, V) like the pkl (sparse there)
    cocoplus_regressor = _regressor(num_kps, 10, 30)       # (K, V)

    if dense_weights:
        W = rng.rand(V, NUM_JOINTS) + 0.01
    else:
        W = np.zeros((V, NUM_JOINTS))
        for v in range(V):
            nnz = rng.randint(1, 5)
            idx = rng.choice(NUM_JOINTS, size=nnz, replace=False)
            W[v, idx] = rng.rand(nnz) + 0.05
    W = W / W.sum(axis=1, keepdims=True)

    kintree = np.stack([SMPL_PARENTS.astype(np.uint32), np.arange(NUM_JOINTS, dtype=np.uint32)])
    return {
        'v_template': v_template.astype(np.float64),
        'shapedirs': shapedirs.astype(np.float64),
        'J_regressor': J_regressor.astype(np.float64),
        'posedirs': posedirs.astype(np.float64),
        'kintree_table': kintree,
        'weights': W.astype(np.float64),
        'cocoplus_regressor': cocoplus_regressor.astype(np.float64),
    }


def make_smooth_mesh(seed: int = 11):
    """A closed genus-0 mesh with SMPL's vertex and face counts for rendering tests and benchmarks: 84 rings of 82 vertices + 2
    poles (V = 6890, F = 2V - 4 = 13776), radially perturbed by a few seeded low-frequency harmonics and stretched to a body-like
    0.5 x 1.7 x 0.4 ellipsoid.  -> (verts float32 [V,3], faces int64 [F,3])."""
    rng = np.random.RandomState(seed)
    Rn, K = 84, 82
    th = np.pi * (np.arange(1, Rn + 1) / (Rn + 1.0))
    ph = 2 * np.pi * np.arange(K) / K
    T, P = np.meshgrid(th, ph, indexing='ij')
    rad = 1.0 + sum(rng.uniform(-0.08, 0.08) * np.cos(a * T + rng.uniform(0, 6)) * np.cos(b * P + rng.uniform(0, 6))
                    for a, b in ((2, 1), (3, 2), (1, 3), (4, 1)))
    pts = np.stack([rad * np.sin(T) * np.cos(P), rad * np.cos(T), rad * np.sin(T) * np.sin(P)], -1).reshape(-1, 3)
    verts = np.concatenate([[[0, 1.0, 0]], pts, [[0, -1.0, 0]]]) * np.array([0.25, 0.85, 0.2])
    ring = lambda r, k: 1 + r * K + (k % K)
    faces = [[0, ring(0, k + 1), ring(0, k)] for k in range(K)]
    for r in range(Rn - 1):
        for k in range(K):
            faces += [[ring(r, k), ring(r, k + 1), ring(r + 1, k)], [ring(r, k + 1), ring(r + 1, k + 1), ring(r + 1, k)]]
    faces += [[len(verts) - 1, ring(Rn - 1, k), ring(Rn - 1, k + 1)] for k in range(K)]
    return verts.astype(np.float32), np.array(faces, np.int64)


def make_mean_param(seed: int = 3) -> np.ndarray:
    """mean_param [1,85] as built by tester.py:118-141: cam [0.9,0,0], pose root [pi,0,0]."""
    rng = np.random.RandomState(seed)
    pose = rng.normal(0, 0.2, size=72)
    pose[:3] = 0.0
    pose[0] = np.pi
    shape = rng.normal(0, 1.0, size=10)
    return np.hstack(([0.9, 0.0, 0.0], pose, shape))[None].astype(np.float32)


def _he(rng, shape, fan_in, gain=1.0):
    return (rng.normal(0, 1.0, size=shape) * gain * np.sqrt(2.0 / fan_in)).astype(np.float32)


def _bn(rng, c, prefix, out):
    out[prefix + '/gamma'] = rng.uniform(0.5, 1.5, size=c).astype(np.float32)
    out[prefix + '/beta'] = rng.normal(0, 0.1, size=c).astype(np.float32)
    out[prefix + '/moving_mean'] = rng.normal(0, 0.1, size=c).astype(np.float32)
    out[prefix + '/moving_variance'] = rng.uniform(0.5, 1.5, size=c).astype(np.float32)


def make_resnet_weights(seed: int = 1, blocks=RESNET_BLOCKS, out: dict | None = None) -> dict:
    """resnet_v2_50 variables (slim names, HWIO)."""
    rng = np.random.RandomState(seed)
    w = {} if out is None else out
    p = 'resnet_v2_50'
    w[p + '/conv1/weights'] = _he(rng, (7, 7, 3, 64), 7 * 7 * 3)
    w[p + '/conv1/biases'] = rng.normal(0, 0.1, size=64).astype(np.float32)
    d_in = 64
    for b, (base, units, _stride) in enumerate(blocks, start=1):
        depth = 4 * base
        for u in range(1, units + 1):
            q = '%s/block%d/unit_%d/bottleneck_v2' % (p, b, u)
            _bn(rng, d_in, q + '/preact', w)
            if d_in != depth:
                w[q + '/shortcut/weights'] = _he(rng, (1, 1, d_in, depth), d_in, 0.7)
                w[q + '/shortcut/biases'] = rng.normal(0, 0.05, size=depth).astype(np.float32)
            w[q + '/conv1/weights'] = _he(rng, (1, 1, d_in, base), d_in)
            _bn(rng, base, q + '/conv1/BatchNorm', w)
            w[q + '/conv2/weights'] = _he(rng, (3, 3, base, base), 9 * base)
            _bn(rng, base, q + '/conv2/BatchNorm', w)
            # residual branch kept small so the un-normalised trunk stays O(1) over 16 units
            w[q + '/conv3/weights'] = _he(rng, (1, 1, base, depth), base, 0.35)
            w[q + '/conv3/biases'] = rng.normal(0, 0.05, size=depth).astype(np.float32)
            d_in = depth
    _bn(rng, d_in, p + '/postnorm', w)
    return w


def _small_xavier(rng, shape, fan_in, fan_out, factor):
    # variance_scaling_initializer(factor, mode='FAN_AVG', uniform=True): models.py:106,206
    limit = np.sqrt(3.0 * factor / ((fan_in + fan_out) / 2.0))
    return rng.uniform(-limit, limit, size=shape).astype(np.float32)


def make_fmovie_weights(seed: int = 4, num_conv_layers: int = 3, C: int = 2048,
                        out: dict | None = None) -> dict:
    """AZ_FC_block* variables (models.py:159,182,192,219)."""
    rng = np.random.RandomState(seed)
    w = {} if out is None else out
    for i in range(num_conv_layers):
        name = 'block_%d' % i
        for k in (1, 2):
            w['AZ_FC_block_preact_gn%d%s/gamma' % (k, name)] = rng.uniform(0.5, 1.5, size=C).astype(np.float32)
            w['AZ_FC_block_preact_gn%d%s/beta' % (k, name)] = rng.normal(0, 0.1, size=C).astype(np.float32)
        w['AZ_FC_block2_conv1%s/weights' % name] = _he(rng, (3, 1, C, C), 3 * C)
        w['AZ_FC_block2_conv1%s/biases' % name] = rng.normal(0, 0.05, size=C).astype(np.float32)
        # reference uses small_xavier(factor=.001) for conv2 (models.py:206); use a larger factor
        # so the temporal branch visibly contributes and parity tests exercise it
        w['AZ_FC_block2_conv2%s/weights' % name] = _small_xavier(rng, (3, 1, C, C), 3 * C, 3 * C, 0.3)
        w['AZ_FC_block2_conv2%s/biases' % name] = rng.normal(0, 0.05, size=C).astype(np.float32)
    return w


def make_ief_weights(seed: int = 5, delta_t_values=(-5, 5), feat: int = 2048,
                     scope: str = 'single_view_ief', out: dict | None = None) -> dict:
    """IEF heads: main (85) + one 72-d head per non-zero delta_t (models.py:344-347)."""
    rng = np.random.RandomState(seed)
    w = {} if out is None else out
    heads = [(scope, 85)]
    for dt in delta_t_values:
        if dt == 0:
            continue
        heads.append((scope + ('_future%d' % dt if dt > 0 else '_past%d' % abs(dt)), 72))
    for sc, d in heads:
        q = sc + '/3D_module'
        w[q + '/fc1/weights'] = _he(rng, (feat + d, 1024), feat + d)
        w[q + '/fc1/biases'] = rng.normal(0, 0.05, size=1024).astype(np.float32)
        w[q + '/fc2/weights'] = _he(rng, (1024, 1024), 1024)
        w[q + '/fc2/biases'] = rng.normal(0, 0.05, size=1024).astype(np.float32)
        w[q + '/fc3/weights'] = _small_xavier(rng, (1024, d), 1024, d, 0.05)
        w[q + '/fc3/biases'] = rng.normal(0, 0.01, size=d).astype(np.float32)
    return w


def make_hal_weights(seed: int = 6, C: int = 2048, out: dict | None = None) -> dict:
    """fc2_res hallucinator (models.py:270-296)."""
    rng = np.random.RandomState(seed)
    w = {} if out is None else out
    for k in (1, 2):
        w['fc2_res/fc%d/weights' % k] = _he(rng, (C, C), C)
        w['fc2_res/fc%d/biases' % k] = rng.normal(0, 0.05, size=C).astype(np.float32)
    w['fc2_res/fc3/weights'] = _small_xavier(rng, (C, C), C, C, 0.3)
    w['fc2_res/fc3/biases'] = rng.normal(0, 0.05, size=C).astype(np.float32)
    return w


DPOSE_LAYERS = [('D_conv1', (1, 1, 9, 32)), ('D_conv2', (1, 1, 32, 32))] + \
    [('pose_out_j%d' % j, (32, 1)) for j in range(23)] + \
    [('D_alljoints_fc1', (736, 1024)), ('D_alljoints_fc2', (1024, 1024)), ('D_alljoints_out', (1024, 1))]


def make_dpose_weights(seed: int = 0, bias_scale: float = 0.0) -> dict:
    """D_pose variables (discriminators.py), in the order the reference creates them: slim's default initialisation, Xavier-uniform
    weights (fan_in = kh*kw*cin, fan_out = kh*kw*cout) and zero biases; bias_scale > 0 draws the biases from U(-bias_scale, bias_scale)
    instead, so tests exercise them."""
    rng = np.random.RandomState(seed)
    w = {}
    for name, shape in DPOSE_LAYERS:
        fan_in, fan_out = int(np.prod(shape[:-1])), int(np.prod(shape[:-2])) * shape[-1]
        limit = np.sqrt(6.0 / (fan_in + fan_out))
        w['D_pose/%s/weights' % name] = rng.uniform(-limit, limit, size=shape).astype(np.float32)
        b = rng.uniform(-bias_scale, bias_scale, size=shape[-1]) if bias_scale > 0 else np.zeros(shape[-1])
        w['D_pose/%s/biases' % name] = b.astype(np.float32)
    return w


def make_synthetic_weights(seed: int = 1, num_conv_layers: int = 3, delta_t_values=(-5, 5),
                           with_hal: bool = False) -> dict:
    """Full HMMR inference weight dict (TF variable names)."""
    w: dict = {}
    make_resnet_weights(seed, out=w)
    make_fmovie_weights(seed + 3, num_conv_layers, out=w)
    make_ief_weights(seed + 4, delta_t_values, out=w)
    if with_hal:
        make_hal_weights(seed + 5, out=w)
    w['mean_param'] = make_mean_param(seed + 2)
    return w


def make_images(n: int, seed: int = 0, size: int = 224) -> np.ndarray:
    """U(-1,1) NHWC float32 frames (run_video.py:73 scales crops to [-1,1])."""
    rng = np.random.RandomState(seed)
    return rng.uniform(-1.0, 1.0, size=(n, size, size, 3)).astype(np.float32)


def make_smpl_inputs(n: int, seed: int = 0, zero_pose: bool = False):
    """beta ~ N(0,1), theta ~ N(0,0.3) (SURVEY 8d); zero pose for config C1."""
    rng = np.random.RandomState(seed)
    beta = rng.normal(0, 1.0, size=(n, 10)).astype(np.float32)
    theta = np.zeros((n, 72), np.float32) if zero_pose else rng.normal(0, 0.3, size=(n, 72)).astype(np.float32)
    return beta, theta


def make_loss_inputs(obj, seed: int = 0, flip_frame: bool = True, dtype=np.float32) -> dict:
    """Seeded inputs of an objective.Objective (numpy, its `shapes()`): cameras with scale in [0.6, 1.4], keypoint visibility mixing
    0, 1 and 0.5, the has_3d patterns [joints, smpl] cycling through (1, 0), (0, 1), (0, 0), (1, 1), and, with `flip_frame`, one frame
    of the first delta set whose prediction is the label mirrored (its optimal scale falls to the 0.7 clip)."""
    from .objective import Objective
    assert isinstance(obj, Objective)
    rng = np.random.RandomState(seed)
    S, B, T, K = len(obj.sets), obj.B, obj.T, obj.K
    out = {}
    om = rng.normal(0, 0.3, size=(S, B, T, 85))
    om[..., 0] = rng.uniform(0.6, 1.4, size=(S, B, T))
    out['omega'] = om
    # labels move slowly in time and the predictions are scaled, shifted, noisy copies, so that the optimal cameras of every window
    # are mostly inside the scale clip
    lab = rng.normal(0, 0.5, size=(B, 1, K, 3)) + rng.normal(0, 0.05, size=(B, T, K, 3))
    js = rng.normal(0, 0.5, size=(S, B, T, K, 3))
    js[..., :2] = lab[None, ..., :2] / rng.uniform(0.8, 1.6, size=(S, B, T, 1, 1)) + rng.normal(0, 0.1, size=(S, B, T, K, 2))
    out['joints'] = js
    out['rots'] = rng.normal(0, 0.5, size=(S, B, T, 216))
    lab[..., 2] = rng.choice([0., 1., 1., 0.5], size=(B, T, K))
    out['labels'] = lab
    out['gt_rots'] = rng.normal(0, 0.5, size=(B, T, 216))
    out['gt_shape'] = rng.normal(0, 0.5, size=(B, 10))
    out['gt3ds'] = rng.normal(0, 0.5, size=(B, T, 14, 3))
    pat = np.array([[1, 0], [0, 1], [0, 0], [1, 1]], np.float64)
    has = pat[np.arange(B) % 4]
    out['w_joints'], out['w_smpl'] = has[:, 0].copy(), has[:, 1].copy()
    if 'strips' in obj.inputs:
        out['strips'] = rng.normal(0, 1, size=(B, T, 2048))
        out['pred_strips'] = out['strips'] + rng.normal(0, 0.3, size=(B, T, 2048))
    if flip_frame and obj.cam_terms:
        i, (group, dt) = obj.cam_terms[0]
        s = obj.sets.index((group, dt))
        t = obj.terms[i]
        pf, qf = t['p'][4], t['q'][4]
        out['labels'][0, qf, :, 2] = 1.
        out['joints'][s, 0, pf, :, 0] = -out['labels'][0, qf, :, 0]
        out['joints'][s, 0, pf, :, 1] = out['labels'][0, qf, :, 1]
    return {k: np.ascontiguousarray(v, dtype=dtype) for k, v in out.items()}
