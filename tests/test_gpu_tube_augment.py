"""GPU: hd_tube_augment (the reference's TubePreprocessor) against the float32 oracle (oracle/tube_ref.py) and the fixture made by
executing the reference's own source, a seeded sweep, the conv1-plane output, compute_augmented_phis, determinism, launches and
synchronisation, the walk generator, and an HMMRTrainer step fed from augmented phis."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import tube_ref

pytestmark = pytest.mark.gpu

CROP_TOL, LAB_TOL, POSE_TOL = 2e-6, 1e-6, 1e-5


def _tubes():
    return tube_ref.load_fixture(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'tube_aug_v1.npz'))


def _run(frames, labels, centers, poses, gt3ds, walks, S, trans_max, rotate, out='crops'):
    """One hd_tube_augment call on CUDA copies; -> dict of host arrays."""
    from human_dynamics_b200.augment import tube_augment
    from human_dynamics_b200.nets import PackedConv1Planes
    cu = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a)).to('cuda', dt).contiguous()
    fr = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    w = {k: v.cuda().contiguous() for k, v in walks.items() if k in ('trans', 'scale', 'rot', 'flip')}
    F = fr.shape[0]
    crops = torch.empty((F, S, S, 3), device='cuda') if out in ('crops', 'both') else None
    planes = None
    if out in ('planes', 'both'):
        sh = (F, S + 6, PackedConv1Planes.plane_width(S), 4)
        planes = (torch.zeros(sh, dtype=torch.float16, device='cuda'), torch.zeros(sh, dtype=torch.float16, device='cuda'))
    lab, cen, pos, g3, geom = tube_augment(fr, cu(labels, torch.float32), cu(centers, torch.int32), cu(poses, torch.float32),
                                           cu(gt3ds, torch.float32), w, S, trans_max, rotate, crops, planes)
    torch.cuda.synchronize()
    r = {'labels': lab.cpu().numpy(), 'centers': cen.cpu().numpy(), 'poses': pos.cpu().numpy(), 'gt3ds': g3.cpu().numpy(),
         'geom': geom[:, :6].cpu().numpy()}
    if crops is not None:
        r['images'] = crops.cpu().numpy()
    if planes is not None:
        r['planes'] = planes
        r['crops_dev'] = crops
    return r


def _compare(got, o):
    assert np.array_equal(got['geom'], o['geom'])
    assert np.array_equal(got['centers'], o['center'])
    assert np.abs(got['images'] - o['images']).max() <= CROP_TOL
    assert np.abs(got['labels'] - o['label']).max() <= LAB_TOL
    assert np.abs(got['gt3ds'] - o['gt3d']).max() <= LAB_TOL
    assert np.abs(got['poses'] - o['pose']).max() <= POSE_TOL


@pytest.mark.parametrize('i', [0, 1, 2])
def test_fixture(i):
    from human_dynamics_b200.augment import random_walks
    x, cfg, S, draws, ref = _tubes()[i]
    T = len(x['frames'])
    w = random_walks([T], cfg, draws=[draws])            # CPU: the sequential cumsum the reference's walk takes
    rotate = cfg['rotate_max'] != 0
    got = _run(x['frames'], x['labels'], x['centers'], x['poses'], x['gt3ds'], w, S, cfg['trans_max'], rotate)
    trans, scale, rot, flip = tube_ref.tube_walks(T, cfg, draws)
    o = tube_ref.augment_tube(x['frames'], x['labels'], x['centers'], x['poses'], x['gt3ds'], trans, scale, rot, flip, S,
                              cfg['trans_max'], rotate)
    _compare(got, o)
    assert np.abs(got['images'] - ref['images']).max() <= CROP_TOL
    assert np.array_equal(got['centers'], ref['centers'][..., 0])
    for k in ('labels', 'gt3ds'):
        assert np.abs(got[k] - ref[k]).max() <= LAB_TOL, k
    assert np.abs(got['poses'] - ref['poses']).max() <= POSE_TOL


SWEEP = [  # T, (H, W), S, uint8, rotate, flip, walk extremes
    (1, (300, 300), 224, True, False, False, 'max'),
    (20, (300, 300), 224, True, True, True, 'min'),
    (77, (240, 320), 64, False, False, True, 'rand'),
    (20, (240, 320), 224, False, True, False, 'max'),
    (77, (300, 300), 64, True, True, True, 'rand'),
    (1, (240, 320), 64, True, True, True, 'min'),
    (20, (240, 320), 224, True, False, True, 'rand'),
    (77, (300, 300), 224, False, False, False, 'min'),
]


def _inputs(T, H, W, u8, seed):
    rng = np.random.RandomState(seed)
    if u8:
        frames = rng.randint(0, 256, size=(T, H, W, 3)).astype(np.uint8)
    else:
        frames = rng.uniform(0, 1, size=(T, H, W, 3)).astype(np.float32)
    lab = np.stack([rng.uniform(0, W, (T, 25)), rng.uniform(0, H, (T, 25)), rng.choice([0., 1.], (T, 25))], 1).astype(np.float32)
    cen = np.stack([rng.randint(W // 4, 3 * W // 4, T), rng.randint(H // 4, 3 * H // 4, T)], 1).astype(np.int32)
    return frames, lab, cen, rng.normal(0, 0.4, (T, 72)).astype(np.float32), rng.normal(0, 0.4, (T, 14, 3)).astype(np.float32)


def _walks(T, extreme, flip, rotate, seed, tm=20, sm=0.3):
    rng = np.random.RandomState(seed)
    if extreme == 'rand':
        trans = rng.randint(-tm, tm + 2, (T, 2))
        scale = rng.uniform(-sm, sm, T)
    else:
        sgn = 1 if extreme == 'max' else -1
        trans = np.full((T, 2), sgn * tm)
        scale = np.full(T, sgn * sm)
    rot = rng.uniform(-0.6, 0.6, T) if rotate else np.zeros(T)
    return {'trans': torch.from_numpy(trans.astype(np.int32)), 'scale': torch.from_numpy(scale.astype(np.float32)),
            'rot': torch.from_numpy(rot.astype(np.float32)), 'flip': torch.full((T,), int(flip), dtype=torch.int32)}


@pytest.mark.parametrize('case', SWEEP, ids=[str(i) for i in range(len(SWEEP))])
def test_seeded_sweep(case):
    T, (H, W), S, u8, rotate, flip, extreme = case
    x = _inputs(T, H, W, u8, seed=T + H + S)
    w = _walks(T, extreme, flip, rotate, seed=T * 7 + S)
    got = _run(*x, w, S, 20, rotate)
    o = tube_ref.augment_tube(*x, w['trans'].numpy(), w['scale'].numpy(), w['rot'].numpy(), flip, S, 20, rotate)
    _compare(got, o)


@pytest.mark.parametrize('rotate', [False, True])
def test_planes_equal_packing_the_crops(rotate):
    from human_dynamics_b200._lib import lib, check, current_stream
    from human_dynamics_b200.nets import PackedConv1Planes
    T, S = 7, 224
    x = _inputs(T, 300, 300, True, seed=3)
    got = _run(*x, _walks(T, 'rand', True, rotate, seed=4), S, 20, rotate, out='both')
    crops = got['crops_dev']
    sh = (T, S + 6, PackedConv1Planes.plane_width(S), 4)
    hi, lo = torch.zeros(sh, dtype=torch.float16, device='cuda'), torch.zeros(sh, dtype=torch.float16, device='cuda')
    check(lib.hd_pack_conv1_planes(C.c_void_p(crops.data_ptr()), C.c_void_p(hi.data_ptr()), C.c_void_p(lo.data_ptr()), T, S, S,
                                   sh[2], current_stream()), 'hd_pack_conv1_planes')
    assert torch.equal(hi.view(torch.int16), got['planes'][0].view(torch.int16))
    assert torch.equal(lo.view(torch.int16), got['planes'][1].view(torch.int16))


def test_deterministic_across_repeats_permutations_and_splits():
    T, S = 24, 64
    x = _inputs(T, 240, 320, True, seed=9)
    w = _walks(T, 'rand', False, True, seed=10)
    w['flip'] = torch.from_numpy((np.arange(T) % 3 == 0).astype(np.int32))
    a = _run(*x, w, S, 20, True)
    b = _run(*x, w, S, 20, True)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    perm = np.random.RandomState(1).permutation(T)
    xp = [v[perm] for v in x]
    wp = {k: v[torch.from_numpy(perm)] for k, v in w.items()}
    c = _run(*xp, wp, S, 20, True)
    for k in a:
        assert np.array_equal(a[k][perm], c[k]), k
    parts = [_run(*[v[s] for v in x], {k: v[s] for k, v in w.items()}, S, 20, True) for s in (slice(0, 5), slice(5, 17), slice(17, T))]
    for k in a:
        assert np.array_equal(a[k], np.concatenate([p[k] for p in parts])), k


def test_two_launches_and_no_host_sync():
    from human_dynamics_b200._lib import lib
    from human_dynamics_b200.augment import TubeAugmentor
    aug = TubeAugmentor(img_size=64, rotate_max=0.3, delta_rotate_max=0.1, seed=3)
    x = [torch.as_tensor(v).cuda() for v in _inputs(40, 120, 160, True, seed=2)]
    aug(*x, out='both', tube_lengths=[10, 30])               # warm up (allocator, module load)
    torch.cuda.synchronize()
    n0 = lib.hd_launch_count()
    torch.cuda.set_sync_debug_mode('error')
    try:
        r = aug(*x, out='both', tube_lengths=[10, 30])
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert lib.hd_launch_count() - n0 == 2
    assert r['images'].shape == (40, 64, 64, 3) and r['labels'].shape == (40, 3, 25)


CFGS = [dict(trans_max=20, delta_trans_max=20, scale_max=0.3, delta_scale_max=0.3, rotate_max=0, delta_rotate_max=0),
        dict(trans_max=20, delta_trans_max=3, scale_max=0.3, delta_scale_max=0.05, rotate_max=0.5, delta_rotate_max=0.1),
        dict(trans_max=5, delta_trans_max=2, scale_max=0.1, delta_scale_max=0.1, rotate_max=0.2, delta_rotate_max=0.05)]


@pytest.mark.parametrize('cfg', CFGS, ids=['iid', 'walk', 'mixed'])
def test_walk_generator(cfg):
    from human_dynamics_b200.augment import random_walks, _walk_kind
    lens = [5, 50, 17]
    g1, g2 = torch.Generator(device='cuda'), torch.Generator(device='cuda')
    g1.manual_seed(11)
    g2.manual_seed(11)
    a, b = random_walks(lens, cfg, g1), random_walks(lens, cfg, g2)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    tm, dtm = cfg['trans_max'], cfg['delta_trans_max']
    tr, sc, ro = a['trans'].cpu().numpy(), a['scale'].cpu().numpy(), a['rot'].cpu().numpy()
    assert tr.dtype == np.int32 and sc.dtype == np.float32 and tr.shape == (72, 2) and sc.shape == (72,)
    assert (tr >= -tm).all() and (tr <= tm + 1).all()        # the walk branch can land on its exclusive upper wall
    eps = 1e-6
    assert (sc >= -cfg['scale_max'] - eps).all() and (sc <= cfg['scale_max'] + eps).all()
    assert (np.abs(ro) <= cfg['rotate_max'] + eps).all()
    kinds = {'trans': _walk_kind(-tm, tm + 1, -dtm, dtm + 1),
             'scale': _walk_kind(-cfg['scale_max'], cfg['scale_max'], -cfg['delta_scale_max'], cfg['delta_scale_max']),
             'rot': _walk_kind(-cfg['rotate_max'], cfg['rotate_max'], -cfg['delta_rotate_max'], cfg['delta_rotate_max'])}
    for name, ref_args in (('trans', (-tm, tm + 1, -dtm, dtm + 1)),
                           ('scale', (-cfg['scale_max'], cfg['scale_max'], -cfg['delta_scale_max'], cfg['delta_scale_max'])),
                           ('rot', (-cfg['rotate_max'], cfg['rotate_max'], -cfg['delta_rotate_max'], cfg['delta_rotate_max']))):
        assert kinds[name] == tube_ref.walk_branch(*ref_args), name
    fl = a['flip'].cpu().numpy()
    o = 0
    for i, T in enumerate(lens):
        seg = slice(o, o + T)
        assert (fl[seg] == int(a['tube_flip'][i])).all()
        if kinds['trans'] == 'walk':
            assert (np.abs(np.diff(tr[seg], axis=0)) <= dtm).all()
        if kinds['scale'] == 'walk':
            assert (np.abs(np.diff(sc[seg])) <= cfg['delta_scale_max'] + eps).all()
        if kinds['rot'] == 'walk':
            assert (np.abs(np.diff(ro[seg])) <= cfg['delta_rotate_max'] + eps).all()
        o += T
    if kinds['trans'] == 'iid':                                  # i.i.d. steps are not bounded by a small delta
        assert np.abs(np.diff(tr, axis=0)).max() > 3


def test_walk_draws_on_device_match_cpu():
    """The walk formula on the device from given draws equals the CPU one (integers exactly; floats within rounding of the
    cumulative sum's order)."""
    from human_dynamics_b200.augment import random_walks
    for x, cfg, S, draws, ref in _tubes():
        T = len(x['frames'])
        d = random_walks([T], cfg, draws=[draws], device='cuda')
        assert np.array_equal(d['trans'].cpu().numpy(), ref['trans_walk'])
        assert np.abs(d['scale'].cpu().numpy() - ref['scale_walk'][:, 0]).max() < 1e-6


def test_compute_augmented_phis_equals_compute_all_phis(weights):
    from src.datasets.resnet_extractor import FeatureExtractor
    from human_dynamics_b200.augment import TubeAugmentor
    S, bs, T = 64, 4, 9
    fx = FeatureExtractor(weights, img_size=S, batch_size=bs)
    frames, lab, cen, pose, g3 = _inputs(T, 120, 100, True, seed=5)
    sizes = np.tile([[120, 100]], (T, 1))
    aug = TubeAugmentor(img_size=S, rotate_max=0.4, delta_rotate_max=0.1, seed=21)
    r = fx.compute_augmented_phis(frames, sizes, lab, cen, pose, g3, aug, keep_images=True)
    ref = fx.compute_all_phis(r['images'].cpu().numpy())
    assert np.array_equal(r['phis'].cpu().numpy(), ref)
    aug2 = TubeAugmentor(img_size=S, rotate_max=0.4, delta_rotate_max=0.1, seed=21)
    r2 = fx.compute_augmented_phis(frames, sizes, lab, cen, pose, g3, aug2)
    assert 'images' not in r2
    assert torch.equal(r2['phis'], r['phis']) and torch.equal(r2['labels'], r['labels'])
    with pytest.raises(ValueError):
        fx.compute_augmented_phis(frames, sizes + 1, lab, cen, pose, g3, aug)


def test_drop_in_driver_shapes_and_checks():
    from src.util.tube_augmentation import TubePreprocessorDriver
    T = 6
    frames, lab, cen, pose, g3 = _inputs(T, 90, 110, True, seed=8)
    drv = TubePreprocessorDriver(img_size=64, seed=1)
    r = drv(frames / 255., np.tile([[90, 110]], (T, 1)), lab.transpose(0, 2, 1), cen, pose, g3)
    assert r['images'].shape == (T, 64, 64, 3) and r['labels'].shape == (T, 3, 25) and r['centers'].shape == (T, 2, 1)
    assert r['trans_walk'].shape == (T, 2) and r['scale_walk'].shape == (T, 1) and r['rot_walk'].shape == (T, 1)
    assert np.abs(r['images']).max() <= 1.0
    with pytest.raises(ValueError):
        drv(frames, np.tile([[100, 110]], (T, 1)), lab, cen, pose, g3)
    with pytest.raises(ValueError):
        drv(frames, np.tile([[90, 110]], (T, 1)), lab, cen + 200, pose, g3)


def test_trainer_step_from_augmented_phis(weights, smpl_model):
    """Two augmented tubes through compute_augmented_phis, labels transposed to the loader's T x K x 3, one HMMRTrainer step; the
    same step fed from the fp32-crop path (compute_all_phis) gives the same losses bit for bit."""
    from src.datasets.resnet_extractor import FeatureExtractor
    from src.tf_smpl.batch_smpl import SMPL
    from human_dynamics_b200.augment import TubeAugmentor
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    B, T, S = 2, 10, 64
    fx = FeatureExtractor(weights, img_size=S, batch_size=8)
    smpl = SMPL(smpl_model)
    tubes = []
    for b in range(B):
        frames, lab, cen, pose, g3 = _inputs(T, 96, 128, True, seed=30 + b)
        r = fx.compute_augmented_phis(frames, np.tile([[96, 128]], (T, 1)), lab, cen, pose, g3,
                                      TubeAugmentor(img_size=S, seed=40 + b), keep_images=True)
        r['phis_crops'] = torch.from_numpy(fx.compute_all_phis(r['images'].cpu().numpy())).cuda()
        r['shape'] = torch.zeros(10, device='cuda')
        tubes.append(r)

    def batch(key):
        return {'phis': torch.stack([t[key] for t in tubes]), 'labels': torch.stack([t['labels'].transpose(1, 2) for t in tubes]).contiguous(),
                'poses': torch.stack([t['poses'] for t in tubes]), 'shape': torch.stack([t['shape'] for t in tubes]),
                'gt3ds': torch.stack([t['gt3ds'] for t in tubes]), 'has_3d': torch.ones((B, 2), device='cuda')}
    from human_dynamics_b200.smpl import batch_rodrigues
    outs = []
    for key in ('phis', 'phis_crops'):
        tr = HMMRTrainer(TrainConfig(), weights, smpl)
        n = tr.n_fake(B, T)
        mocap = batch_rodrigues(torch.from_numpy(np.random.RandomState(3).normal(0, 0.3, (n * 24, 3)).astype(np.float32)).cuda())
        outs.append(tr.step(batch(key), mocap.reshape(n, 216)))
    a, b = outs
    assert all(torch.isfinite(v).all() for v in a.values())
    for k in a:
        assert torch.equal(a[k], b[k]), k
