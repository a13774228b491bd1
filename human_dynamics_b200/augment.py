"""Training-time tube augmentation on the GPU: TubePreprocessor (src/util/tube_augmentation.py of the reference) as two CUDA launches.

The reference jitters every frame of a video tube before the frozen trunk turns it into phis (the tfrecord converters'
TubePreprocessorDriver, then FeatureExtractor.compute_all_phis).  Here the walks are drawn with torch on the device
(`random_walks`) and `hd_tube_augment` writes each frame's geometry and labels (one thread per frame) and the S x S crop straight
from the source frame (one thread per pixel), either as fp32 NHWC in [-1, 1] or directly as the tensor-core conv1's input planes.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import lib, check, current_stream
from .nets import PackedConv1Planes

GEOM_WORDS = 16                 # hd_tube_aug_args.geom row: {Hs, Ws, cx, cy, x0, y0, flip, 0}, then float bits
NUM_KPS_FLIP = 25               # flip_image's name lists


def _walk_kind(lo, hi, dlo, dhi):
    """bounded_random_walk's branches (data_utils.py:808-821): 'zeros' when max <= min, the 'old data augmentation' ('iid')
    when the walk's bounds equal its step's bounds, else 'walk'."""
    if hi <= lo:
        return 'zeros'
    if lo == dlo and hi == dhi:
        return 'iid'
    return 'walk'


def _uniform(u, lo, hi, is_int):
    """tf.random_uniform from draws u in [0, 1): float32 u * (max - min) + min; int32 min + floor(u * (max - min)) (in float64,
    clamped below max)."""
    if is_int:
        r = int(hi) - int(lo)
        return (int(lo) + torch.clamp(torch.floor(u.double() * r), max=r - 1)).to(torch.int32)
    lo32, hi32 = np.float32(lo), np.float32(hi)
    return u.float() * float(hi32 - lo32) + float(lo32)


def _bounded_walk(lo, hi, dlo, dhi, is_int, start_u, delta_u):
    """data_utils.bounded_random_walk over the second-to-last axis of delta_u ([..., T, dim]); start_u [..., 1, dim]."""
    kind = _walk_kind(lo, hi, dlo, dhi)
    if kind == 'zeros':
        return torch.full(delta_u.shape, float(np.float32(lo)), dtype=torch.float32, device=delta_u.device)
    if kind == 'iid':
        return _uniform(delta_u, lo, hi, is_int)
    start = _uniform(start_u, lo, hi, is_int)
    walk = torch.cumsum(_uniform(delta_u, dlo, dhi, is_int), dim=-2, dtype=torch.int32 if is_int else torch.float32)
    size = hi - lo
    if is_int:
        x = ((walk + start) - int(lo)) + int(size)
        return (torch.abs(torch.remainder(x, 2 * int(size)) - int(size)) + int(lo)).to(torch.int32)
    f = lambda v: float(np.float32(v))
    x = ((walk + start) - f(lo)) + f(size)
    y = f(2 * size)
    r = torch.fmod(x, y)
    r = torch.where(x < 0, torch.fmod(r + y, y), r)          # TF's floormod on floats (google_floor_fmod), y > 0
    return torch.abs(r - f(size)) + f(lo)


def _walk_specs(cfg):
    tm, dtm = int(cfg['trans_max']), int(cfg['delta_trans_max'])
    return (('trans', -tm, tm + 1, -dtm, dtm + 1, True, 2),
            ('scale', -cfg['scale_max'], cfg['scale_max'], -cfg['delta_scale_max'], cfg['delta_scale_max'], False, 1),
            ('rot', -cfg['rotate_max'], cfg['rotate_max'], -cfg['delta_rotate_max'], cfg['delta_rotate_max'], False, 1))


def random_walks(F_per_tube, cfg, generator=None, draws=None, device=None):
    """Per-frame walks for tubes of F_per_tube[i] frames, as TubePreprocessor.__call__ draws them (tube_augmentation.py:56-85):
    `trans` int32 [F,2] from bounded_random_walk(-trans_max, trans_max + 1, -delta_trans_max, delta_trans_max + 1), `scale` and
    `rot` float32 [F] likewise, `flip` int32 [F] constant within a tube (u < 0.5), and `tube_flip` bool [n_tubes].

    cfg: a dict (or object) with trans_max, delta_trans_max, scale_max, delta_scale_max, rotate_max, delta_rotate_max.
    The draws come from `generator` (a torch.Generator; its device is the walks' device) and never leave the device.  TensorFlow's
    random stream is not reproduced: seeded runs are reproducible here, not equal to the reference's.  `draws` replaces the
    generator with given uniforms in [0, 1), one dict per tube with keys flip_u (), trans_start_u (1,2), trans_u (T,2),
    scale_start_u / scale_u, rot_start_u / rot_u (the *_start_u only in the walk branch), so the walk formula can be checked on
    known inputs.  Note the reference's walk branch reaches max (= trans_max + 1 for the translation) where the reflected value
    lands exactly on the upper wall."""
    if not isinstance(cfg, dict):
        cfg = {k: getattr(cfg, k) for k in ('trans_max', 'delta_trans_max', 'scale_max', 'delta_scale_max', 'rotate_max',
                                             'delta_rotate_max')}
    lens = [int(t) for t in F_per_tube]
    if not lens or min(lens) <= 0:
        raise ValueError('random_walks: every tube needs at least one frame')
    specs = _walk_specs(cfg)
    out = {}
    if draws is not None:
        if len(draws) != len(lens):
            raise ValueError('random_walks: one draws dict per tube')
        dev = torch.device(device) if device is not None else torch.device('cpu')
        t = lambda v: torch.as_tensor(np.asarray(v, np.float32), device=dev)
        per = {name: [] for name, *_ in specs}
        flips = []
        for T, d in zip(lens, draws):
            flips.append(t(d['flip_u']).reshape(()) < 0.5)
            for name, lo, hi, dlo, dhi, is_int, dim in specs:
                kind = _walk_kind(lo, hi, dlo, dhi)
                du = t(d[name + '_u']) if kind != 'zeros' else torch.zeros((T, dim), device=dev)
                su = t(d[name + '_start_u']) if kind == 'walk' else None
                per[name].append(_bounded_walk(lo, hi, dlo, dhi, is_int, su, du.reshape(T, dim)))
        for name in per:
            out[name] = torch.cat(per[name], 0)
        tube_flip = torch.stack(flips)
    else:
        if generator is None:
            raise ValueError('random_walks: pass a torch.Generator (or draws)')
        dev = generator.device
        n, Tm = len(lens), max(lens)
        rand = lambda *shape: torch.rand(shape, generator=generator, device=dev)
        tube_flip = rand(n) < 0.5
        for name, lo, hi, dlo, dhi, is_int, dim in specs:
            w = _bounded_walk(lo, hi, dlo, dhi, is_int, rand(n, 1, dim), rand(n, Tm, dim))
            out[name] = w.reshape(n * Tm, dim) if all(T == Tm for T in lens) else torch.cat([w[i, :T] for i, T in enumerate(lens)], 0)
    out['scale'] = out['scale'].reshape(-1).float().contiguous()
    out['rot'] = out['rot'].reshape(-1).float().contiguous()
    out['trans'] = out['trans'].to(torch.int32).contiguous()
    out['flip'] = torch.cat([tube_flip[i:i + 1].expand(T) for i, T in enumerate(lens)]).to(torch.int32)
    out['tube_flip'] = tube_flip
    return out


def tube_augment(frames, labels, centers, poses, gt3ds, walks, img_size, trans_max, rotate, crops=None, planes=None,
                 labels_out=None, centers_out=None, poses_out=None, gt3ds_out=None, geom=None):
    """One hd_tube_augment call over F frames (CUDA tensors, contiguous): frames uint8 or float32 [F,H,W,3]; labels float32
    [F,3,K]; centers int32 [F,2]; poses [F,72]; gt3ds [F,14,3]; walks from random_walks (trans, scale, rot, flip for these
    frames).  Writes crops (float32 [F,S,S,3]) and / or planes ((hi, lo) fp16 [F,S+6,WP,4], the plan's conv1 input) and the label
    outputs, allocating the ones not given.  Returns (labels, centers, poses, gt3ds, geom)."""
    F, H, W = frames.shape[0], frames.shape[1], frames.shape[2]
    K = labels.shape[2]
    dev = frames.device
    if frames.dtype not in (torch.uint8, torch.float32) or frames.dim() != 4 or frames.shape[3] != 3:
        raise _lib.HDError('tube_augment: frames must be (F,H,W,3) uint8 or float32')
    want = {'labels': (labels, (F, 3, K), torch.float32), 'centers': (centers, (F, 2), torch.int32),
            'poses': (poses, (F, 72), torch.float32), 'gt3ds': (gt3ds, (F, 14, 3), torch.float32),
            'trans': (walks['trans'], (F, 2), torch.int32), 'scale': (walks['scale'], (F,), torch.float32),
            'rot': (walks['rot'], (F,), torch.float32), 'flip': (walks['flip'], (F,), torch.int32)}
    for name, (t, shape, dt) in want.items():
        if tuple(t.shape) != shape or t.dtype != dt or not t.is_contiguous() or t.device != dev:
            raise _lib.HDError('tube_augment: %s must be a contiguous %s %s tensor on %s' % (name, dt, shape, dev))
    new = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)
    labels_out = new((F, 3, K), torch.float32) if labels_out is None else labels_out
    centers_out = new((F, 2), torch.int32) if centers_out is None else centers_out
    poses_out = new((F, 72), torch.float32) if poses_out is None else poses_out
    gt3ds_out = new((F, 14, 3), torch.float32) if gt3ds_out is None else gt3ds_out
    geom = new((F, GEOM_WORDS), torch.int32) if geom is None else geom
    # the flips are per-tube draws that stay on the device, so a call must be able to flip: K = 25 (flip_image's names)
    flags = _lib.HD_AUG_FLIP | (_lib.HD_AUG_SRC_U8 if frames.dtype == torch.uint8 else 0) | (_lib.HD_AUG_ROTATE if rotate else 0)
    if K != NUM_KPS_FLIP:
        raise _lib.HDError('tube_augment: flip_image swaps %d keypoints, labels have %d' % (NUM_KPS_FLIP, K))
    a = _lib.TubeAugArgs()
    a.frames, a.F, a.H, a.W, a.flags = frames.data_ptr(), F, H, W, flags
    a.trans, a.scale, a.rot, a.flip = (walks['trans'].data_ptr(), walks['scale'].data_ptr(), walks['rot'].data_ptr(),
                                       walks['flip'].data_ptr())
    a.labels, a.K, a.centers, a.poses, a.gt3ds = labels.data_ptr(), K, centers.data_ptr(), poses.data_ptr(), gt3ds.data_ptr()
    a.S, a.trans_max, a.geom = img_size, int(trans_max), geom.data_ptr()
    a.labels_out, a.centers_out = labels_out.data_ptr(), centers_out.data_ptr()
    a.poses_out, a.gt3ds_out = poses_out.data_ptr(), gt3ds_out.data_ptr()
    a.crops = crops.data_ptr() if crops is not None else None
    if planes is not None:
        if planes[1] is None:                 # hd_tube_augment writes both planes: a training-data path, FP32-class input
            raise _lib.HDError("tube_augment: conv1 planes without a remainder (impl 'tc1h') are not a training input; use impl 'auto'")
        a.plane_hi, a.plane_lo, a.WP = planes[0].data_ptr(), planes[1].data_ptr(), planes[0].shape[2]
    check(lib.hd_tube_augment(C.byref(a), current_stream()), 'hd_tube_augment')
    return labels_out, centers_out, poses_out, gt3ds_out, geom


class TubeAugmentor(object):
    """TubePreprocessor (tube_augmentation.py:11-186) on the GPU, with the reference's constructor arguments.

    Calling it with (frames [F,H,W,3] uint8 or float32 in [0,1], labels [F,3,K], centers [F,2] (x, y) inside the frame, poses
    [F,72], gt3ds [F,14,3]) returns device tensors under the reference's keys: images ([F,S,S,3] float32 in [-1,1]; with
    out='planes' or 'both' also `planes`, conv1's fp16 input), labels [F,3,K], poses, gt3ds, centers [F,2] (int32), trans_walk
    [F,2], scale_walk [F,1], rot_walk [F,1], plus `geometry` (int32 [F,6]: Hs, Ws, cx, cy, x0, y0).  The frames form one tube
    unless tube_lengths splits them; walks (random_walks' dict) may be given, else they are drawn from the augmentor's generator.
    Labels need the 25 keypoints flip_image swaps (K = 25): the reference fails on a flipped tube with another K, and the flips
    are drawn on the device, so every call must be able to flip."""

    def __init__(self, img_size=224, trans_max=20, delta_trans_max=3, scale_max=0.3, delta_scale_max=0.05, rotate_max=0,
                 delta_rotate_max=0, seed=None, device=None):
        if img_size % 2:
            raise ValueError('img_size must be even')
        self.img_size = int(img_size)
        self.trans_max, self.delta_trans_max = int(trans_max), int(delta_trans_max)
        self.scale_max, self.delta_scale_max = scale_max, delta_scale_max
        self.rotate_max, self.delta_rotate_max = rotate_max, delta_rotate_max
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        self.generator = torch.Generator(device=self.device)
        if seed is not None:
            self.generator.manual_seed(int(seed))
        else:
            self.generator.seed()

    @property
    def config(self):
        return {k: getattr(self, k) for k in ('trans_max', 'delta_trans_max', 'scale_max', 'delta_scale_max', 'rotate_max',
                                              'delta_rotate_max')}

    @property
    def rotate(self):
        return self.rotate_max != 0          # tube_augmentation.py:157, a static switch

    def walks(self, tube_lengths):
        return random_walks(tube_lengths, self.config, generator=self.generator)

    def prepare(self, frames, labels, centers, poses, gt3ds):
        """Inputs as contiguous CUDA tensors of the dtypes hd_tube_augment takes (numpy / host tensors are uploaded); labels given
        as [F,K,3] are transposed to [F,3,K] as TubePreprocessorDriver does for [...,3]-last labels."""
        dev = self.device
        up = lambda x, dt: torch.as_tensor(x).to(device=dev, dtype=dt).contiguous()
        if not (isinstance(centers, torch.Tensor) and centers.is_cuda):
            # the reference's tf.slice fails for a centre outside the frame; the kernel would clamp, so refuse here (centres
            # already on the device are not checked: that would synchronise)
            c = np.asarray(centers.cpu() if isinstance(centers, torch.Tensor) else centers).reshape(-1, 2)
            H, W = frames.shape[1], frames.shape[2]
            if (c < 0).any() or (c[:, 0] >= W).any() or (c[:, 1] >= H).any():
                raise ValueError('TubeAugmentor: a centre lies outside the %dx%d frame' % (H, W))
        if not isinstance(frames, torch.Tensor):
            frames = torch.from_numpy(np.ascontiguousarray(frames))
        if frames.dtype not in (torch.uint8, torch.float32):
            frames = frames.float()
        frames = frames.to(dev).contiguous()
        labels = up(labels, torch.float32)
        if labels.dim() == 3 and labels.shape[-1] == 3 and labels.shape[1] != 3:
            labels = labels.transpose(1, 2).contiguous()
        return (frames, labels, up(centers, torch.int32).reshape(-1, 2).contiguous(), up(poses, torch.float32).reshape(-1, 72),
                up(gt3ds, torch.float32).reshape(-1, 14, 3))

    def __call__(self, frames, labels, centers, poses, gt3ds, walks=None, out='crops', tube_lengths=None):
        if out not in ('crops', 'planes', 'both'):
            raise ValueError("out must be 'crops', 'planes' or 'both'")
        frames, labels, centers, poses, gt3ds = self.prepare(frames, labels, centers, poses, gt3ds)
        F, S = frames.shape[0], self.img_size
        if walks is None:
            walks = self.walks(tube_lengths if tube_lengths is not None else [F])
        crops = torch.empty((F, S, S, 3), dtype=torch.float32, device=self.device) if out in ('crops', 'both') else None
        planes = None
        if out in ('planes', 'both'):
            shape = (F, S + 6, PackedConv1Planes.plane_width(S), 4)
            planes = (torch.zeros(shape, dtype=torch.float16, device=self.device), torch.zeros(shape, dtype=torch.float16, device=self.device))
        lab, cen, pos, g3, geom = tube_augment(frames, labels, centers, poses, gt3ds, walks, S, self.trans_max, self.rotate, crops, planes)
        res = {'labels': lab, 'poses': pos, 'gt3ds': g3, 'centers': cen, 'trans_walk': walks['trans'],
               'scale_walk': walks['scale'].reshape(-1, 1), 'rot_walk': walks['rot'].reshape(-1, 1), 'geometry': geom[:, :6]}
        if crops is not None:
            res['images'] = crops
        if planes is not None:
            res['planes'] = planes
        return res
