"""Times the training-time tube augmentation (hd_tube_augment, human_dynamics_b200/augment.py) on the GPU and prints one JSON line.

Workload: --batches batches of 64 frames (one FeatureExtractor plan's batch) of 300 x 300 uint8 frames, S = 224, the converters'
augmentation (trans 20 / 20, scale 0.3 / 0.3, no rotation) and, separately, with rotation (rotate_max 0.3 / 0.1).  Per batch:
  aug_planes:  hd_tube_augment writing conv1's fp16 input planes;
  aug_crops:   hd_tube_augment writing fp32 NHWC crops;
  aug_phi:     augment into the planes + the ResNet-50 trunk (what compute_augmented_phis runs per batch);
  phi_crops:   the trunk on the same crops made beforehand, device-resident (pack + trunk: compute_all_phis' device work);
  compute_all_phis: the public call on host crops (upload included), per batch.
The four device timings are CUDA-event medians over --rounds rounds in which the variants alternate.  The CPU alternative a user
has today, the float32 oracle (oracle/tube_ref.py) per frame, is timed on --cpu-frames frames.  The card's name, power limit and
max SM clock are read (never set) in the same run; bytes are what the pixel kernel must move per frame (source taps read once,
planes or crops written), from shapes.

    python tools/bench_tube_augment.py [--batches 8] [--rounds 7] [--cpu-frames 8]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_smpl_grad import card          # noqa: E402

BS, S, H, W = 64, 224, 300, 300


def events(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, default=8)
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--cpu-frames', type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_tube_augment needs a CUDA device')
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.augment import TubeAugmentor, tube_augment
    from src.datasets.resnet_extractor import FeatureExtractor
    from oracle import tube_ref
    torch.cuda.set_device(0)
    n = a.batches * BS
    rng = np.random.RandomState(0)
    frames = torch.from_numpy(rng.randint(0, 256, size=(n, H, W, 3)).astype(np.uint8)).cuda()
    lab = np.stack([rng.uniform(0, W, (n, 25)), rng.uniform(0, H, (n, 25)), np.ones((n, 25))], 1).astype(np.float32)
    cen = np.stack([rng.randint(100, 200, n), rng.randint(100, 200, n)], 1).astype(np.int32)
    pose = rng.normal(0, 0.3, (n, 72)).astype(np.float32)
    g3 = rng.normal(0, 0.3, (n, 14, 3)).astype(np.float32)
    fx = FeatureExtractor(synthetic.make_synthetic_weights(seed=1), img_size=S, batch_size=BS)
    planes = fx.plan.planes
    if planes is None:
        raise SystemExit('the plan has no conv1 planes (non tensor-core build)')
    res = {'tool': 'bench_tube_augment', **card(), 'frames': n, 'batch': BS, 'source': [H, W], 'S': S, 'rounds': a.rounds, 'configs': {}}
    for name, kw in (('converters', dict(trans_max=20, delta_trans_max=20, scale_max=0.3, delta_scale_max=0.3)),
                     ('rotate', dict(rotate_max=0.3, delta_rotate_max=0.1))):
        aug = TubeAugmentor(img_size=S, seed=1, **kw)
        fr, lb, ce, po, gg = aug.prepare(frames, lab, cen, pose, g3)
        walks = aug.walks([n])
        crops = torch.empty((n, S, S, 3), device='cuda')
        outs = [dict(labels_out=torch.empty((BS, 3, 25), device='cuda'), centers_out=torch.empty((BS, 2), dtype=torch.int32, device='cuda'),
                     poses_out=torch.empty((BS, 72), device='cuda'), gt3ds_out=torch.empty((BS, 14, 3), device='cuda'),
                     geom=torch.empty((BS, 16), dtype=torch.int32, device='cuda'))]

        def call(b, crops_out, planes_out):
            sl = slice(b * BS, (b + 1) * BS)
            tube_augment(fr[sl], lb[sl], ce[sl], po[sl], gg[sl], {k: walks[k][sl] for k in ('trans', 'scale', 'rot', 'flip')}, S,
                         aug.trans_max, aug.rotate, crops_out, planes_out, **outs[0])

        def aug_planes():
            for b in range(a.batches):
                call(b, None, planes)

        def aug_crops():
            for b in range(a.batches):
                call(b, crops[b * BS:(b + 1) * BS], None)

        def aug_phi():
            for b in range(a.batches):
                call(b, None, planes)
                fx.plan.run(None, fx.phis)

        def phi_crops():
            for b in range(a.batches):
                fx.plan.run(crops[b * BS:(b + 1) * BS], fx.phis)
        variants = {'aug_planes': aug_planes, 'aug_crops': aug_crops, 'aug_phi': aug_phi, 'phi_crops': phi_crops}
        for fn in variants.values():          # warm-up of every shape the timed window uses
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in variants}
        for _ in range(a.rounds):
            for k, fn in variants.items():
                ms[k].append(events(fn))
        host_crops = crops.cpu().numpy()
        t0 = time.perf_counter()
        fx.compute_all_phis(host_crops)
        t_all = (time.perf_counter() - t0) * 1e3
        r = {}
        for k, v in ms.items():
            med = statistics.median(v)
            r[k] = {'ms_per_batch': round(med / a.batches, 4), 'frames_per_s': round(n / med * 1e3, 1),
                    'spread_ms_per_batch': [round(min(v) / a.batches, 4), round(max(v) / a.batches, 4)]}
        r['compute_all_phis_host'] = {'ms_per_batch': round(t_all / a.batches, 3), 'frames_per_s': round(n / t_all * 1e3, 1)}
        r['aug_share_of_aug_phi'] = round(r['aug_planes']['ms_per_batch'] / r['aug_phi']['ms_per_batch'], 4)
        # bytes the pixel kernel must move per frame: the source taps (at most the whole frame, once) and the outputs
        src_b = min(H * W, S * S * 4) * 3
        r['bytes_per_frame'] = {'source_read_max': src_b, 'planes_written': 2 * S * S * 8, 'crops_written': S * S * 12}
        r['aug_planes_achieved_GBps'] = round((src_b + 2 * S * S * 8) * n / (statistics.median(ms['aug_planes']) * 1e-3) / 1e9, 1)
        # CPU alternative: the float32 oracle per frame
        cfr = fr[:a.cpu_frames].cpu().numpy()
        w = {k: v[:a.cpu_frames].cpu().numpy() for k, v in walks.items() if k != 'tube_flip'}
        t0 = time.perf_counter()
        for i in range(a.cpu_frames):
            tube_ref.preprocess_frame((cfr[i] / 255.).astype(np.float32), lab[i], cen[i], pose[i], g3[i], w['trans'][i], w['scale'][i],
                                      w['rot'][i], bool(w['flip'][i]), S, aug.trans_max, aug.rotate)
        cpu_ms = (time.perf_counter() - t0) * 1e3 / a.cpu_frames
        r['cpu_oracle'] = {'ms_per_frame': round(cpu_ms, 2), 'frames_per_s': round(1e3 / cpu_ms, 1)}
        res['configs'][name] = r
    print(json.dumps(res))


if __name__ == '__main__':
    main()
