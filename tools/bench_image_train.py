"""Times the training-mode ResNet (nets.ResNetTrainPlan, batch statistics) and an image-input HMMRTrainer step on the GPU; prints one
JSON line.

  trunk_train_ms / trunk_infer_ms   the whole trunk at 224 x 224 over n frames (n = 160 and 640 by default), training mode against the
                                    inference ResNetPlan over the same n, alternated in one run (CUDA events, --iters per round, --rounds
                                    rounds, medians)
  stats_ms                          the 98 hd_bn_batch_stats kernels of one training-mode pass (bn_partial_kernel + bn_finish_kernel),
                                    from a separate torch.profiler run, against hbm_floor_ms: the 49 normalised maps read once at the
                                    data-sheet 3.35 TB/s (counted from shapes here)
  step_images_ms / step_phis_ms     HMMRTrainer.step at B = 8, T = 20 with do_train.sh's flags (do_hallucinate, do_hallucinate_preds,
                                    delta_t = +-5), from 224 x 224 images (precomputed_phi=False) and from phis
The card's name, power limit and max SM clock are read in the same run.  Synthetic weights and seeded data.

    python tools/bench_image_train.py [--n 160 640] [--iters 5] [--rounds 3]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_smpl_grad import card, time_call          # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def trunk(w, n, iters, rounds):
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.nets import PackedResNet, ResNetBatchNorm, ResNetPlan, ResNetTrainPlan
    packed = PackedResNet(w, 'cuda', tc='auto')
    bn = ResNetBatchNorm(w, 'cuda')
    img = torch.from_numpy(synthetic.make_images(8, seed=1, size=224)).cuda().repeat(n // 8 + 1, 1, 1, 1)[:n].contiguous()
    out = torch.empty((n, 2048), device='cuda')
    tp = ResNetTrainPlan(packed, bn, n, 224)
    tt, ti = [], []
    ip = ResNetPlan(packed, n, 224, 'auto')
    for _ in range(rounds):
        tt.append(time_call(lambda: tp.run(img, out), iters, 1))
        ti.append(time_call(lambda: ip.run(img, out), iters, 1))
    del ip
    from torch.profiler import profile, ProfilerActivity
    tp.run(img, out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tp.run(img, out)
        torch.cuda.synchronize()
    stats_us = sum(e.self_device_time_total for e in prof.key_averages() if 'bn_partial_kernel' in e.key or 'bn_finish_kernel' in e.key)
    nbytes = sum(op.rows * op.C * 4 for op in tp.stats)
    return {'n': n, 'trunk_train_ms': float(np.median(tt)), 'trunk_infer_ms': float(np.median(ti)),
            'trunk_train_runs_ms': tt, 'trunk_infer_runs_ms': ti, 'stats_ms': round(stats_us / 1e3, 4),
            'stats_gb_read': round(nbytes / 1e9, 3), 'hbm_floor_ms': round(nbytes / HBM_BYTES_PER_S * 1e3, 4)}


def steps(w, smpl_model, iters):
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from human_dynamics_b200.smpl import batch_rodrigues
    from src.tf_smpl.batch_smpl import SMPL
    B, T, S = 8, 20, 224
    smpl = SMPL(smpl_model)
    rng = np.random.RandomState(5)
    batch = {'labels': torch.from_numpy(np.concatenate([rng.uniform(-1, 1, (B, T, 25, 2)), np.ones((B, T, 25, 1))], -1)
                                        .astype(np.float32)).cuda(),
             'poses': torch.from_numpy(rng.normal(0, 0.3, (B, T, 72)).astype(np.float32)).cuda(),
             'shape': torch.from_numpy(rng.normal(0, 0.5, (B, 10)).astype(np.float32)).cuda(),
             'gt3ds': torch.from_numpy(rng.normal(0, 0.3, (B, T, 14, 3)).astype(np.float32)).cuda(),
             'has_3d': torch.ones((B, 2), device='cuda')}
    img = torch.from_numpy(synthetic.make_images(8, seed=2, size=S)).cuda().repeat(B * T // 8, 1, 1, 1).view(B, T, S, S, 3).contiguous()
    out = {}
    for mode in ('images', 'phis'):
        cfg = TrainConfig(do_hallucinate=True, do_hallucinate_preds=True, precomputed_phi=(mode == 'phis'))
        tr = HMMRTrainer(cfg, w, smpl)
        n = tr.n_fake(B, T)
        aa = torch.from_numpy(np.random.RandomState(3).normal(0, 0.3, (n * 24, 3)).astype(np.float32)).cuda()
        mocap = batch_rodrigues(aa).reshape(n, 216)
        b = dict(batch)
        if mode == 'images':
            b['images'] = img
        else:
            b['phis'] = torch.from_numpy(rng.normal(0, 1, (B, T, 2048)).astype(np.float32)).cuda()
        out['step_%s_ms' % mode] = time_call(lambda: tr.step(b, mocap), iters, 2)
        del tr
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, nargs='+', default=[160, 640])
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_image_train: needs a CUDA device')
    from human_dynamics_b200 import synthetic
    w = synthetic.make_synthetic_weights(seed=1, with_hal=True)
    res = dict(card())
    res['trunk'] = []
    for n in a.n:
        res['trunk'].append(trunk(w, n, a.iters, a.rounds))
        torch.cuda.empty_cache()
    res.update(steps(w, synthetic.make_synthetic_smpl(seed=2), a.iters))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
