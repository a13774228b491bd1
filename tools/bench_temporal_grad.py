"""Times one training step of the temporal model (human_dynamics_b200/trainable.py) on the H100 and prints one JSON line.

Shape: B clips x T frames of synthetic phi (default 32 x 20 = 640 frames), f_movie + the three IEF heads (main, past5, future5),
synthetic weights.  Two losses: a fixed random contraction of theta and the delta outputs ('heads'), and the keypoint reprojection
loss of the main and delta heads through predict_from_features and the SMPL backward ('kps').  For each: forward, backward, repack
(every weight changed in place, then the forward + backward-data packs rebuilt) and Adam step, each timed with CUDA events over --iters
repetitions after --warmup; a separate torch.profiler run gives the per-kernel split of one step.  The card's name and power limit are
read in the same run.  The bound printed beside the numbers is ESTIMATED from FLOPs and bytes at data-sheet rates, not measured.

    python tools/bench_temporal_grad.py [--B 32] [--T 20] [--iters 10] [--warmup 3]
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

from bench_smpl_grad import card, kernel_ms, time_call          # noqa: E402

TF32_DENSE_TFLOPS = 494.7     # H100 SXM data sheet, dense TF32 tensor core
HBM_TBPS = 3.35               # H100 SXM data sheet


def bound(B, T, n_params):
    M = B * T
    fm = 6 * 2 * (2 * M * 6144 * 2048)                          # 6 convs: dX and dW, 2*M*K*N each
    ief = 3 * 3 * 2 * 2 * M * 1024 * 1024 + 3 * 2 * 2 * M * 2048 * 1024 + 3 * 3 * 2 * 2 * M * 85 * 1024   # fc2 x3 stages, fc1 phi, small
    adam_bytes = 7 * 4 * n_params                               # read p, g, m, v; write p, m, v
    r = {'fmovie_bwd_gflop': round(fm / 1e9, 1), 'fmovie_bwd_ms': round(3 * fm / (TF32_DENSE_TFLOPS * 1e9), 3),
         'ief_bwd_gflop': round(ief / 1e9, 1), 'ief_bwd_ms': round(3 * ief / (TF32_DENSE_TFLOPS * 1e9), 3),
         'adam_gb': round(adam_bytes / 1e9, 2), 'adam_ms': round(adam_bytes / (HBM_TBPS * 1e9), 3)}
    r['step_floor_ms'] = round(r['fmovie_bwd_ms'] * 1.5 + r['ief_bwd_ms'] * 1.5 + r['adam_ms'], 3)   # forward ~ half a backward
    r['note'] = 'estimated from FLOPs / bytes at data-sheet rates (3 TF32 passes per GEMM), not measured'
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--B', type=int, default=32)
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.trainable import TemporalModel
    from src.tf_smpl.batch_smpl import SMPL
    torch.cuda.set_device(0)
    w = synthetic.make_synthetic_weights(seed=1)
    model = TemporalModel(w)
    smpl = SMPL(synthetic.make_synthetic_smpl(seed=2))
    B, T = a.B, a.T
    N = B * T
    g = torch.Generator(device='cuda').manual_seed(0)
    phi = torch.randn((B, T, 2048), device='cuda', generator=g)
    U = torch.randn((N, 85), device='cuda', generator=g)
    K = smpl.consts.num_kps
    gt = torch.rand((B, T, K, 2), device='cuda', generator=g) * 1.6 - 0.8
    gtd = torch.rand((B, T, 2, K, 2), device='cuda', generator=g) * 1.6 - 0.8
    opt = torch.optim.Adam(model.parameters(), lr=1e-6)
    n_params = sum(p.numel() for p in model.parameters())

    def loss_heads():
        th, dl = model.regress(model.temporal_encode(phi).reshape(N, 2048))
        return (th * U).sum() + sum((v * U).sum() for v in dl.values())

    def loss_kps():
        out = model.predict_from_features(phi, smpl)
        return (out['kps'] - gt).abs().mean() + (out['kps_delta'] - gtd).abs().mean()

    def touch():
        with torch.no_grad():
            for p in model.parameters():
                p.add_(0.0)                       # bumps every version counter: the next forward / backward repack everything

    def repack():
        touch()
        model.sync_packs()
        model.sync_bwd_packs()

    res = {'tool': 'bench_temporal_grad', **card(), 'B': B, 'T': T, 'frames': N, 'params': n_params, 'bound': bound(B, T, n_params),
           'losses': {}}
    def fwd_bwd(lf):
        """(forward ms, backward ms): CUDA events around each half of every repetition, summed."""
        for _ in range(a.warmup):
            lf().backward()
        torch.cuda.synchronize()
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(a.iters)]
        for e in ev:
            e[0].record()
            loss = lf()
            e[1].record()
            loss.backward()
            e[2].record()
            del loss
        torch.cuda.synchronize()
        return (round(sum(e[0].elapsed_time(e[1]) for e in ev) / a.iters, 4), round(sum(e[1].elapsed_time(e[2]) for e in ev) / a.iters, 4))

    for name, lf in (('heads', loss_heads), ('kps', loss_kps)):
        def step():
            opt.zero_grad(set_to_none=True)
            lf().backward()
            opt.step()
        t_fwd, t_bwd = fwd_bwd(lf)
        with torch.no_grad():
            t_fwd_nograd = time_call(lambda: lf(), a.iters, a.warmup)
        r = {'forward_ms': t_fwd, 'forward_nograd_ms': t_fwd_nograd, 'backward_ms': t_bwd,
             'repack_ms': time_call(repack, a.iters, a.warmup), 'touch_ms': time_call(touch, a.iters, a.warmup),
             'optimizer_ms': time_call(opt.step, a.iters, a.warmup), 'step_ms': time_call(step, a.iters, a.warmup)}
        r['repack_ms'] = round(r['repack_ms'] - r['touch_ms'], 4)
        r['step_kernels_ms'] = kernel_ms(step)
        res['losses'][name] = r
    print(json.dumps(res))


if __name__ == '__main__':
    main()
