"""Times the SMPL backward (csrc/smpl_grad.cu + the two tensor-core GEMMs) on the H100 and prints one JSON line.

For each N (default 64, 640, 8192, 65536 poses of the synthetic SMPL model): forward alone (SMPLConstants.forward, what the
no-grad path runs), backward alone (SMPLConstants.backward with random upstream gradients on verts, joints, Rs and Jtr) and
forward + backward, each timed with CUDA events over --iters calls after --warmup calls.  Per-kernel times of one backward come from
a separate torch.profiler run.  The card's name and power limit are read in the same run.

    python tools/bench_smpl_grad.py [--sizes 64,640,8192,65536] [--iters 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def time_call(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / iters, 4)


def kernel_ms(fn):
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        key = ev.key.replace('(anonymous namespace)::', '').replace('void ', '')
        if 'kernel' not in key:
            continue
        name = key.split('(')[0].split('<')[0].split('::')[-1]
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = ev.cuda_time_total
        out[name] = round(out.get(name, 0.0) + t / 1000.0, 4)
    return out


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(',')]
        return {'gpu': name, 'power_limit': power, 'max_sm_clock': clock}
    except Exception as e:                    # report, do not guess
        return {'gpu': torch.cuda.get_device_name(0), 'power_limit': 'unknown (%s)' % e}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='64,640,8192,65536')
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    a = ap.parse_args()
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.smpl import SMPLConstants
    torch.cuda.set_device(0)
    c = SMPLConstants(synthetic.make_synthetic_smpl(seed=2))
    c.grad_state()
    V, K = c.num_verts, c.num_kps
    res = {'tool': 'bench_smpl_grad', **card(), 'sizes': {}}
    for N in [int(x) for x in a.sizes.split(',')]:
        beta, theta = synthetic.make_smpl_inputs(N, seed=1)
        b, t = torch.from_numpy(beta).cuda(), torch.from_numpy(theta).cuda()
        g = torch.Generator(device='cuda').manual_seed(0)
        ups = [torch.randn(s, device='cuda', generator=g) for s in ((N, V, 3), (N, K, 3), (N, 24, 3, 3), (N, 24, 3))]
        fwd = lambda: c.forward(b, t)
        bwd = lambda: c.backward(b, t, *ups)

        def both():
            c.forward(b, t)
            c.backward(b, t, *ups)
        r = {'forward_ms': time_call(fwd, a.iters, a.warmup), 'backward_ms': time_call(bwd, a.iters, a.warmup),
             'fwd_bwd_ms': time_call(both, a.iters, a.warmup), 'backward_kernels_ms': kernel_ms(bwd)}
        r['backward_over_forward'] = round(r['backward_ms'] / r['forward_ms'], 3)
        res['sizes'][str(N)] = r
        del ups
        c._bw_bufs.clear()
        c._tc_bufs.clear()
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
