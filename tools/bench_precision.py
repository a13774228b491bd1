"""The two precision modes of the networks in one process: 'tc3h' (FP32-class, 3xFP16) and 'tc1h' (half-precision inference,
1xFP16), alternated over several rounds on the same frames.  Reports medians of
  - C3 device-resident: B = 32 clips x T = 20 at 224^2, one CUDA-graph step (HMMREngine.predict_graphed), frames / s;
  - Tester.predict end to end on a plain numpy array of the same frames (host -> device -> host), frames / s;
  - C2: single-frame batch of 64 (HMMREngine.predict_graphed, single_frame=True), frames / s;
  - peak device memory of each mode's engine (torch.cuda.max_memory_allocated, reset before the mode's warm-up);
and the deviation of 'tc1h' from 'tc3h' per output key (max |err| / max |ref| over the C3 step), with the card name, its power limit
and max SM clock read in the same run.  One JSON line on stdout (and in --out)."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

MODES = ('tc3h', 'tc1h')


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader'], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().split(',')] if q.returncode == 0 else (torch.cuda.get_device_name(), None, None)
    return {'name': name, 'power_limit': power, 'max_sm_clock': clock}


def timed(fn, steps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=10, help='steps per timed window (C3 / C2); Tester.predict takes steps // 2 + 1')
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    from human_dynamics_b200 import synthetic, HMMRConfig
    from human_dynamics_b200.engine import HMMREngine
    from src.evaluation.tester import Tester

    B, T, S = 32, 20, 224
    w = synthetic.make_synthetic_weights(seed=1, with_hal=True)
    smpl = synthetic.make_synthetic_smpl(seed=2)
    img = synthetic.make_images(B * T, seed=0).reshape(B, T, S, S, 3)
    img_dev = torch.from_numpy(img).cuda()
    img_np = np.array(img, copy=True)
    img64 = torch.from_numpy(synthetic.make_images(64, seed=300)).cuda().view(64, 1, S, S, 3)

    eng, tester, eng64, peak, outs = {}, {}, {}, {}, {}
    for m in MODES:
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        cfg = HMMRConfig(batch_size=B, sequence_length=T, impl=m)
        eng[m] = HMMREngine(w, smpl, cfg)
        out, _ = eng[m].predict_graphed(img_dev)
        torch.cuda.synchronize()
        outs[m] = {k: v.detach().double().cpu() for k, v in eng[m].predict(img_dev).items()}
        tester[m] = Tester(cfg, engine=eng[m])
        tester[m].predict(img_np)
        torch.cuda.synchronize()
        peak[m] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        eng64[m] = HMMREngine(w, smpl, HMMRConfig(batch_size=64, sequence_length=1, impl=m))
        eng64[m].predict_graphed(img64, single_frame=True)
        torch.cuda.synchronize()
    dev = {}
    for k, ref in outs['tc3h'].items():
        dev[k] = float((outs['tc1h'][k] - ref).abs().max() / max(float(ref.abs().max()), 1e-12))

    res = {m: {'c3': [], 'e2e': [], 'c2': []} for m in MODES}
    for _ in range(args.rounds):
        for m in MODES:
            res[m]['c3'].append(B * T / (timed(lambda: eng[m].predict_graphed(img_dev), args.steps) * 1e-3))
            res[m]['c2'].append(64 / (timed(lambda: eng64[m].predict_graphed(img64, single_frame=True), args.steps) * 1e-3))
            res[m]['e2e'].append(B * T / (timed(lambda: tester[m].predict(img_np), args.steps // 2 + 1) * 1e-3))
    line = {'card': card(), 'rounds': args.rounds, 'steps': args.steps, 'unit': 'frames/sec',
            'deviation_tc1h_vs_tc3h': dev, 'peak_device_mib': peak}
    for m in MODES:
        line[m] = {k: {'median': float(np.median(v)), 'min': float(min(v)), 'max': float(max(v))} for k, v in res[m].items()}
    line['speedup'] = {k: line['tc1h'][k]['median'] / line['tc3h'][k]['median'] for k in ('c3', 'e2e', 'c2')}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
