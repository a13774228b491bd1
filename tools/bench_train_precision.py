"""The two gradient precisions of training in one process: grad_precision 'fp32' (3xTF32 backward GEMMs) and 'tf32' (1xTF32), alternated
over several rounds on the same batches.  Reports medians of
  - the phi-input step of the reference's do_train.sh (B = 8, T = 20, delta_t = +-5, do_hallucinate, do_hallucinate_preds), ms;
  - the image-input step that trains the trunk (precomputed_phi=False, freeze_phi=False, B = 8, T = 20, 224^2), ms;
  - inside that step's trunk backward, CUDA events around the weight-gradient launches (hd_conv_wgrad / _ex) and the data-gradient
    GEMMs (hd_conv_gemm), ms each, from one instrumented backward per round (the instrumented backward is not part of the step times);
  - peak device memory of each mode's two trainers through their first steps (torch.cuda.max_memory_allocated above what was
    allocated before them);
with the card name, its power limit and max SM clock read in the same run.  One JSON line on stdout (and in --out).

    python tools/bench_train_precision.py [--rounds 5] [--steps 3] [--S 224] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

MODES = ('fp32', 'tf32')


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


def make_batch(B, T, S, seed):
    """Seeded labels / poses / shapes / 3-D joints, plus phis (phi input) or synthetic frames (image input, S > 0)."""
    from human_dynamics_b200 import synthetic
    rng = np.random.RandomState(seed)
    b = {'labels': torch.from_numpy(np.concatenate([rng.uniform(-1, 1, (B, T, 25, 2)), np.ones((B, T, 25, 1))], -1).astype(np.float32)),
         'poses': torch.from_numpy(rng.normal(0, 0.3, (B, T, 72)).astype(np.float32)),
         'shape': torch.from_numpy(rng.normal(0, 0.5, (B, 10)).astype(np.float32)),
         'gt3ds': torch.from_numpy(rng.normal(0, 0.3, (B, T, 14, 3)).astype(np.float32)),
         'has_3d': torch.ones((B, 2))}
    if S:
        b['images'] = torch.from_numpy(synthetic.make_images(B * T, seed=seed, size=S).reshape(B, T, S, S, 3))
    else:
        b['phis'] = torch.from_numpy(rng.normal(0, 1, (B, T, 2048)).astype(np.float32))
    return b


def mocap(n, seed):
    from human_dynamics_b200.smpl import batch_rodrigues
    aa = torch.from_numpy(np.random.RandomState(seed).normal(0, 0.3, size=(n * 24, 3)).astype(np.float32)).cuda()
    return batch_rodrigues(aa).reshape(n, 216)


def split_backward(plan, images):
    """One trunk backward with CUDA events around every weight-gradient call and every data-gradient GEMM: (wgrad ms, dgrad ms)."""
    n = plan.n
    dphi = torch.randn((n, 2048), device='cuda') * 1e-3
    events = []
    orig = plan._wgrad

    def wgrad(*a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        orig(*a, **k)
        e1.record()
        events.append(('wgrad', e0, e1))

    class Timed(object):
        def __init__(self, op):
            self.op = op

        def run(self, st):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            self.op.run(st)
            e1.record()
            events.append(('dgrad', e0, e1))
    units = plan._backward_state()['units']
    saved = [dict(u) for u in units]
    plan._wgrad = wgrad
    for u in units:
        for c in ('conv1', 'conv2', 'conv3', 'shortcut'):
            if c in u:
                u[c] = Timed(u[c])
    try:
        plan.backward(dphi, images)
        torch.cuda.synchronize()
    finally:
        del plan._wgrad
        for u, s in zip(units, saved):
            u.update(s)
    out = {'wgrad': 0.0, 'dgrad': 0.0}
    for kind, e0, e1 in events:
        out[kind] += e0.elapsed_time(e1)
    return out['wgrad'], out['dgrad']


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=3, help='steps per timed window')
    ap.add_argument('--B', type=int, default=8)
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--S', type=int, default=224)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from src.tf_smpl.batch_smpl import SMPL

    B, T, S = args.B, args.T, args.S
    w = synthetic.make_synthetic_weights(seed=1, with_hal=True)
    smpl_model = synthetic.make_synthetic_smpl(seed=2)
    phi_batch, img_batch = make_batch(B, T, 0, 3), make_batch(B, T, S, 4)
    info = card()                                  # the first device call
    smpl = SMPL(smpl_model)
    phi_batch = {k: v.cuda() for k, v in phi_batch.items()}
    img_batch = {k: v.cuda() for k, v in img_batch.items()}
    flags = dict(do_hallucinate=True, do_hallucinate_preds=True)
    tr, peak = {}, {}
    for m in MODES:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        tr[m] = (HMMRTrainer(TrainConfig(grad_precision=m, **flags), w, smpl),
                 HMMRTrainer(TrainConfig(grad_precision=m, precomputed_phi=False, freeze_phi=False), w, smpl))
        mc = (mocap(tr[m][0].n_fake(B, T), 5), mocap(tr[m][1].n_fake(B, T), 6))
        tr[m] = tr[m] + mc
        tr[m][0].step(phi_batch, mc[0])
        tr[m][1].step(img_batch, mc[1])
        torch.cuda.synchronize()
        peak[m] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    res = {m: {'phi_step_ms': [], 'image_step_ms': [], 'wgrad_ms': [], 'dgrad_ms': []} for m in MODES}
    n = B * T
    for _ in range(args.rounds):
        for m in MODES:
            tp, ti, mp, mi = tr[m]
            res[m]['phi_step_ms'].append(timed(lambda: tp.step(phi_batch, mp), args.steps))
            res[m]['image_step_ms'].append(timed(lambda: ti.step(img_batch, mi), args.steps))
            plan = ti.trunk.net.plan(n, S)
            wg, dg = split_backward(plan, img_batch['images'].reshape(n, S, S, 3))
            res[m]['wgrad_ms'].append(wg)
            res[m]['dgrad_ms'].append(dg)
    out = {'tool': 'bench_train_precision', **info, 'B': B, 'T': T, 'S': S, 'rounds': args.rounds, 'steps': args.steps,
           'phi_flags': 'delta_t=+-5 do_hallucinate do_hallucinate_preds', 'peak_mib': {m: round(peak[m]) for m in MODES}}
    for m in MODES:
        out[m] = {k: round(float(np.median(v)), 2) for k, v in res[m].items()}
        out[m]['runs'] = {k: [round(x, 2) for x in v] for k, v in res[m].items()}
    for k in ('phi_step_ms', 'image_step_ms', 'wgrad_ms', 'dgrad_ms'):
        out['speedup_' + k[:-3]] = round(out['fp32'][k] / out['tf32'][k], 3)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
