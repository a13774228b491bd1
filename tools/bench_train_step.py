"""Times one HMMRTrainer step (human_dynamics_b200/objective.py) on the GPU and prints one JSON line.

Shapes: B = 8, T = 20 with the flags of the reference's do_train.sh (delta_t = +-5, do_hallucinate, do_hallucinate_preds: six
prediction sets, n_fake = 960), and B = 32, T = 20 with the same flags.  Synthetic weights (f_movie, IEF heads, fc2_res), a synthetic
SMPL and seeded data.  Per shape, CUDA events over --iters steps after --warmup:
  step_ms          the whole step (forward, objective, D, both backwards, both Adam updates);
  forward_ms       f_movie, fc2_res, the IEF heads, SMPL, the objective's forward and D's forward, on the graph;
  objective_ms     the objective's forward + backward alone (LossFunction on fixed inputs);
  d_ms             D_pose forward + backward on the reals + fakes alone;
  adam_ms          the two optimizer steps alone;
  backward_ms      step - forward - adam: the network, SMPL, objective and D backwards;
  launches         libhd_b200 kernel launches of one step (torch's own launches are not counted);
  objective_launches  the same for the objective's forward + backward.
In the same run, alternating with the fused objective, the same objective as float32 torch expressions on the GPU (oracle/losses_ref.py
on CUDA tensors, forward + backward): torch_objective_ms, and the largest relative difference of the named losses; above 1e-5 the
script exits non-zero.
The card's name and power limit are read in the same run.

    python tools/bench_train_step.py [--B 8 32] [--T 20] [--iters 20] [--warmup 5]
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


def launches(fn):
    from human_dynamics_b200 import _lib
    torch.cuda.synchronize()
    _lib.lib.hd_launch_count_reset()
    fn()
    torch.cuda.synchronize()
    return int(_lib.lib.hd_launch_count())


def batch_for(B, T, K, seed):
    from human_dynamics_b200.smpl import batch_rodrigues
    g = torch.Generator(device='cuda').manual_seed(seed)
    lab = torch.randn((B, T, K, 3), device='cuda', generator=g) * 0.5
    lab[..., 2] = (torch.rand((B, T, K), device='cuda', generator=g) > 0.2).float()
    return {'phis': torch.randn((B, T, 2048), device='cuda', generator=g), 'labels': lab,
            'poses': 0.3 * torch.randn((B, T, 72), device='cuda', generator=g), 'shape': torch.randn((B, 10), device='cuda', generator=g),
            'gt3ds': torch.randn((B, T, 14, 3), device='cuda', generator=g), 'has_3d': torch.ones((B, 2), device='cuda')}, \
        lambda n: batch_rodrigues(0.3 * torch.randn((n * 24, 3), device='cuda', generator=g)).reshape(n, 216)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--B', type=int, nargs='+', default=[8, 32])
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    a = ap.parse_args()
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig, evaluate
    from oracle import losses_ref
    from src.tf_smpl.batch_smpl import SMPL
    torch.cuda.set_device(0)
    cfg = TrainConfig(do_hallucinate=True, do_hallucinate_preds=True)
    smpl = SMPL(synthetic.make_synthetic_smpl(seed=2))
    tr = HMMRTrainer(cfg, synthetic.make_synthetic_weights(seed=1, with_hal=True), smpl)
    K = smpl.consts.num_kps
    res = {'tool': 'bench_train_step', **card(), 'iters': a.iters, 'warmup': a.warmup, 'flags': 'delta_t=+-5 do_hallucinate '
           'do_hallucinate_preds', 'shapes': {}}
    for B in a.B:
        T = a.T
        batch, mocap_fn = batch_for(B, T, K, B)
        mocap = mocap_fn(tr.n_fake(B, T))
        r = {'n_fake': tr.n_fake(B, T)}
        r['step_ms'] = time_call(lambda: tr.step(batch, mocap), a.iters, a.warmup)
        r['launches'] = launches(lambda: tr.step(batch, mocap))
        r['forward_ms'] = time_call(lambda: tr.forward(batch, mocap), a.iters, a.warmup)
        params = tr.e_params + tr.d_params
        for p in params:
            p.grad = torch.zeros_like(p)
        r['adam_ms'] = time_call(lambda: (tr.e_opt.step(), tr.d_opt.step()), a.iters, a.warmup)
        for p in params:
            p.grad = None
        r['backward_ms'] = round(r['step_ms'] - r['forward_ms'] - r['adam_ms'], 4)
        # D alone
        fakes = mocap_fn(tr.n_fake(B, T)).reshape(-1, 24, 9)[:, 1:].contiguous().requires_grad_()
        reals = mocap.reshape(-1, 24, 9)[:, 1:].contiguous()

        def d_fb():
            lg = tr.disc(torch.cat([reals, fakes], 0))
            lg.square().sum().backward()
        r['d_ms'] = time_call(d_fb, a.iters, a.warmup)
        # the objective alone: fused kernels against torch expressions, alternating
        obj = tr.objective(B, T, K)
        x = synthetic.make_loss_inputs(obj, seed=B)
        xin = {k: torch.from_numpy(v).cuda().requires_grad_(k in ('omega', 'joints', 'rots', 'strips', 'pred_strips'))
               for k, v in x.items()}

        def fused():
            named, _ = evaluate(obj, xin)
            sum(named.values()).backward()
            return named

        def torch_expr():
            named, _ = losses_ref.objective(cfg, xin)
            sum(named.values()).backward()
            return named
        fm, tm = [], []
        for _ in range(3):
            fm.append(time_call(fused, a.iters, a.warmup))
            tm.append(time_call(torch_expr, a.iters, a.warmup))
        r['objective_ms'], r['torch_objective_ms'] = min(fm), min(tm)
        r['objective_launches'] = launches(fused)
        with torch.no_grad():
            f = evaluate(obj, xin)[0]
            t = losses_ref.objective(cfg, xin)[0]
        r['objective_max_rel_diff'] = max(abs(f[k].item() - t[k].item()) / max(abs(t[k].item()), 1e-30) for k in obj.names)
        res['shapes']['B=%d,T=%d' % (B, T)] = r
    bad = [k for k, r in res['shapes'].items() if not r['objective_max_rel_diff'] <= 1e-5]
    res['objective_agrees'] = not bad
    print(json.dumps(res))
    if bad:
        sys.exit('fused and torch-expression objectives differ by more than 1e-5 at %s' % ', '.join(bad))


if __name__ == '__main__':
    main()
