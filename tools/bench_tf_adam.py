"""TF's Adam (optim.TFAdam, one hd_adam_tf launch plus the powers) against torch.optim.Adam (foreach, the trainer's default) and
torch.optim.Adam(fused=True), alternated in one process over several rounds.  Reports medians of
  - one optimizer step over E's parameter set of the phi-input trainer (do_train.sh's flags) and of the trunk-training trainer
    (precomputed_phi=False, freeze_phi=False), ms, with the bytes it must move (28 B per element: p, g, m, v read, p, m, v written)
    over that time and its share of the H100 SXM's 3.35 TB/s;
  - HMMRTrainer.step with each optimizer (the phi-input do_train.sh step, B = 8, T = 20, and the trunk-training step from S x S images);
with the card name, its power limit and max SM clock read in the same run.  One JSON line on stdout (and in --out).

    python tools/bench_tf_adam.py [--rounds 5] [--iters 20] [--steps 3] [--S 224] [--out FILE]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np
import torch

from bench_train_precision import card, make_batch, mocap, timed

HBM_BYTES_PER_S = 3.35e12
OPTS = ('tf_adam', 'torch_foreach', 'torch_fused')


def factory(kind):
    from human_dynamics_b200.optim import TFAdam
    if kind == 'tf_adam':
        return lambda params, lr: TFAdam(params, lr)
    if kind == 'torch_foreach':
        return lambda params, lr: torch.optim.Adam(params, lr, foreach=True)
    return lambda params, lr: torch.optim.Adam(params, lr, fused=True)


def trainer_config(which, S):
    from human_dynamics_b200.objective import TrainConfig
    if which == 'phi':
        return TrainConfig(num_conv_layers=3, do_hallucinate=True, do_hallucinate_preds=True), 0
    return TrainConfig(precomputed_phi=False, freeze_phi=False), S


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=20, help='optimizer steps per timed window')
    ap.add_argument('--steps', type=int, default=3, help='trainer steps per timed window')
    ap.add_argument('--B', type=int, default=8)
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--S', type=int, default=224)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_tf_adam: needs a CUDA device')
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import HMMRTrainer
    from src.tf_smpl.batch_smpl import SMPL
    torch.cuda.set_device(0)
    w = synthetic.make_synthetic_weights(seed=1, with_hal=True)
    smpl = SMPL(synthetic.make_synthetic_smpl(seed=2))
    res = {'card': card(), 'B': a.B, 'T': a.T, 'S': a.S, 'rounds': a.rounds, 'optimizer_step': {}, 'trainer_step_ms': {}}
    for which in ('phi', 'trunk'):
        cfg, S = trainer_config(which, a.S)
        # the optimizer alone, over the trainer's E parameters with fixed gradients (one parameter copy per optimizer)
        base = HMMRTrainer(cfg, w, smpl)
        numel = sum(p.numel() for p in base.e_params)
        gen = torch.Generator(device='cuda').manual_seed(0)
        grads = [torch.randn(p.shape, device='cuda', generator=gen) * 1e-3 for p in base.e_params]
        sets = {}
        for k in OPTS:
            ps = [torch.nn.Parameter(p.detach().clone()) for p in base.e_params]
            for p, g in zip(ps, grads):
                p.grad = g
            sets[k] = factory(k)(ps, cfg.e_lr)
            sets[k].step()                                   # slots created, kernels loaded
        del base
        times = {k: [] for k in OPTS}
        for _ in range(a.rounds):
            for k in OPTS:
                times[k].append(timed(sets[k].step, a.iters))
        out = {'tensors': len(grads), 'elements': numel, 'bytes_per_step': 28 * numel}
        for k in OPTS:
            ms = float(np.median(times[k]))
            out[k] = {'ms': round(ms, 4), 'GB_per_s': round(28 * numel / ms / 1e6, 1),
                      'share_of_3.35TB_per_s': round(28 * numel / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}
        out['hbm_floor_ms'] = round(28 * numel / HBM_BYTES_PER_S * 1e3, 4)
        res['optimizer_step'][which] = out
        del sets, grads
        torch.cuda.empty_cache()
        # the whole trainer step with each optimizer
        batch = {k: v.cuda() for k, v in make_batch(a.B, a.T, S, 3).items()}
        trs = {}
        steps = {k: [] for k in OPTS}
        for k in OPTS:
            tr = HMMRTrainer(cfg, w, smpl, optimizer=factory(k))
            mc = mocap(tr.n_fake(a.B, a.T), 4)
            tr.step(batch, mc)
            trs[k] = (tr, mc)
            if which == 'trunk':                              # one trunk trainer alive at a time: each holds ~14 GB
                for _ in range(a.rounds):
                    steps[k].append(timed(lambda: tr.step(batch, mc), a.steps))
                del tr, trs[k]
                torch.cuda.empty_cache()
        if which == 'phi':
            for _ in range(a.rounds):
                for k in OPTS:
                    tr, mc = trs[k]
                    steps[k].append(timed(lambda: tr.step(batch, mc), a.steps))
        res['trainer_step_ms'][which] = {k: round(float(np.median(v)), 3) for k, v in steps.items()}
        res['trainer_step_ms'][which]['alternated'] = which == 'phi'
        del trs
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
