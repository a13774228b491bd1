"""Times HMMRTrainer.step with and without the IEF heads' dropout and prints one JSON line.

B = 8, T = 20 with the flags of the reference's do_train.sh (delta_t = +-5, do_hallucinate, do_hallucinate_preds: two IEF calls of
three heads per step), synthetic weights and SMPL, seeded data (tools/bench_train_step.py's).  Two trainers in one process, one with
ief_keep_prob 1.0 (the inference graph) and one with 0.5 (the reference's dropout), timed in alternating rounds of --iters steps
after --warmup; per round CUDA events over the round.  Reports the median step time of each over --rounds rounds and the relative
difference of the medians.  The same for the IEF call alone (TemporalModel.regress over the B*T rows, forward + backward, every
head), where the masks are drawn, with its outputs' backward seeded by ones.  Mask elements per step: rows x 1024 x 2 layers x 3
stages x 3 heads x 2 calls.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/bench_ief_dropout.py [--B 8] [--T 20] [--rounds 9] [--iters 10] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_smpl_grad import card, time_call          # noqa: E402
from bench_train_step import batch_for               # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--B', type=int, default=8)
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=9)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from src.tf_smpl.batch_smpl import SMPL
    torch.cuda.set_device(0)
    smpl = SMPL(synthetic.make_synthetic_smpl(seed=2))
    w = synthetic.make_synthetic_weights(seed=1, with_hal=True)
    trainers = {p: HMMRTrainer(TrainConfig(do_hallucinate=True, do_hallucinate_preds=True, ief_keep_prob=p), w, smpl) for p in (1.0, 0.5)}
    B, T = a.B, a.T
    batch, mocap_fn = batch_for(B, T, smpl.consts.num_kps, B)
    mocap = mocap_fn(trainers[1.0].n_fake(B, T))
    times = {p: [] for p in trainers}
    for _ in range(a.rounds):
        for p, tr in trainers.items():
            times[p].append(time_call(lambda: tr.step(batch, mocap), a.iters, a.warmup))
    model = trainers[1.0].model
    feats = batch['phis'].reshape(B * T, 2048).contiguous().requires_grad_()

    def ief(p):
        th, dl = model.regress(feats, dropout=None if p == 1.0 else (1, 0, 0, p))
        torch.autograd.backward([th] + list(dl.values()), [torch.ones_like(th)] + [torch.ones_like(v) for v in dl.values()])
    ief_times = {p: [] for p in trainers}
    for _ in range(a.rounds):
        for p in ief_times:
            ief_times[p].append(time_call(lambda: ief(p), a.iters, a.warmup))
    med = {p: statistics.median(v) for p, v in times.items()}
    imed = {p: statistics.median(v) for p, v in ief_times.items()}
    res = {'tool': 'bench_ief_dropout', **card(), 'B': B, 'T': T, 'rounds': a.rounds, 'iters': a.iters, 'warmup': a.warmup,
           'mask_elements_per_step': B * T * 1024 * 2 * 3 * 3 * 2,
           'step_ms_keep_1.0': round(med[1.0], 4), 'step_ms_keep_0.5': round(med[0.5], 4),
           'dropout_cost_rel': round(med[0.5] / med[1.0] - 1, 5),
           'rounds_ms_keep_1.0': times[1.0], 'rounds_ms_keep_0.5': times[0.5],
           'ief_fwd_bwd_ms_keep_1.0': round(imed[1.0], 4), 'ief_fwd_bwd_ms_keep_0.5': round(imed[0.5], 4),
           'ief_dropout_cost_rel': round(imed[0.5] / imed[1.0] - 1, 5),
           'ief_rounds_ms_keep_1.0': ief_times[1.0], 'ief_rounds_ms_keep_0.5': ief_times[0.5]}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
