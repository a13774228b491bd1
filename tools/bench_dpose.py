"""Times the adversarial pose prior (human_dynamics_b200/adversarial.py) on the GPU and prints one JSON line.

Per N (default 800 = the reference's B=8, T=20, delta_t = +-5 batch of reals + fakes, and 3200 = B=32), N/2 reals and N/2 fakes:
  d_step: forward on reals and on detached fakes, d_real + d_fake, backward (weight gradients only), Adam step;
  e_step: theta (N/2, 72) -> batch_rodrigues -> D frozen -> e_fake, backward to theta (input gradients only).
Plus a no-grad forward of --big poses (default 65 536).  Each is timed with CUDA events over --iters repetitions after --warmup; the
libhd_b200 kernel launches of one repetition are counted (torch's own elementwise launches of the loss and Adam are not).  The card's
name and power limit are read in the same run.

    python tools/bench_dpose.py [--N 800 3200] [--big 65536] [--iters 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--N', type=int, nargs='+', default=[800, 3200])
    ap.add_argument('--big', type=int, default=65536)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    a = ap.parse_args()
    from human_dynamics_b200.adversarial import PoseDiscriminator
    from src import ops
    from src.tf_smpl.batch_lbs import batch_rodrigues
    torch.cuda.set_device(0)
    d = PoseDiscriminator(seed=0)
    opt = torch.optim.Adam(d.parameters(), lr=1e-4)
    g = torch.Generator(device='cuda').manual_seed(0)
    res = {'tool': 'bench_dpose', **card(), 'iters': a.iters, 'warmup': a.warmup, 'steps': {}}
    for N in a.N:
        h = N // 2
        real = batch_rodrigues(torch.randn((h * 23, 3), device='cuda', generator=g)).reshape(h, 23, 9)
        theta = (0.5 * torch.randn((h, 72), device='cuda', generator=g)).requires_grad_()

        def fakes():
            return batch_rodrigues(theta.reshape(-1, 3)).reshape(h, 24, 9)[:, 1:]

        def d_step():
            d.requires_grad_(True)
            opt.zero_grad(set_to_none=True)
            fake = fakes().detach()
            (ops.compute_loss_d_real(d(real)) + ops.compute_loss_d_fake(d(fake))).backward()
            opt.step()

        def e_step():
            d.requires_grad_(False)
            theta.grad = None
            ops.compute_loss_e_fake(d(fakes())).backward()
        res['steps']['N=%d' % N] = {'d_step_ms': time_call(d_step, a.iters, a.warmup), 'd_step_launches': launches(d_step),
                                    'e_step_ms': time_call(e_step, a.iters, a.warmup), 'e_step_launches': launches(e_step)}
    x = batch_rodrigues(torch.randn((a.big * 23, 3), device='cuda', generator=g)).reshape(a.big, 23, 9)
    with torch.no_grad():
        res['forward'] = {'N': a.big, 'ms': time_call(lambda: d(x), a.iters, a.warmup), 'launches': launches(lambda: d(x))}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
