"""Time one HMMRTrainer step that trains the ResNet trunk (precomputed_phi=False, freeze_phi=False) against the frozen-trunk image step,
alternated in one run, at B x T frames of S x S, and split the unfrozen step:

  python tools/bench_trunk_train.py [--B 8 --T 20 --S 224 --iters 5]

Prints: both step times (median over --iters alternated pairs, CUDA events); the trunk's training forward and its backward, the
backward split into weight gradients (hd_conv_wgrad, with achieved TF/s against the 3xTF32 tensor-core bound of 495/3 TF/s dense),
data-gradient GEMMs, batch-norm backward and pool1 / zero insertion (each timed by wrapping the plan's calls in events, one extra
backward); peak device memory; the card's name and power limit, read in the same run."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _ms(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--B', type=int, default=8)
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--S', type=int, default=224)
    ap.add_argument('--iters', type=int, default=5)
    args = ap.parse_args()
    from human_dynamics_b200 import synthetic, nets
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from human_dynamics_b200.smpl import batch_rodrigues
    from src.tf_smpl.batch_smpl import SMPL
    B, T, S = args.B, args.T, args.S
    w = synthetic.make_synthetic_weights(seed=1)
    smpl = SMPL(synthetic.make_synthetic_smpl(seed=2))
    rng = np.random.RandomState(0)
    batch = {'labels': torch.from_numpy(np.concatenate([rng.uniform(-1, 1, (B, T, 25, 2)), np.ones((B, T, 25, 1))], -1).astype(np.float32)).cuda(),
             'poses': torch.from_numpy(rng.normal(0, 0.3, (B, T, 72)).astype(np.float32)).cuda(),
             'shape': torch.from_numpy(rng.normal(0, 0.5, (B, 10)).astype(np.float32)).cuda(),
             'gt3ds': torch.from_numpy(rng.normal(0, 0.3, (B, T, 14, 3)).astype(np.float32)).cuda(),
             'has_3d': torch.ones((B, 2), device='cuda'),
             'images': torch.from_numpy(synthetic.make_images(B * T, seed=1, size=S).reshape(B, T, S, S, 3)).cuda()}
    un = HMMRTrainer(TrainConfig(precomputed_phi=False, freeze_phi=False), w, smpl)
    fz = HMMRTrainer(TrainConfig(precomputed_phi=False), w, smpl)
    mocap = batch_rodrigues(torch.from_numpy(rng.normal(0, 0.3, (un.n_fake(B, T) * 24, 3)).astype(np.float32)).cuda()).reshape(-1, 216)
    for tr in (un, fz):
        tr.step(batch, mocap)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t_un, t_fz = [], []
    for _ in range(args.iters):
        t_un.append(_ms(lambda: un.step(batch, mocap)))
        t_fz.append(_ms(lambda: fz.step(batch, mocap)))
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    net = un.trunk.net
    n = B * T
    imgs = batch['images'].reshape(n, S, S, 3)
    plan = net.plan(n, S)
    phis = torch.empty((n, 2048), device='cuda')
    dphi = torch.randn((n, 2048), device='cuda') * 1e-3
    t_fwd = _ms(lambda: plan.run(imgs, phis), 3)
    t_bwd = _ms(lambda: plan.backward(dphi, imgs), 3)
    # split the backward by wrapping its calls in events
    parts = {'wgrad': 0.0, 'dgrad': 0.0, 'dgrad_s2': 0.0, 'bn': 0.0, 'other': 0.0}
    flops = {}
    events = []
    orig_w, orig_b = plan._wgrad, plan._bn_backward

    def timed(kind, fn, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(*a, **k)
        e1.record()
        events.append((kind, e0, e1, a))
    plan._wgrad = lambda *a, **k: timed('wgrad', orig_w, *a, **k)
    plan._bn_backward = lambda *a, **k: timed('bn', orig_b, *a, **k)
    class Timed(object):
        def __init__(self, op, kind):
            self.op, self.kind = op, kind

        def run(self, st):
            timed(self.kind, self.op.run, st)
    for unit, u in zip(plan.p.units, plan._backward_state()['units']):
        for c in ('conv1', 'conv2', 'conv3', 'shortcut'):
            if c in u:
                u[c] = Timed(u[c], 'dgrad_s2' if c == 'conv2' and unit['stride'] > 1 else 'dgrad')
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    plan.backward(dphi, imgs)
    e1.record()
    torch.cuda.synchronize()
    total = e0.elapsed_time(e1)
    for kind, a, b, arg in events:
        ms = a.elapsed_time(b)
        parts[kind] += ms
        if kind == 'wgrad':
            nn_, H, W, Cin, Ho, Wo, KH, KW = arg[1][:8]
            cls = '%dx%d' % (KH, KW) + (' s2' if arg[1][8] > 1 else '')
            f, t = flops.get(cls, (0.0, 0.0))
            flops[cls] = (f + 2.0 * nn_ * Ho * Wo * KH * KW * Cin * arg[4], t + ms)
    parts['other'] = total - parts['wgrad'] - parts['dgrad'] - parts['dgrad_s2'] - parts['bn']
    # the zero insertions of the three strided units (the same calls as the backward's, timed on their own)
    import ctypes as C
    from human_dynamics_b200._lib import lib, check, fptr, current_stream
    S_ = plan._backward_state()
    zi = []
    for unit, u in zip(plan.p.units, S_['units']):
        if unit['stride'] > 1:
            zi.append((u['Ho'], u['H'], unit['base']))

    def zero_insert():
        for Ho, H, base in zi:
            check(lib.hd_zero_insert(fptr(S_['D2']), fptr(S_['Z']), n, Ho, Ho, base, 2, H, H, current_stream()), 'hd_zero_insert')
    t_zi = _ms(zero_insert, 5)
    # Adam over the trunk's 172 parameters (values do not change its cost) and the repacks a changed weight triggers
    for p in net.parameters():
        p.grad = torch.zeros_like(p)
    t_adam = _ms(lambda: un.e_opt.step(), 3)
    un.e_opt.zero_grad(set_to_none=True)
    t_rep_f = _ms(net.sync_packs)
    t_rep_b = _ms(net.sync_bwd_packs)
    name = torch.cuda.get_device_name()
    try:
        plim = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        plim = 'unknown'
    print('device: %s, power limit %s' % (name, plim))
    print('B=%d T=%d S=%d: step with the trunk training %.1f ms, frozen-trunk image step %.1f ms (medians of %d alternated pairs)'
          % (B, T, S, float(np.median(t_un)), float(np.median(t_fz)), args.iters))
    print('trunk training forward %.2f ms, backward %.2f ms (%d launches); peak memory of the steps %.2f GiB'
          % (t_fwd, t_bwd, plan.num_backward_launches, peak))
    print('backward split (one instrumented pass, %.2f ms): wgrad %.2f, dgrad GEMMs %.2f (stride-2 3x3 ones %.2f more, plus %.2f of zero '
          'insertion), BN backward %.2f, pool1 / zero insertion / tail %.2f ms' % (total, parts['wgrad'], parts['dgrad'], parts['dgrad_s2'],
                                                                                  t_zi, parts['bn'], parts['other']))
    print('stride-2 data gradients (zero insertion + 3 GEMMs): %.2f ms = %.1f %% of the step' % (
        parts['dgrad_s2'] + t_zi, 100 * (parts['dgrad_s2'] + t_zi) / float(np.median(t_un))))
    print('E Adam step (temporal model + trunk) %.2f ms; repack after a step: forward packs %.2f ms, data-gradient packs %.2f ms'
          % (t_adam, t_rep_f, t_rep_b))
    for cls, (f, t) in sorted(flops.items()):
        print('  hd_conv_wgrad %-6s %.2f ms, %.1f TF/s (3xTF32 bound 165 TF/s)' % (cls, t, f / t / 1e9))
    print('step remainder outside the trunk forward / backward, Adam and repack (temporal model, losses, D): %.1f ms'
          % (float(np.median(t_un)) - t_fwd - t_bwd - t_adam - t_rep_f - t_rep_b))


if __name__ == '__main__':
    main()
