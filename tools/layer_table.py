"""Per-layer table of one C3 trunk pass: time, TFLOP/s, and the layer's compulsory HBM traffic / time (GB/s).  A chained launch
(hd_conv_gemm_chain: conv3 and the next unit's conv1) is one row with K < 0: both GEMMs' FLOPs, and as bytes its input pair, residual,
fp32 output (or its subsample) and the conv1 pair.
--impl picks the precision mode of the trunk (default 'auto'; 'tc1h' = the half-precision inference mode)."""
import argparse, sys, os, ctypes
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from human_dynamics_b200 import synthetic, HMMRConfig, _lib
from human_dynamics_b200.engine import HMMREngine
ap = argparse.ArgumentParser()
ap.add_argument('--impl', default='auto', help="HMMRConfig.impl of the engine: auto | tc3h | tc1h | tc3 | tc1 | simt")
args = ap.parse_args()
B, T = 32, 20
N = B * T
w = synthetic.make_synthetic_weights(seed=1)
smpl = synthetic.make_synthetic_smpl(seed=2)
eng = HMMREngine(w, smpl, HMMRConfig(batch_size=B, sequence_length=T, impl=args.impl))
img = torch.from_numpy(synthetic.make_images(N, seed=0)).cuda()
phi = eng.encode_images(img)
torch.cuda.synchronize()
stp = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
rows = []
for stage, c in (('A', min(eng.config.frame_chunk, N)), ('B', min(eng.config.late_chunk, N))):
    plan = eng._resnet_plan(c, 224, stage)
    reps = N // c
    ops = ([plan.conv1_op] if plan.conv1_op is not None else []) + plan.ops
    for _ in range(2):
        evs = []
        for op in ops:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); op.run(stp); b.record()
            evs.append((a, b, op))
        torch.cuda.synchronize()
    for a, b, op in evs:
        d = op.d
        if d is None:
            print('  (%s subsample %.3f ms)' % (stage, a.elapsed_time(b) * reps))
            continue
        if d.flags & 2:                   # conv1 over padded planes: report the algorithmic 7x7x3 conv, not the padded K=256 GEMM
            M, K, Nn = d.n_img * d.Ho * d.Wo, 147, d.Cout
            t = a.elapsed_time(b) * 1e-3 * reps
            rows.append((t, stage, M, K, Nn, 7, 2, False, False, 2.0 * M * K * Nn * reps / t / 1e12, (d.n_img * 224 * 224 * 3 * 4 + M * Nn * 4) * reps / t / 1e9, d.impl))
            continue
        M, K, Nn = d.n_img * d.Ho * d.Wo, d.KH * d.KW * d.Cin, d.Cout
        t = a.elapsed_time(b) * 1e-3 * reps
        fl = 2.0 * M * K * Nn * reps
        inb = d.n_img * d.H * d.W * d.Cin * 4
        outb = M * Nn * ((4 if d.out else 0) + (4 if d.out_hi else 0)) + (M * Nn * 4 if d.res else 0)
        chain = getattr(op, 'second', None)
        if chain is not None:             # hd_conv_gemm_chain: both GEMMs' FLOPs, and the second conv's pair is its only other traffic
            fl += 2.0 * M * chain.d.Cin * chain.d.Cout * reps
            outb += M * chain.d.Cout * 4
            K = -K                        # a negative K marks the chained row
        rows.append((t, stage, M, K, Nn, d.KH, d.stride, bool(d.res), bool(d.out_hi), fl / t / 1e12, (inb + outb) * reps / t / 1e9, d.impl))
tot = sum(r[0] for r in rows)
print('trunk conv total %.2f ms  (%.0f TFLOP/s avg)' % (tot * 1e3, sum(r[0] * r[9] for r in rows) / tot))
agg = {}
for r in rows:
    a = agg.setdefault(r[1:9] + (r[11],), [0, 0.0, 0.0, 0.0]); a[0] += 1; a[1] += r[0]; a[2] += r[0] * r[9]; a[3] += r[0] * r[10]
print('%2s %8s %5s %5s k s res spl impl  cnt    ms   TF/s   GB/s' % ('st', 'M', 'K', 'N'))
for k, (c, t, f, g) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print('%2s %8d %5d %5d %d %d %3d %3d %4d %4d %6.2f %6.1f %6.0f' % (k[0], k[1], k[2], k[3], k[4], k[5], k[6], k[7], k[8], c, t * 1e3, f / t, g / t))
