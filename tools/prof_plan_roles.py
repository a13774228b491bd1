"""Per-role cycle counters (hd_conv_gemm_profile, CTA 0) + CUDA-event time of every distinct conv layer of the REAL trunk plans
(stage A: 160 frames root + blocks 1-2; stage B: 640 frames blocks 3-4), in plan order.    python tools/prof_plan_roles.py [A|B|AB]"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                                     # noqa: E402
from human_dynamics_b200 import synthetic                         # noqa: E402
from human_dynamics_b200._lib import lib, check                   # noqa: E402
from human_dynamics_b200.nets import PackedResNet, ResNetPlan     # noqa: E402

# dbg[0..6] (conv_simt.cu); the last two are parts of `epilogue`, the rest of it is arithmetic and issuing stores
NAMES = ['prod_loop', 'prod_wait_empty', 'cons_loop', 'cons_wait_full', 'epilogue', 'epi_wait_res', 'epi_wait_stores']


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else 'AB'
    dev = torch.device('cuda')
    w = synthetic.make_synthetic_weights(seed=1)
    packed = PackedResNet(w, dev, tc='auto')
    nu = len(packed.units)
    cut = 7
    plans = []
    if 'A' in which:
        nxt = packed.units[cut]
        pa = ResNetPlan(packed, 160, 224, 'auto', units=(0, cut), root=True, tail=False, next_pre=nxt['pre'], next_has_shortcut='shortcut' in nxt)
        img = torch.from_numpy(synthetic.make_images(160, seed=3)).to(dev)
        pa.run(img, None)
        plans.append(('A', pa, [pa.conv1_op] + pa.ops))
    if 'B' in which:
        pb = ResNetPlan(packed, 640, 224, 'auto', units=(cut, nu), root=False, tail=True)
        pb.in_split[0].normal_(); pb.in_split[1].zero_(); pb.in_buf.normal_()
        phi = torch.empty((640, 2048), device=dev)
        pb.run(None, phi)
        plans.append(('B', pb, pb.ops))
    torch.cuda.synchronize()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    seen = set()
    for tag, plan, ops in plans:
        for op in ops:
            d = getattr(op, 'd', None)
            if d is None:
                continue
            K = d.KH * d.KW * d.Cin
            M = d.n_img * d.Ho * d.Wo
            sig = (tag, M, K, d.Cout, d.KH, d.stride, bool(d.res), bool(d.out), bool(d.out_hi))
            if sig in seen:
                continue
            seen.add(sig)
            dbg = torch.zeros(16, dtype=torch.int64, device=dev)
            for _ in range(2):
                check(lib.hd_conv_gemm_profile(op.ref, st, C.c_void_p(dbg.data_ptr())))
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                op.run(st)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / 5 * 1e3
            v = dbg.cpu().numpy()
            print('%s M=%7d K=%5d N=%4d k%d s%d res=%d o32=%d o16=%d : %7.1f us  %6.1f TF/s' % (tag, M, K, d.Cout, d.KH, d.stride, bool(d.res), bool(d.out),
                  bool(d.out_hi), us, 2.0 * M * K * d.Cout / us / 1e6))
            print('     ' + '  '.join('%s=%d' % (nm, x) for nm, x in zip(NAMES, v)), flush=True)


if __name__ == '__main__':
    main()
