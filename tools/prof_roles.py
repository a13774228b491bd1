"""Per-role cycle counters of CTA (0,0) of the wgmma conv kernel (hd_conv_gemm_profile) for representative layers."""
import sys, os, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from human_dynamics_b200.nets import PackedConv
from human_dynamics_b200._lib import lib, check

NAMES = ['prod_loop', 'prod_wait_empty', 'cons_loop', 'cons_wait_full', 'epilogue']
dev = torch.device('cuda')
rng = np.random.RandomState(0)
cases = [  # n, H, Cin, Cout, k, stride, residual, pre
    (32, 56, 64, 256, 1, 1, True, False),
    (48, 14, 256, 256, 3, 1, False, False),
    (32, 28, 128, 128, 3, 1, False, False),
    (32, 56, 64, 256, 1, 1, True, False),
    (32, 56, 256, 64, 1, 1, False, True),
    (32, 7, 512, 512, 3, 1, False, False),
    (32, 14, 1024, 256, 1, 1, False, True),
]
for n, H, Cin, Cout, k, s, res, pre in cases:
    w = (rng.normal(0, 1, size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(np.float32)
    pc = PackedConv(w, dev, np.ones(Cout, np.float32), np.zeros(Cout, np.float32), True, stride=s, pad=(k // 2, k // 2), tc=os.environ.get('HD_IMPL', 'tc3h'))
    x = torch.randn((n, H, H, Cin), device=dev)
    out = torch.empty((n, H, H, Cout), device=dev)
    r = torch.randn((n, H, H, Cout), device=dev) if res else None
    pr = (torch.ones(Cin, device=dev), torch.zeros(Cin, device=dev), 0, 1) if pre else None
    if os.environ.get('HD_SPLIT', '0') == '1' and not pre:
        xs = (x.half(), ((x - x.half().float()) * 2048).half())
        osp = (torch.empty((n, H, H, Cout), dtype=torch.float16, device=dev), torch.empty((n, H, H, Cout), dtype=torch.float16, device=dev))
        op = pc.bind(None, n, H, H, out if res else None, inp_split=xs, out_split=osp, res=r, impl='tc3h')
    else:
        op = pc.bind(x, n, H, H, out, pre=pr, res=r, impl=os.environ.get('HD_IMPL', 'tc3h'))
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    dbg = torch.zeros(16, dtype=torch.int64, device=dev)
    for _ in range(3):
        check(lib.hd_conv_gemm_profile(op.ref, st, C.c_void_p(dbg.data_ptr())))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        op.run(st)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / 5 * 1e3
    M, K = n * H * H, k * k * Cin
    d = dbg.cpu().numpy()
    print('M=%6d K=%5d N=%4d res=%d pre=%d: %.1f us, %.1f TF/s, chunks=%d, ctas=%d' % (M, K, Cout, res, pre, us, 2.0 * M * K * Cout / us / 1e6, K // 32,
          ((M + 127) // 128) * ((Cout + 127) // 128 if Cout > 64 else 1)))
    print('   ' + '  '.join('%s=%d' % (nm, v) for nm, v in zip(NAMES, d)))
