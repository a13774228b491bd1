"""The ResNet root conv1 over the fp16 planes (Cout = 64) runs conv_gemm_tc's channels-on-M tile: 64 output channels x 256 pixels,
the weights as the wgmma A operand and the pixels as its B operand.

- The probe: one wgmma ...f32.f16.f16 gives the same bits for an element with its operands swapped (same products, same accumulator),
  m64n64k16 and m64n128k16 over four K steps from non-zero accumulators.  The 128 x 64 tile and the 64 x 256 tile rest on that.
- The layer, through hd_conv_gemm with real descriptors, in 'tc3h' and 'tc1h', at 224 and at a size with a ragged last tile: the
  tile is taken (hd_conv_gemm_profile reports it), the output matches a float64 restatement at the bar of the other conv tests,
  nothing past row M is written, and the first image's output is bit-identical to a one-image launch of the same layer, which runs
  the 128 x 64 tile."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROBE_SRC = r'''
#include "tc_ptx.cuh"
using namespace hd::ptx;

// smem: K-major rows of 64 fp16 (128 bytes), 16-byte piece j of row r at (j ^ (r & 7)) * 16 -- the layout of conv_gemm_tc's tiles
__device__ void fill(uint8_t *dst, const __half *src, int rows) {
  for (int i = threadIdx.x; i < rows * 8; i += blockDim.x) {
    const int r = i >> 3, j = i & 7;
    *reinterpret_cast<uint4 *>(dst + r * 128 + ((j ^ (r & 7)) << 4)) = *reinterpret_cast<const uint4 *>(src + r * 64 + j * 8);
  }
}
// fragment element i of thread t: row 16 (t / 32) + (t % 32) / 4 + 8 ((i % 4) / 2), column 8 (i / 4) + 2 (t % 4) + i % 2
template <int N>
__device__ void frag_io(float (&d)[N / 2], float *g, int ld, bool store) {
  const int t = threadIdx.x;
  for (int i = 0; i < N / 2; ++i) {
    const int r = 16 * (t / 32) + (t % 32) / 4 + 8 * ((i % 4) / 2), c = 8 * (i / 4) + 2 * (t % 4) + i % 2;
    if (store) g[r * ld + c] = d[i]; else d[i] = g[r * ld + c];
  }
}
template <int N, typename F>
__device__ void mma4(float (&d)[N / 2], uint32_t a, uint32_t b, F op) {
  fence_regs(d);
  wgmma_fence();
  for (int k = 0; k < 4; ++k) op(d, make_smem_desc(a) + 2 * k, make_smem_desc(b) + 2 * k);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(d);
}

// Per block (one warpgroup): P [128 x 64] (pixels), W [64 x 64] (channels), accumulators D [128 x 64] (D^T given transposed).
//   normal:  D[64 g .. 64 g + 63, :] += P[64 g ..] W^T    two m64n64k16 x 4 (P as A, W as B)
//   swapped: D^T += W P^T                                   one m64n128k16 x 4 (W as A, P as B), and m64n64k16 over P's first 64 rows
extern "C" __global__ void __launch_bounds__(128) probe(const __half *P, const __half *W, float *Dn, float *Dt, float *Dt64) {
  extern __shared__ uint8_t raw[];
  uint8_t *sm = raw + ((1024 - (smem_u32(raw) & 1023u)) & 1023u);
  P += blockIdx.x * 128 * 64; W += blockIdx.x * 64 * 64;
  Dn += blockIdx.x * 128 * 64; Dt += blockIdx.x * 64 * 128; Dt64 += blockIdx.x * 64 * 64;
  fill(sm, P, 128);
  fill(sm + 128 * 128, W, 64);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const uint32_t sp = smem_u32(sm), sw = sp + 128 * 128;
  for (int g = 0; g < 2; ++g) {
    float d[32];
    frag_io<64>(d, Dn + 64 * g * 64, 64, false);
    mma4<64>(d, sp + 64 * g * 128, sw, [](float (&x)[32], uint64_t a, uint64_t b) { wgmma_m64n64k16_f16(x, a, b, 1u); });
    frag_io<64>(d, Dn + 64 * g * 64, 64, true);
  }
  float t[64];
  frag_io<128>(t, Dt, 128, false);
  mma4<128>(t, sw, sp, [](float (&x)[64], uint64_t a, uint64_t b) { wgmma_m64n128k16_f16(x, a, b, 1u); });
  frag_io<128>(t, Dt, 128, true);
  float u[32];
  frag_io<64>(u, Dt64, 64, false);
  mma4<64>(u, sw, sp, [](float (&x)[32], uint64_t a, uint64_t b) { wgmma_m64n64k16_f16(x, a, b, 1u); });
  frag_io<64>(u, Dt64, 64, true);
}
'''


def _probe_lib(tmp_path):
    src = tmp_path / 'probe.cu'
    src.write_text(PROBE_SRC)
    cubin = tmp_path / 'probe.cubin'
    subprocess.check_call(['/usr/local/cuda/bin/nvcc', '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-cubin',
                           '-I', os.path.join(ROOT, 'human_dynamics_b200', 'csrc'), '-o', str(cubin), str(src)])
    return cubin


def test_wgmma_operand_swap_is_bit_identical(tmp_path):
    cubin = _probe_lib(tmp_path)
    cuda = C.CDLL('libcuda.so.1')
    torch.cuda.init()
    torch.zeros(1, device='cuda')                          # the primary context, current on this thread
    mod, fn = C.c_void_p(), C.c_void_p()
    assert cuda.cuModuleLoad(C.byref(mod), str(cubin).encode()) == 0
    assert cuda.cuModuleGetFunction(C.byref(fn), mod, b'probe') == 0
    smem = 128 * 128 + 64 * 128 + 1024
    assert cuda.cuFuncSetAttribute(fn, 8, smem) == 0       # CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES
    blocks = 96
    rng = np.random.RandomState(5)
    # operands over many binades (and some exact zeros), accumulators of every sign and of several magnitudes
    P = (rng.normal(0, 1, (blocks, 128, 64)) * 2.0 ** rng.randint(-12, 6, (blocks, 128, 64))).astype(np.float16)
    W = (rng.normal(0, 1, (blocks, 64, 64)) * 2.0 ** rng.randint(-12, 6, (blocks, 64, 64))).astype(np.float16)
    P[rng.uniform(size=P.shape) < 0.05] = 0
    D = (rng.normal(0, 1, (blocks, 128, 64)) * 2.0 ** rng.randint(-20, 12, (blocks, 128, 64))).astype(np.float32)
    dev = torch.device('cuda')
    tP, tW = torch.from_numpy(P).to(dev), torch.from_numpy(W).to(dev)
    Dn = torch.from_numpy(D).to(dev)
    Dt = torch.from_numpy(np.ascontiguousarray(D.transpose(0, 2, 1))).to(dev)
    Dt64 = torch.from_numpy(np.ascontiguousarray(D[:, :64].transpose(0, 2, 1))).to(dev)
    args = [C.c_void_p(t.data_ptr()) for t in (tP, tW, Dn, Dt, Dt64)]
    argv = (C.c_void_p * 5)(*[C.cast(C.pointer(a), C.c_void_p) for a in args])
    torch.cuda.synchronize()
    assert cuda.cuLaunchKernel(fn, blocks, 1, 1, 128, 1, 1, smem, None, argv, None) == 0
    torch.cuda.synchronize()
    n, t, t64 = Dn.cpu().numpy(), Dt.cpu().numpy().transpose(0, 2, 1), Dt64.cpu().numpy().transpose(0, 2, 1)
    cuda.cuModuleUnload(mod)
    ref = D.astype(np.float64) + np.einsum('bpk,bck->bpc', P.astype(np.float64), W.astype(np.float64))
    assert np.abs(n - ref).max() <= 1e-5 * np.abs(ref).max()          # the probe computed the products at all
    diff = n.view(np.uint32) != t.view(np.uint32)
    assert not diff.any(), 'm64n128k16 swapped differs from m64n64k16 in %d of %d elements' % (diff.sum(), diff.size)
    diff64 = n[:, :64].view(np.uint32) != t64.view(np.uint32)
    assert not diff64.any(), 'm64n64k16 swapped differs in %d of %d elements' % (diff64.sum(), diff64.size)


def rel_err(a, b):
    b = np.asarray(b, np.float64)
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


def _f16(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def _tile(op):
    """(pixels, channels) of the tile the layer's kernel runs, from hd_conv_gemm_profile; the profiled launch is a normal one too."""
    from human_dynamics_b200._lib import lib, check
    dbg = torch.zeros(16, dtype=torch.int64, device='cuda')
    check(lib.hd_conv_gemm_profile(op.ref, torch.cuda.current_stream().cuda_stream, C.c_void_p(dbg.data_ptr())), 'hd_conv_gemm_profile')
    torch.cuda.synchronize()
    return int(dbg[7]), int(dbg[8])


@pytest.mark.parametrize('impl', ['tc3h', 'tc1h'])
@pytest.mark.parametrize('n,size', [(2, 224), (3, 200)])
def test_root_conv1_planes_cout64(n, size, impl):
    from human_dynamics_b200 import nets
    from human_dynamics_b200._lib import lib, check, fptr
    rng = np.random.RandomState(n * 1000 + size)
    dev = torch.device('cuda')
    x = rng.uniform(-1, 1, size=(n, size, size, 3)).astype(np.float32)
    w = (rng.normal(0, 1, size=(7, 7, 3, 64)) / np.sqrt(147)).astype(np.float32)
    if impl == 'tc1h':
        x, w = _f16(x), _f16(w)
    b = rng.normal(0, 0.2, size=64).astype(np.float32)
    pc = nets.PackedConv1Planes(w, b, dev)
    st = torch.cuda.current_stream().cuda_stream
    Ho = size // 2
    M, extra = n * Ho * Ho, 29

    def run(nn):
        planes = pc.alloc_planes(nn, size, impl)
        out = torch.full((nn * Ho * Ho + extra, 64), float('nan'), device=dev)
        op = pc.bind(planes, nn, size, out, impl=impl)
        xt = torch.from_numpy(x[:nn]).to(dev)
        check(lib.hd_pack_conv1_planes(fptr(xt), C.c_void_p(planes[0].data_ptr()),
                                       C.c_void_p(planes[1].data_ptr() if planes[1] is not None else None), nn, size, size,
                                       planes[0].shape[2], st), 'pack')
        tile = _tile(op)
        return tile, out.cpu().numpy()

    tile, out = run(n)
    tile1, out1 = run(1)
    assert M % 256 != 0 or size == 224
    assert tile == (256, 64), tile
    assert tile1 == (128, 64), tile1
    assert np.isnan(out[M:]).all() and not np.isnan(out[:M]).any()
    ac = F.pad(torch.from_numpy(x).double().permute(0, 3, 1, 2), (3, 3, 3, 3))
    y = F.conv2d(ac, torch.from_numpy(w).double().permute(3, 2, 0, 1), stride=2).permute(0, 2, 3, 1) + torch.from_numpy(b).double()
    assert rel_err(out[:M], y.reshape(M, 64).numpy()) < 2e-5
    m1 = Ho * Ho
    assert np.array_equal(out[:m1].view(np.uint32), out1[:m1].view(np.uint32))
