// FP32 CUDA-core implicit-GEMM convolution / FC with fused prologue + epilogue (see hd_b200.h).
// This is the exact-FP32 path: used for ragged shapes (IEF 85/72-wide heads, K not multiple of 32)
// and as the in-tree cross-check of the wgmma kernel.  128x{128,64}x16 tiles, 8x{8,4} per thread,
// register-prefetch double buffering.
#include "conv_common.cuh"

namespace hd {
namespace {

constexpr int BM = 128, BK = 16, NT = 256;

template <int BN, bool FASTA, bool VECB>
__global__ void __launch_bounds__(NT) conv_gemm_simt_kernel(const ConvParams p) {
  constexpr int TN = BN / 16;            // output columns per thread: 8 or 4
  constexpr int NB4 = (BK * BN / 4) / NT;  // float4 B loads per thread: 2 or 1
  __shared__ __align__(16) float As[2][BK][BM];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int K = p.K;

  // ---- A gather coordinates (fixed per thread) ----
  const int arow = tid & (BM - 1);
  const int akh = tid >> 7;               // 0/1: which 8-wide half of the k chunk
  const int am = m0 + arow;
  const bool avalid = am < p.M;
  int an = 0, aiy0 = 0, aix0 = 0;
  if (avalid) {
    const int hw = p.Ho * p.Wo;
    an = am / hw;
    const int r = am - an * hw;
    const int oy = r / p.Wo, ox = r - oy * p.Wo;
    aiy0 = oy * p.stride - p.pad_t;
    aix0 = ox * p.stride - p.pad_l;
  }
  const float *pre_s = p.pre_scale ? p.pre_scale + (size_t)an * p.pre_img_stride : nullptr;
  const float *pre_b = p.pre_scale ? p.pre_shift + (size_t)an * p.pre_img_stride : nullptr;

  float areg[8];
  float4 breg[NB4];

  auto load_a = [&](int k0) {
    const int kb = k0 + akh * 8;
    if (FASTA) {
#pragma unroll
      for (int j = 0; j < 8; ++j) areg[j] = 0.f;
      if (avalid && kb < K) {
        const int tap = kb / p.Cin, ci = kb - tap * p.Cin;
        const int ky = tap / p.KW, kx = tap - ky * p.KW;
        const int iy = aiy0 + ky, ix = aix0 + kx;
        if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
          const float *src = p.in + ((size_t)((size_t)an * p.H + iy) * p.W + ix) * p.in_ld + ci;
          const float4 v0 = __ldg(reinterpret_cast<const float4 *>(src));
          const float4 v1 = __ldg(reinterpret_cast<const float4 *>(src) + 1);
          areg[0] = v0.x; areg[1] = v0.y; areg[2] = v0.z; areg[3] = v0.w;
          areg[4] = v1.x; areg[5] = v1.y; areg[6] = v1.z; areg[7] = v1.w;
          if (pre_s) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float a = areg[j] * __ldg(pre_s + ci + j) + __ldg(pre_b + ci + j);
              areg[j] = p.pre_relu ? fmaxf(a, 0.f) : a;
            }
          }
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = kb + j;
        float a = 0.f;
        if (avalid && k < K) {
          const int tap = k / p.Cin, ci = k - tap * p.Cin;
          const int ky = tap / p.KW, kx = tap - ky * p.KW;
          const int iy = aiy0 + ky, ix = aix0 + kx;
          if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
            a = __ldg(p.in + ((size_t)((size_t)an * p.H + iy) * p.W + ix) * p.in_ld + ci);
            if (pre_s) {
              a = a * __ldg(pre_s + ci) + __ldg(pre_b + ci);
              a = p.pre_relu ? fmaxf(a, 0.f) : a;
            }
          }
        }
        areg[j] = a;
      }
    }
  };

  auto load_b = [&](int k0) {
#pragma unroll
    for (int i = 0; i < NB4; ++i) {
      const int f = tid + i * NT;             // float4 index within the BK x BN tile
      const int kr = f / (BN / 4), c4 = (f % (BN / 4)) * 4;
      const int k = k0 + kr, co = n0 + c4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k < K) {
        const float *src = p.w_kn + (size_t)k * p.Cout + co;
        if (VECB) {
          if (co < p.Cout) v = __ldg(reinterpret_cast<const float4 *>(src));
        } else {
          if (co + 0 < p.Cout) v.x = __ldg(src + 0);
          if (co + 1 < p.Cout) v.y = __ldg(src + 1);
          if (co + 2 < p.Cout) v.z = __ldg(src + 2);
          if (co + 3 < p.Cout) v.w = __ldg(src + 3);
        }
      }
      breg[i] = v;
    }
  };

  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int j = 0; j < 8; ++j) As[buf][akh * 8 + j][arow] = areg[j];
#pragma unroll
    for (int i = 0; i < NB4; ++i) {
      const int f = tid + i * NT;
      const int kr = f / (BN / 4), c4 = (f % (BN / 4)) * 4;
      *reinterpret_cast<float4 *>(&Bs[buf][kr][c4]) = breg[i];
    }
  };

  const int ty = tid >> 4, tx = tid & 15;
  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = (K + BK - 1) / BK;
  load_a(0);
  load_b(0);
  store_tiles(0);
  __syncthreads();
  for (int it = 0; it < nk; ++it) {
    const int buf = it & 1;
    if (it + 1 < nk) { load_a((it + 1) * BK); load_b((it + 1) * BK); }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][k][64 + ty * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[TN];
      const float4 b0 = *reinterpret_cast<const float4 *>(&Bs[buf][k][tx * 4]);
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
      if (TN == 8) {
        const float4 b1 = *reinterpret_cast<const float4 *>(&Bs[buf][k][(BN / 2) + tx * 4]);
        b[TN - 4] = b1.x; b[TN - 3] = b1.y; b[TN - 2] = b1.z; b[TN - 1] = b1.w;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] += a[i] * b[j];
    }
    if (it + 1 < nk) store_tiles(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue: scale/shift, residual, relu ----
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= p.M) continue;
    size_t res_row = 0;
    if (p.res) {
      const int hw = p.Ho * p.Wo;
      const int n = m / hw;
      const int r = m - n * hw;
      const int oy = r / p.Wo, ox = r - oy * p.Wo;
      res_row = ((size_t)n * p.res_H + (size_t)oy * p.res_stride) * p.res_W + (size_t)ox * p.res_stride;
    }
#pragma unroll
    for (int h = 0; h < TN / 4; ++h) {
      const int co = n0 + (h == 0 ? tx * 4 : (BN / 2) + tx * 4);
      if (co >= p.Cout) continue;
      float v[4] = {acc[i][h * 4 + 0], acc[i][h * 4 + 1], acc[i][h * 4 + 2], acc[i][h * 4 + 3]};
      if (p.vec_out) {
        if (p.post_scale) {
          const float4 s = __ldg(reinterpret_cast<const float4 *>(p.post_scale + co));
          v[0] *= s.x; v[1] *= s.y; v[2] *= s.z; v[3] *= s.w;
        }
        if (p.post_shift) {
          const float4 s = __ldg(reinterpret_cast<const float4 *>(p.post_shift + co));
          v[0] += s.x; v[1] += s.y; v[2] += s.z; v[3] += s.w;
        }
        if (p.res) {
          const float4 r = *reinterpret_cast<const float4 *>(p.res + res_row * p.res_ld + co);
          v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
        }
        if (p.post_relu) {
#pragma unroll
          for (int j = 0; j < 4; ++j) v[j] = fmaxf(v[j], 0.f);
        }
        *reinterpret_cast<float4 *>(p.out + (size_t)m * p.out_ld + co) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (co + j >= p.Cout) continue;
          float x = v[j];
          if (p.post_scale) x *= __ldg(p.post_scale + co + j);
          if (p.post_shift) x += __ldg(p.post_shift + co + j);
          if (p.res) x += p.res[res_row * p.res_ld + co + j];
          if (p.post_relu) x = fmaxf(x, 0.f);
          p.out[(size_t)m * p.out_ld + co + j] = x;
        }
      }
    }
  }
}

template <int BN, bool FASTA, bool VECB>
int launch(const ConvParams &p, cudaStream_t st) {
  dim3 grid(ceil_div(p.M, BM), ceil_div(p.Cout, BN));
  conv_gemm_simt_kernel<BN, FASTA, VECB><<<grid, NT, 0, st>>>(p);
  return check_launch("conv_gemm_simt_kernel");
}

}  // namespace

int launch_conv_simt(const ConvParams &p, cudaStream_t st) {
  if (p.out_sub) {
    set_last_error_text("hd_conv_gemm(simt): out_subsample is only implemented by the tensor-core kernel");
    return HD_ERR_UNSUPPORTED;
  }
  if (!p.w_kn || !p.in || !p.out || p.out_hi) {
    set_last_error_text("hd_conv_gemm(simt): needs w_kn and fp32 in/out (no pre-split activations)");
    return HD_ERR_INVALID;
  }
  const bool fasta = (p.Cin % 8 == 0) && (p.in_ld % 4 == 0) && aligned16(p.in) &&
                     (!p.pre_scale || true);
  const bool vecb = (p.Cout % 4 == 0) && aligned16(p.w_kn);
  const bool wide = p.Cout > 64;
  if (wide) {
    if (fasta) return vecb ? launch<128, true, true>(p, st) : launch<128, true, false>(p, st);
    return vecb ? launch<128, false, true>(p, st) : launch<128, false, false>(p, st);
  }
  if (fasta) return vecb ? launch<64, true, true>(p, st) : launch<64, true, false>(p, st);
  return vecb ? launch<64, false, true>(p, st) : launch<64, false, false>(p, st);
}

}  // namespace hd

static int conv_gemm_impl(const hd_conv_desc *d, void *stream, long long *dbg) {
  hd::ConvParams p;
  int rc = hd::fill_params(d, p);
  if (rc) return rc;
  p.dbg = dbg;
  cudaStream_t st = (cudaStream_t)stream;
  if (d->impl == HD_IMPL_SIMT) return hd::launch_conv_simt(p, st);
  if (d->impl == HD_IMPL_TC_3XTF32 || d->impl == HD_IMPL_TC_1XTF32 || d->impl == HD_IMPL_TC_3XF16 || d->impl == HD_IMPL_TC_1XF16)
    return hd::launch_conv_tc(p, d, st);
  hd::set_last_error_text("hd_conv_gemm: unknown impl");
  return HD_ERR_INVALID;
}

extern "C" int hd_conv_gemm(const hd_conv_desc *d, void *stream) { return conv_gemm_impl(d, stream, nullptr); }

// Same launch, but CTA (0,0) of the tensor-core kernel writes per-role cycle counters to dbg[0..15] (device int64):
// [0] producer loop, [1] producer wait-empty (the B loads are issued by a producer thread, inside this loop),
// [2] consumer loop (wgmma + drains + epilogue), [3] consumer wait-full, [4] epilogue, and of the epilogue: [5] waiting for the
// residual to land in shared memory, [6] waiting for earlier TMA stores to have read a buffer before it is refilled (with the
// warpgroup barriers around those waits); [4] - [5] - [6] is arithmetic, staging and issuing stores.  [7] and [8] are the kernel's tile: pixels x output channels.
extern "C" int hd_conv_gemm_profile(const hd_conv_desc *d, void *stream, long long *dbg) { return conv_gemm_impl(d, stream, dbg); }
