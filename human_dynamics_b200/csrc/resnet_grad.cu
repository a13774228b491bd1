// Backward of the training-mode ResNet trunk (slim resnet_v2_50 with is_training=True): the convolutions' weight gradients, the
// training-mode batch norm + ReLU backward, pool1's backward and the zero-insertion that turns the data gradient of a stride-2 3x3 conv
// into a stride-1 conv for hd_conv_gemm.  The other data gradients are hd_conv_gemm itself (3xTF32, in = dY) over
// hd_pack_weight(HD_PACK_BACKWARD_DATA).
//
// Nothing here uses atomics: every sum runs over a partition that depends only on the shapes, and partials are merged in a fixed order,
// so results are bit-identical from run to run and do not depend on the GPU's SM count.
#include <cuda_runtime.h>
#include <stdint.h>
#include "common.cuh"
#include "tc_ptx.cuh"

namespace {

// ------------------------------------------------------------------------------------------------------------------------------------
// hd_conv_wgrad: dW[(ky,kx,ci), co] = sum_p a[p, (ky,kx,ci)] * dY[p, co] as an implicit GEMM, M = KH*KW*Cin, N = Cout, reduced over the
// pixels p in chunks of kChunk.  A CTA owns a 64 x 64 tile of dW and one chunk, and is split into two warpgroups:
//   producer  gathers 32 pixels of A (from the input, the prologue applied) and of dY per stage, splits every value into a TF32 head and
//             remainder in registers and writes the four 64-row x 128-byte tiles (A hi / lo, dY hi / lo, both K-major: the pixels are
//             the GEMM's K) in the 128-byte swizzle wgmma reads; kStages stages in flight on full / empty mbarriers.  The CTAs of the
//             first M tile also sum the dY values they load per column in fp64: the bias gradient, without a padding tile.
//   consumer  per stage, 4 K steps of wgmma m64n64k8 in the 3xTF32 split (a_lo b_hi + a_hi b_lo + a_hi b_hi: gradients have an
//             arbitrary scale, so no fp16 operand).  The tensor cores' own fp32 accumulation does not round to nearest, so each stage
//             is accumulated from zero and added to the running sums with ordinary round-to-nearest adds.
// Tile partials go to the workspace [chunks, K + bias, Cout] and wgrad_merge_kernel adds them in chunk order in fp64.
// ------------------------------------------------------------------------------------------------------------------------------------
constexpr int kChunk = 2048;           // pixels per partial sum: fixed, so the rounding depends on the shapes alone
constexpr int kBM = 64, kBN = 64, kBP = 32;
constexpr int kStages = 3;
constexpr int kTileBytes = 64 * 128;                  // 64 rows x one 128-byte swizzle row (32 tf32 pixels)
constexpr int kStageBytes = 4 * kTileBytes;           // A hi, A lo, dY hi, dY lo
constexpr int kWgradSmem = kStages * kStageBytes + 1024;
constexpr int kWgradThreads = 256;

struct WgradArgs {
  const float *x;
  long long x_ld;
  int n_img, H, W, Cin, Ho, Wo, KH, KW, stride, pad_t, pad_l;
  const float *pre_scale, *pre_shift;
  const float *dy;
  long long dy_ld;
  int Cout, K, M;                      // M = K + 1 with a bias row (in the workspace only)
  long long P;                         // pixels = n_img * Ho * Wo
  int vec;                             // Cin, Cout, x_ld, dy_ld % 4 == 0 and 16-byte aligned x / dy: float4 gathers
  float *part;                         // [chunks, M, Cout]
};

__device__ __forceinline__ void split4(const float *v, uint4 &hi, uint4 &lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float hf = hd::ptx::rn_tf32(v[e]);
    h[e] = __float_as_uint(hf);
    l[e] = __float_as_uint(hd::ptx::rn_tf32(v[e] - hf));
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

__global__ void __launch_bounds__(kWgradThreads, 2) wgrad_kernel(const WgradArgs a) {
  namespace P = hd::ptx;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kStages], empty_bar[kStages];
  __shared__ int pix_n[kBP], pix_y[kBP], pix_x[kBP];       // per staged pixel: image, top-left input row / column (n = -1: past the chunk)
  __shared__ double bias_sh[128][4];
  const uint32_t base = (P::smem_u32(smem_raw) + 1023u) & ~1023u;      // wgmma's swizzle atoms are 1024-byte aligned
  uint8_t *smem = smem_raw + (base - P::smem_u32(smem_raw));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.z * kBN;
  const long long p_begin = (long long)blockIdx.x * kChunk;
  const long long p_end = p_begin + kChunk < a.P ? p_begin + kChunk : a.P;
  const int steps = (int)((p_end - p_begin + kBP - 1) / kBP);
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      P::mbar_init(P::smem_u32(&full_bar[s]), 4);          // one arrive per producer warp
      P::mbar_init(P::smem_u32(&empty_bar[s]), 4);         // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= 4) {
    // =============================== producer warpgroup ===============================
    const int t = tid - 128;
    const int r = t & 63, jg = t >> 6;                     // tile row r (A: k index m0 + r; dY: column n0 + r), 16-byte pieces jg + 2i
    const int k = m0 + r;
    int ky = 0, kx = 0, ci = 0;
    const bool krow = k < a.K;
    if (krow) {
      ci = k % a.Cin;
      const int kk = k / a.Cin;
      kx = kk % a.KW;
      ky = kk / a.KW;
    }
    const bool pro = a.pre_scale != nullptr && krow;
    const float sc = pro ? __ldg(a.pre_scale + ci) : 1.f, sh = pro ? __ldg(a.pre_shift + ci) : 0.f;
    const int co = n0 + r;
    const bool co_ok = co < a.Cout;
    const bool bias = a.M > a.K && blockIdx.y == 0;
    double bsum = 0.;
    // the float4 path's role: row group vrg (rows / columns 4 vrg .. 4 vrg + 3), piece vj
    const int vj = t & 7, vrg = t >> 3;
    const int vk = m0 + 4 * vrg;
    const bool vkrow = a.vec && vk < a.K;
    int vky = 0, vkx = 0, vci = 0;
    float vsc[4] = {1.f, 1.f, 1.f, 1.f}, vsh[4] = {0.f, 0.f, 0.f, 0.f};
    if (vkrow) {
      vci = vk % a.Cin;
      const int kk = vk / a.Cin;
      vkx = kk % a.KW;
      vky = kk / a.KW;
      if (a.pre_scale)
        for (int c4 = 0; c4 < 4; ++c4) { vsc[c4] = __ldg(a.pre_scale + vci + c4); vsh[c4] = __ldg(a.pre_shift + vci + c4); }
    }
    const int vco = n0 + 4 * vrg;
    const bool vco_ok = vco < a.Cout;
    double vbsum[4] = {0., 0., 0., 0.};
    for (int q = 0; q < steps; ++q) {
      const int s = q % kStages;
      const long long p0 = p_begin + (long long)q * kBP;
      P::named_bar_sync(1, 128);                             // every producer has read the previous step's pixels
      if (t < kBP) {
        const long long p = p0 + t;
        if (p < p_end) {
          const int pi = (int)p;                                   // P < 2^31 (checked on the host)
          const int ox = pi % a.Wo, qq = pi / a.Wo;
          pix_x[t] = ox * a.stride - a.pad_l;
          pix_y[t] = (qq % a.Ho) * a.stride - a.pad_t;
          pix_n[t] = qq / a.Ho;
        } else {
          pix_n[t] = -1;
        }
      }
      P::named_bar_sync(1, 128);
      if (q >= kStages) P::mbar_wait(P::smem_u32(&empty_bar[s]), (uint32_t)((q / kStages) - 1) & 1u);
      uint8_t *st = smem + s * kStageBytes;
      if (a.vec) {
        // float4 gathers: thread (row group rg, piece j) loads channels 4rg .. 4rg + 3 of A's and dY's rows at pixels 4j .. 4j + 3 and
        // transposes them in registers into four K-major 16-byte pieces per tile (lanes cover all 8 swizzle slots: no extra conflicts)
        float av[4][4], bv[4][4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int pr = 4 * vj + e;
          const int nn = pix_n[pr];
          float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
          if (nn >= 0) {
            if (vkrow) {
              const int iy = pix_y[pr] + vky, ix = pix_x[pr] + vkx;
              if (iy >= 0 && iy < a.H && ix >= 0 && ix < a.W) {
                va = __ldg(reinterpret_cast<const float4 *>(a.x + ((nn * a.H + iy) * (long long)a.W + ix) * a.x_ld + vci));
                if (a.pre_scale) {
                  va.x = fmaxf(__fmaf_rn(va.x, vsc[0], vsh[0]), 0.f); va.y = fmaxf(__fmaf_rn(va.y, vsc[1], vsh[1]), 0.f);
                  va.z = fmaxf(__fmaf_rn(va.z, vsc[2], vsh[2]), 0.f); va.w = fmaxf(__fmaf_rn(va.w, vsc[3], vsh[3]), 0.f);
                }
              }
            }
            if (vco_ok) vb = __ldg(reinterpret_cast<const float4 *>(a.dy + (p0 + pr) * a.dy_ld + vco));
          }
          av[0][e] = va.x; av[1][e] = va.y; av[2][e] = va.z; av[3][e] = va.w;
          bv[0][e] = vb.x; bv[1][e] = vb.y; bv[2][e] = vb.z; bv[3][e] = vb.w;
        }
#pragma unroll
        for (int c4 = 0; c4 < 4; ++c4) {
          const int rr = 4 * vrg + c4;
          const uint32_t off = (uint32_t)rr * 128u + ((uint32_t)(vj ^ (rr & 7)) << 4);
          uint4 h, l;
          split4(av[c4], h, l);
          *reinterpret_cast<uint4 *>(st + off) = h;
          *reinterpret_cast<uint4 *>(st + kTileBytes + off) = l;
          split4(bv[c4], h, l);
          *reinterpret_cast<uint4 *>(st + 2 * kTileBytes + off) = h;
          *reinterpret_cast<uint4 *>(st + 3 * kTileBytes + off) = l;
          if (bias) vbsum[c4] += ((double)bv[c4][0] + (double)bv[c4][1]) + ((double)bv[c4][2] + (double)bv[c4][3]);
        }
      } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = jg + 2 * i;                          // pixels 4j .. 4j + 3 of the step
        float av[4], bv[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int pr = 4 * j + e;
          const int nn = pix_n[pr];
          av[e] = 0.f;
          bv[e] = 0.f;
          if (nn >= 0) {
            if (krow) {
              const int iy = pix_y[pr] + ky, ix = pix_x[pr] + kx;
              if (iy >= 0 && iy < a.H && ix >= 0 && ix < a.W) {
                float v = __ldg(a.x + (((long long)nn * a.H + iy) * a.W + ix) * a.x_ld + ci);
                if (pro) v = fmaxf(__fmaf_rn(v, sc, sh), 0.f);      // hd_conv_gemm's prologue; padding stays 0
                av[e] = v;
              }
            }
            if (co_ok) bv[e] = __ldg(a.dy + (p0 + pr) * a.dy_ld + co);
          }
        }
        if (bias) {
#pragma unroll
          for (int e = 0; e < 4; ++e) bsum += (double)bv[e];
        }
        const uint32_t off = (uint32_t)r * 128u + ((uint32_t)(j ^ (r & 7)) << 4);
        uint4 h, l;
        split4(av, h, l);
        *reinterpret_cast<uint4 *>(st + off) = h;
        *reinterpret_cast<uint4 *>(st + kTileBytes + off) = l;
        split4(bv, h, l);
        *reinterpret_cast<uint4 *>(st + 2 * kTileBytes + off) = h;
        *reinterpret_cast<uint4 *>(st + 3 * kTileBytes + off) = l;
      }
      }
      P::fence_proxy_async();                                // generic-proxy stores -> visible to wgmma (async proxy)
      __syncwarp();
      if (lane == 0) P::mbar_arrive(P::smem_u32(&full_bar[s]));
    }
    if (bias) {                                              // the bias row of this chunk's partial: the threads of a column, in order
      if (a.vec) {
        for (int c4 = 0; c4 < 4; ++c4) bias_sh[t][c4] = vbsum[c4];
      } else {
        bias_sh[t][0] = bsum;
      }
      P::named_bar_sync(1, 128);
      if (a.vec) {
        if (t < 64 && n0 + t < a.Cout) {
          const int rg = t >> 2, c4 = t & 3;
          double v = 0.;
          for (int j = 0; j < 8; ++j) v += bias_sh[rg * 8 + j][c4];
          a.part[((size_t)blockIdx.x * a.M + a.K) * a.Cout + n0 + t] = (float)v;
        }
      } else if (t < 64 && co_ok) {
        a.part[((size_t)blockIdx.x * a.M + a.K) * a.Cout + co] = (float)(bias_sh[t][0] + bias_sh[t + 64][0]);
      }
    }
  } else {
    // =============================== consumer warpgroup ===============================
    float acc[32], tmp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    for (int q = 0; q < steps; ++q) {
      const int s = q % kStages;
      P::mbar_wait(P::smem_u32(&full_bar[s]), (uint32_t)(q / kStages) & 1u);
      const uint32_t sa = base + s * kStageBytes;
      const uint64_t da_hi = P::make_smem_desc(sa), da_lo = P::make_smem_desc(sa + kTileBytes);
      const uint64_t db_hi = P::make_smem_desc(sa + 2 * kTileBytes), db_lo = P::make_smem_desc(sa + 3 * kTileBytes);
      P::fence_regs(tmp);
      P::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {                       // K = 8 tf32 = 32 bytes per wgmma: advance inside the swizzle row
        const uint64_t adv = (uint64_t)((kk * 32) >> 4);
        P::wgmma_m64n64k8_tf32(tmp, da_lo + adv, db_hi + adv, kk != 0);     // small products first, then the head product
        P::wgmma_m64n64k8_tf32(tmp, da_hi + adv, db_lo + adv, 1u);
        P::wgmma_m64n64k8_tf32(tmp, da_hi + adv, db_hi + adv, 1u);
      }
      P::wgmma_commit();
      P::wgmma_wait<0>();
      P::fence_regs(tmp);
      __syncwarp();
      if (lane == 0) P::mbar_arrive(P::smem_u32(&empty_bar[s]));
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] += tmp[i];       // round-to-nearest fp32 adds
    }
    float *dst = a.part + (size_t)blockIdx.x * a.M * a.Cout;
    const int row = m0 + 16 * warp + (lane >> 2);
#pragma unroll
    for (int jn = 0; jn < 8; ++jn)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int m = row + (e >= 2 ? 8 : 0);
        const int n = n0 + 8 * jn + 2 * (lane & 3) + (e & 1);
        if (m < a.K && n < a.Cout) dst[(size_t)m * a.Cout + n] = acc[4 * jn + e];
      }
  }
}

// out[m, co] = sum over the chunks, in chunk order, in fp64; row K (when there is a bias row) goes to db.
__global__ void wgrad_merge_kernel(const float *__restrict__ part, int chunks, int K, int M, int Cout, float *__restrict__ dw,
                                   float *__restrict__ db) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long MN = (long long)M * Cout;
  if (i >= MN) return;
  double s = 0.;
  int j = 0;
  for (; j + 4 <= chunks; j += 4) {
    const float v0 = __ldg(part + (size_t)j * MN + i), v1 = __ldg(part + (size_t)(j + 1) * MN + i),
                v2 = __ldg(part + (size_t)(j + 2) * MN + i), v3 = __ldg(part + (size_t)(j + 3) * MN + i);
    s += (double)v0;
    s += (double)v1;
    s += (double)v2;
    s += (double)v3;
  }
  for (; j < chunks; ++j) s += (double)__ldg(part + (size_t)j * MN + i);
  const int m = (int)(i / Cout), co = (int)(i % Cout);
  if (m < K)
    dw[i] = (float)s;
  else
    db[co] = (float)s;
}

// ------------------------------------------------------------------------------------------------------------------------------------
// hd_bn_relu_backward.  Per channel, with z = fma(x, scale, shift) (the forward's pre-activation, as the conv prologue computes it),
// g = dz * (z > 0), d = x - x[row 0]:
//   pass 1 (bnb_partial_kernel): fixed chunks of rows sum d, g and g*d in fp64 (the stats kernel's chunking);
//   pass 2 (bnb_finish_kernel): the chunks in order -> exact fp64 batch mean, dbeta = sum g, dgamma = rstd * sum g (x - mean);
//   pass 3 (bnb_apply_kernel): dx = gamma * rstd * (g - mean(g) - xhat * mean(g xhat)) + addend, element-wise in fp64.
// ------------------------------------------------------------------------------------------------------------------------------------
constexpr int kBnThreads = 256;
constexpr int kBnColGroup = 64;        // float4 columns per block of pass 1
constexpr int kBnLanes = 16;

struct BnGeometry {
  int C4, cw, rl, groups, chunks;
  long long chunk_rows;
};

BnGeometry bn_geometry(long long rows, int C) {
  BnGeometry g;
  g.C4 = C / 4;
  g.cw = g.C4 < kBnColGroup ? g.C4 : kBnColGroup;
  g.rl = kBnThreads / g.cw;
  g.groups = (g.C4 + g.cw - 1) / g.cw;
  const long long most = (rows + 4LL * g.rl - 1) / (4LL * g.rl);
  long long want = 2048 / g.groups;
  if (want < 1) want = 1;
  const long long chunks = most < want ? most : want;
  g.chunk_rows = (rows + chunks - 1) / chunks;
  g.chunks = (int)((rows + g.chunk_rows - 1) / g.chunk_rows);
  return g;
}

struct BnArgs {
  const float *x, *dz, *scale, *shift, *var, *gamma, *addend;
  long long rows;
  int C, dz_group;
  float eps;
  int add_H, add_W, add_stride;
  float *dx, *dgamma, *dbeta;
  double4 *part;                       // [chunks, C]: (sum d, sum g, sum g d, 0)
  double4 *coef;                       // [C]: (mean, rstd, mean g, mean g xhat)
};

__device__ __forceinline__ float upstream(const BnArgs &a, long long r, int c) {
  if (a.dz_group <= 1) return __ldg(a.dz + r * a.C + c);
  return __fdiv_rn(__ldg(a.dz + (r / a.dz_group) * a.C + c), (float)a.dz_group);    // d mean over the group of rows
}

__global__ void __launch_bounds__(kBnThreads) bnb_partial_kernel(const BnArgs a, int C4, int cw, int rl, long long chunk_rows) {
  __shared__ double sh[kBnThreads][12];
  const int t = threadIdx.x, cl = t % cw, r = t / cw;
  const int c4 = blockIdx.y * cw + cl;
  const bool active = r < rl && c4 < C4;
  const long long r0 = (long long)blockIdx.x * chunk_rows;
  const long long r1 = r0 + chunk_rows < a.rows ? r0 + chunk_rows : a.rows;
  double s[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) s[k] = 0.;
  if (active) {
    float piv[4], sc[4], sf[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      piv[k] = __ldg(a.x + 4 * c4 + k);
      sc[k] = __ldg(a.scale + 4 * c4 + k);
      sf[k] = __ldg(a.shift + 4 * c4 + k);
    }
    for (long long i = r0 + r; i < r1; i += rl) {
      const float4 v = __ldg(reinterpret_cast<const float4 *>(a.x + i * a.C) + c4);
      const float xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float z = __fmaf_rn(xv[k], sc[k], sf[k]);
        const double gk = z > 0.f ? (double)upstream(a, i, 4 * c4 + k) : 0.;
        const double d = (double)xv[k] - (double)piv[k];
        s[3 * k] += d;
        s[3 * k + 1] += gk;
        s[3 * k + 2] = fma(gk, d, s[3 * k + 2]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 12; ++k) sh[t][k] = s[k];
  __syncthreads();
  if (r == 0 && c4 < C4) {
    for (int j = 1; j < rl; ++j)
#pragma unroll
      for (int k = 0; k < 12; ++k) s[k] += sh[j * cw + cl][k];
    double4 *dst = a.part + (size_t)blockIdx.x * a.C + 4 * (size_t)c4;
#pragma unroll
    for (int k = 0; k < 4; ++k) dst[k] = make_double4(s[3 * k], s[3 * k + 1], s[3 * k + 2], 0.);
  }
}

__global__ void __launch_bounds__(32 * kBnLanes) bnb_finish_kernel(const BnArgs a, int chunks) {
  __shared__ double sh[3][kBnLanes][32];
  const int cl = threadIdx.x & 31, lane = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  double sd = 0., sg = 0., sgd = 0.;
  if (c < a.C) {
    for (int j = lane; j < chunks; j += kBnLanes) {
      const double4 p = a.part[(size_t)j * a.C + c];
      sd += p.x;
      sg += p.y;
      sgd += p.z;
    }
  }
  sh[0][lane][cl] = sd;
  sh[1][lane][cl] = sg;
  sh[2][lane][cl] = sgd;
  __syncthreads();
  if (lane != 0 || c >= a.C) return;
  for (int j = 1; j < kBnLanes; ++j) {
    sd += sh[0][j][cl];
    sg += sh[1][j][cl];
    sgd += sh[2][j][cl];
  }
  const double n = (double)a.rows;
  const double dm = sd / n;                                  // mean - x[row 0]
  const double rstd = 1. / sqrt((double)__ldg(a.var + c) + (double)a.eps);
  const double sgx = rstd * (sgd - dm * sg);                 // sum g * xhat
  a.dbeta[c] = (float)sg;
  a.dgamma[c] = (float)sgx;
  a.coef[c] = make_double4((double)__ldg(a.x + c) + dm, rstd, sg / n, sgx / n);
}

__global__ void bnb_apply_kernel(const BnArgs a) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.rows * a.C) return;
  const int c = (int)(i % a.C);
  const long long r = i / a.C;
  const float xv = __ldg(a.x + i);
  const float z = __fmaf_rn(xv, __ldg(a.scale + c), __ldg(a.shift + c));
  const double gk = z > 0.f ? (double)upstream(a, r, c) : 0.;
  const double4 k = a.coef[c];
  const double xhat = ((double)xv - k.x) * k.y;
  double v = (double)__ldg(a.gamma + c) * k.y * (gk - k.z - xhat * k.w);
  float out = (float)v;
  if (a.addend) {
    if (a.add_stride <= 1) {
      out += __ldg(a.addend + i);
    } else {
      const int s = a.add_stride;
      const int ix = (int)(r % a.add_W);
      const long long q = r / a.add_W;
      const int iy = (int)(q % a.add_H);
      const long long nn = q / a.add_H;
      if (iy % s == 0 && ix % s == 0) {
        const int Hs = (a.add_H + s - 1) / s, Ws = (a.add_W + s - 1) / s;
        out += __ldg(a.addend + ((nn * Hs + iy / s) * Ws + ix / s) * a.C + c);
      }
    }
  }
  a.dx[i] = out;
}

// ------------------------------------------------------------------------------------------------------------------------------------
// pool1 backward (3x3, stride 2, SAME) as a gather: each input pixel adds, in window order, the upstream gradient of every window whose
// first maximum (scan order ky, kx) it is.
// ------------------------------------------------------------------------------------------------------------------------------------
__global__ void maxpool_backward_kernel(const float *__restrict__ in, const float *__restrict__ dout, float *__restrict__ din, int N, int H,
                                        int W, int C, int Ho, int Wo, int pt, int pl) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * H * W * C) return;
  const int c = (int)(i % C);
  long long q = i / C;
  const int ix = (int)(q % W);
  q /= W;
  const int iy = (int)(q % H);
  const int n = (int)(q / H);
  const float *img = in + (size_t)n * H * W * C + c;
  float acc = 0.f;
  const int oy_lo = (iy + pt - 2 + 1) >= 0 ? (iy + pt - 1) / 2 : 0;     // ceil((iy + pt - 2) / 2), clamped at 0
  const int oy_hi = min((iy + pt) / 2, Ho - 1);
  const int ox_lo = (ix + pl - 2 + 1) >= 0 ? (ix + pl - 1) / 2 : 0;
  const int ox_hi = min((ix + pl) / 2, Wo - 1);
  for (int oy = oy_lo; oy <= oy_hi; ++oy)
    for (int ox = ox_lo; ox <= ox_hi; ++ox) {
      int by = -1, bx = -1;
      float best = 0.f;
      for (int ky = 0; ky < 3; ++ky) {
        const int y = 2 * oy - pt + ky;
        if (y < 0 || y >= H) continue;
        for (int kx = 0; kx < 3; ++kx) {
          const int x = 2 * ox - pl + kx;
          if (x < 0 || x >= W) continue;
          const float v = __ldg(img + ((size_t)y * W + x) * C);
          if (by < 0 || v > best) { best = v; by = y; bx = x; }
        }
      }
      if (by == iy && bx == ix) acc += __ldg(dout + (((size_t)n * Ho + oy) * Wo + ox) * C + c);
    }
  din[i] = acc;
}

// out[n, y, x, c] = in[n, y / s, x / s, c] where y % s == 0 and x % s == 0, else 0
__global__ void zero_insert_kernel(const float *__restrict__ in, float *__restrict__ out, int N, int Hi, int Wi, int C, int s, int Ho, int Wo) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * Ho * Wo * C) return;
  const int c = (int)(i % C);
  long long q = i / C;
  const int x = (int)(q % Wo);
  q /= Wo;
  const int y = (int)(q % Ho);
  const long long n = q / Ho;
  float v = 0.f;
  if (y % s == 0 && x % s == 0 && y / s < Hi && x / s < Wi) v = __ldg(in + ((n * Hi + y / s) * Wi + x / s) * C + c);
  out[i] = v;
}

inline bool aligned16(const void *p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace

extern "C" size_t hd_conv_wgrad_workspace_bytes(long long pixels, int K, int Cout, int bias) {
  if (pixels <= 0 || K <= 0 || Cout <= 0) return 0;
  const long long chunks = (pixels + kChunk - 1) / kChunk;
  return (size_t)chunks * (size_t)(K + (bias ? 1 : 0)) * (size_t)Cout * sizeof(float);
}

extern "C" int hd_conv_wgrad(const float *x, long long x_ld, int n_img, int H, int W, int Cin, int Ho, int Wo, int KH, int KW, int stride,
                             int pad_t, int pad_l, const float *pre_scale, const float *pre_shift, const float *dy, long long dy_ld, int Cout,
                             float *dw, float *db, void *workspace, size_t workspace_bytes, void *stream) {
  HD_REQUIRE(x && dy && dw && workspace, "hd_conv_wgrad: null pointer");
  HD_REQUIRE(n_img > 0 && H > 0 && W > 0 && Cin > 0 && Ho > 0 && Wo > 0 && KH > 0 && KW > 0 && stride > 0 && Cout > 0 && pad_t >= 0 &&
                 pad_l >= 0 && x_ld >= Cin && dy_ld >= Cout,
             "hd_conv_wgrad: bad geometry (positive sizes, x_ld >= Cin, dy_ld >= Cout)");
  HD_REQUIRE((pre_scale == nullptr) == (pre_shift == nullptr), "hd_conv_wgrad: pre_scale and pre_shift go together");
  HD_REQUIRE((long long)(Ho - 1) * stride - pad_t < H && (long long)(Wo - 1) * stride - pad_l < W,
             "hd_conv_wgrad: output pixels past the input");
  const long long P = (long long)n_img * Ho * Wo;
  const int K = KH * KW * Cin;
  HD_REQUIRE(P < (1LL << 31) && (long long)KH * KW * Cin < (1LL << 24), "hd_conv_wgrad: problem too large");
  HD_REQUIRE(workspace_bytes >= hd_conv_wgrad_workspace_bytes(P, K, Cout, db != nullptr), "hd_conv_wgrad: workspace too small");
  WgradArgs a;
  a.x = x; a.x_ld = x_ld; a.n_img = n_img; a.H = H; a.W = W; a.Cin = Cin; a.Ho = Ho; a.Wo = Wo; a.KH = KH; a.KW = KW;
  a.stride = stride; a.pad_t = pad_t; a.pad_l = pad_l; a.pre_scale = pre_scale; a.pre_shift = pre_shift; a.dy = dy; a.dy_ld = dy_ld;
  a.Cout = Cout; a.K = K; a.M = K + (db ? 1 : 0); a.P = P;
  a.vec = Cin % 4 == 0 && Cout % 4 == 0 && x_ld % 4 == 0 && dy_ld % 4 == 0 && aligned16(x) && aligned16(dy);
  a.part = reinterpret_cast<float *>(workspace);
  const int chunks = (int)((P + kChunk - 1) / kChunk);
  cudaStream_t st = (cudaStream_t)stream;
  static bool smem_set = false;               // (benign race: every caller sets the same value)
  if (!smem_set) {
    const cudaError_t e = cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgradSmem);
    if (e != cudaSuccess) {
      hd::set_last_error("hd_conv_wgrad: cudaFuncSetAttribute", e);
      return HD_ERR_CUDA;
    }
    smem_set = true;
  }
  wgrad_kernel<<<dim3(chunks, hd::ceil_div(K, kBM), hd::ceil_div(Cout, kBN)), kWgradThreads, kWgradSmem, st>>>(a);
  int rc = hd::check_launch("wgrad_kernel");
  if (rc) return rc;
  wgrad_merge_kernel<<<hd::ceil_div((long long)a.M * Cout, 256), 256, 0, st>>>(a.part, chunks, K, a.M, Cout, dw, db);
  return hd::check_launch("wgrad_merge_kernel");
}

extern "C" size_t hd_bn_relu_backward_workspace_bytes(long long rows, int C) {
  if (rows < 2 || C <= 0 || C % 4 != 0) return 0;
  const BnGeometry g = bn_geometry(rows, C);
  return ((size_t)g.chunks + 1) * (size_t)C * sizeof(double4);
}

extern "C" int hd_bn_relu_backward(const float *x, const float *dz, int dz_group, long long rows, int C, const float *scale,
                                   const float *shift, const float *var, const float *gamma, float eps, const float *addend, int add_H,
                                   int add_W, int add_stride, float *dx, float *dgamma, float *dbeta, void *workspace,
                                   size_t workspace_bytes, void *stream) {
  HD_REQUIRE(x && dz && scale && shift && var && gamma && dx && dgamma && dbeta && workspace, "hd_bn_relu_backward: null pointer");
  HD_REQUIRE(rows >= 2 && C > 0 && C % 4 == 0 && eps >= 0.f && dz_group >= 1 && rows % dz_group == 0,
             "hd_bn_relu_backward: need rows >= 2, C % 4 == 0, eps >= 0, dz_group >= 1 dividing rows");
  HD_REQUIRE(aligned16(x) && aligned16(workspace), "hd_bn_relu_backward: x and workspace must be 16-byte aligned");
  HD_REQUIRE(dx != x && dx != dz && (addend == nullptr || dx != addend), "hd_bn_relu_backward: dx must not alias x, dz or the addend");
  HD_REQUIRE(add_stride <= 1 || (addend && add_H > 0 && add_W > 0 && rows % ((long long)add_H * add_W) == 0),
             "hd_bn_relu_backward: a subsampled addend needs add_H, add_W > 0 dividing rows into frames");
  HD_REQUIRE(workspace_bytes >= hd_bn_relu_backward_workspace_bytes(rows, C), "hd_bn_relu_backward: workspace too small");
  const BnGeometry g = bn_geometry(rows, C);
  BnArgs a;
  a.x = x; a.dz = dz; a.scale = scale; a.shift = shift; a.var = var; a.gamma = gamma; a.addend = addend;
  a.rows = rows; a.C = C; a.dz_group = dz_group; a.eps = eps; a.add_H = add_H; a.add_W = add_W; a.add_stride = add_stride;
  a.dx = dx; a.dgamma = dgamma; a.dbeta = dbeta;
  a.part = reinterpret_cast<double4 *>(workspace);
  a.coef = a.part + (size_t)g.chunks * C;
  cudaStream_t st = (cudaStream_t)stream;
  bnb_partial_kernel<<<dim3(g.chunks, g.groups), kBnThreads, 0, st>>>(a, g.C4, g.cw, g.rl, g.chunk_rows);
  int rc = hd::check_launch("bnb_partial_kernel");
  if (rc) return rc;
  bnb_finish_kernel<<<hd::ceil_div(C, 32), 32 * kBnLanes, 0, st>>>(a, g.chunks);
  rc = hd::check_launch("bnb_finish_kernel");
  if (rc) return rc;
  bnb_apply_kernel<<<hd::ceil_div(rows * C, 256), 256, 0, st>>>(a);
  return hd::check_launch("bnb_apply_kernel");
}

extern "C" int hd_maxpool3x3s2_same_backward(const float *in, const float *dout, float *din, int N, int H, int W, int C, void *stream) {
  HD_REQUIRE(in && dout && din && din != in && din != dout && N > 0 && H > 0 && W > 0 && C > 0,
             "hd_maxpool3x3s2_same_backward: bad arguments (din must not alias in / dout)");
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const int pt = max((Ho - 1) * 2 + 3 - H, 0) / 2, pl = max((Wo - 1) * 2 + 3 - W, 0) / 2;
  maxpool_backward_kernel<<<hd::ceil_div((long long)N * H * W * C, 256), 256, 0, (cudaStream_t)stream>>>(in, dout, din, N, H, W, C, Ho, Wo,
                                                                                                         pt, pl);
  return hd::check_launch("maxpool_backward_kernel");
}

extern "C" int hd_zero_insert(const float *in, float *out, int N, int Hi, int Wi, int C, int stride, int Ho, int Wo, void *stream) {
  HD_REQUIRE(in && out && in != out && N > 0 && Hi > 0 && Wi > 0 && C > 0 && stride >= 1 && Ho > 0 && Wo > 0,
             "hd_zero_insert: bad arguments");
  zero_insert_kernel<<<hd::ceil_div((long long)N * Ho * Wo * C, 256), 256, 0, (cudaStream_t)stream>>>(in, out, N, Hi, Wi, C, stride, Ho,
                                                                                                      Wo);
  return hd::check_launch("zero_insert_kernel");
}
