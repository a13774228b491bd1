// Training-mode batch normalisation (slim batch_norm with is_training=True under resnet_arg_scope): the per-channel moments of an
// NHWC map over every pixel of every frame, folded into the scale / shift the conv prologue applies, and the moving-average step of
// the layer's UPDATE_OPS.
//
// Two launches, no atomics, so every result is bit-identical from run to run:
//   1. bn_partial_kernel: block (chunk, channel group) sums d = x - pivot and d^2 in fp64 over its fixed range of rows (pivot = row 0
//      of the channel: the shift keeps the sums small when a channel's mean is large against its spread); threads meet in shared
//      memory in a fixed order and the block writes one (sum, sumsq) pair per channel into the workspace.
//   2. bn_finish_kernel: per channel, the chunk partials are added in chunk order (16 fixed lanes, merged in lane order), giving the
//      biased variance, scale = gamma / sqrt(var + eps), shift = beta - mean * scale and, when asked, the moving-average update.
#include <cuda_runtime.h>
#include <stdint.h>
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kColGroup = 64;            // float4 columns (256 channels) per block of the first pass
constexpr int kFinishLanes = 16;         // chunk lanes per channel in the second pass

struct Geometry {
  int C4, cw, rl, groups, chunks;
  long long chunk_rows;
};

// Depends on (rows, C) only: the chunking, and with it every rounding, is the same on every call.
Geometry geometry(long long rows, int C) {
  Geometry g;
  g.C4 = C / 4;
  g.cw = g.C4 < kColGroup ? g.C4 : kColGroup;
  g.rl = kThreads / g.cw;
  g.groups = (g.C4 + g.cw - 1) / g.cw;
  const long long most = (rows + 4LL * g.rl - 1) / (4LL * g.rl);        // at least 4 rows per thread
  long long want = 2048 / g.groups;
  if (want < 1) want = 1;
  const long long chunks = most < want ? most : want;
  g.chunk_rows = (rows + chunks - 1) / chunks;
  g.chunks = (int)((rows + g.chunk_rows - 1) / g.chunk_rows);
  return g;
}

__device__ __forceinline__ void accumulate(const float4 v, const float4 p, double *s, double *q) {
  const double d0 = (double)v.x - (double)p.x, d1 = (double)v.y - (double)p.y, d2 = (double)v.z - (double)p.z,
               d3 = (double)v.w - (double)p.w;
  s[0] += d0; s[1] += d1; s[2] += d2; s[3] += d3;
  q[0] = fma(d0, d0, q[0]); q[1] = fma(d1, d1, q[1]); q[2] = fma(d2, d2, q[2]); q[3] = fma(d3, d3, q[3]);
}

__global__ void __launch_bounds__(kThreads) bn_partial_kernel(const float *__restrict__ x, long long rows, long long ld, int C4, int cw,
                                                              int rl, long long chunk_rows, double2 *__restrict__ part) {
  __shared__ double sh_s[kThreads][4], sh_q[kThreads][4];
  const int t = threadIdx.x, cl = t % cw, r = t / cw;
  const int c4 = blockIdx.y * cw + cl;
  const bool active = r < rl && c4 < C4;
  const long long r0 = (long long)blockIdx.x * chunk_rows;
  const long long r1 = r0 + chunk_rows < rows ? r0 + chunk_rows : rows;
  double s[4] = {0., 0., 0., 0.}, q[4] = {0., 0., 0., 0.};
  if (active) {
    const float4 *col = reinterpret_cast<const float4 *>(x) + c4;
    const long long ld4 = ld / 4;
    const float4 piv = __ldg(col);
    long long i = r0 + r;
    for (; i + 3LL * rl < r1; i += 4LL * rl) {         // four independent loads in flight, summed in row order
      const float4 v0 = __ldg(col + i * ld4), v1 = __ldg(col + (i + rl) * ld4), v2 = __ldg(col + (i + 2LL * rl) * ld4),
                   v3 = __ldg(col + (i + 3LL * rl) * ld4);
      accumulate(v0, piv, s, q);
      accumulate(v1, piv, s, q);
      accumulate(v2, piv, s, q);
      accumulate(v3, piv, s, q);
    }
    for (; i < r1; i += rl) accumulate(__ldg(col + i * ld4), piv, s, q);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) { sh_s[t][k] = s[k]; sh_q[t][k] = q[k]; }
  __syncthreads();
  if (r == 0 && c4 < C4) {
    for (int j = 1; j < rl; ++j) {
#pragma unroll
      for (int k = 0; k < 4; ++k) { s[k] += sh_s[j * cw + cl][k]; q[k] += sh_q[j * cw + cl][k]; }
    }
    double2 *dst = part + (size_t)blockIdx.x * (4 * (size_t)C4) + 4 * (size_t)c4;
#pragma unroll
    for (int k = 0; k < 4; ++k) dst[k] = make_double2(s[k], q[k]);
  }
}

// TF's assign_moving_average in float32: m -= (m - v) * (1 - decay), with the batch mean and the Bessel-corrected batch variance.
__device__ __forceinline__ void moving_step(float mean, float var_b, long long rows, float momentum, float *mm, float *mv) {
  const float var_u = (float)((double)var_b * (double)rows / (double)(rows - 1));
  const float m = *mm, v = *mv;
  *mm = __fsub_rn(m, __fmul_rn(__fsub_rn(m, mean), momentum));
  *mv = __fsub_rn(v, __fmul_rn(__fsub_rn(v, var_u), momentum));
}

__global__ void __launch_bounds__(32 * kFinishLanes) bn_finish_kernel(const float *__restrict__ x, long long rows, int C, int chunks,
                                                                      const double2 *__restrict__ part, const float *__restrict__ gamma,
                                                                      const float *__restrict__ beta, float eps, float *__restrict__ scale,
                                                                      float *__restrict__ shift, float *__restrict__ mean_out,
                                                                      float *__restrict__ var_out, float *__restrict__ moving_mean,
                                                                      float *__restrict__ moving_var, float momentum) {
  __shared__ double sh_s[kFinishLanes][32], sh_q[kFinishLanes][32];
  const int cl = threadIdx.x & 31, lane = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  double s = 0., q = 0.;
  if (c < C) {
    for (int j = lane; j < chunks; j += kFinishLanes) {
      const double2 p = part[(size_t)j * C + c];
      s += p.x;
      q += p.y;
    }
  }
  sh_s[lane][cl] = s;
  sh_q[lane][cl] = q;
  __syncthreads();
  if (lane != 0 || c >= C) return;
  for (int j = 1; j < kFinishLanes; ++j) { s += sh_s[j][cl]; q += sh_q[j][cl]; }
  const double n = (double)rows;
  const double dm = s / n;
  double var = q / n - dm * dm;                       // biased; the shift keeps both terms of the size of the spread
  if (var < 0.) var = 0.;
  const double mean = (double)__ldg(x + c) + dm;
  const double sc = (double)__ldg(gamma + c) / sqrt(var + (double)eps);
  scale[c] = (float)sc;
  shift[c] = (float)((double)__ldg(beta + c) - mean * sc);
  const float mean_f = (float)mean, var_f = (float)var;
  if (mean_out) mean_out[c] = mean_f;
  if (var_out) var_out[c] = var_f;
  if (moving_mean) moving_step(mean_f, var_f, rows, momentum, moving_mean + c, moving_var + c);
}

__global__ void bn_moving_update_kernel(const float *__restrict__ mean, const float *__restrict__ var, long long rows, int C, float momentum,
                                        float *__restrict__ moving_mean, float *__restrict__ moving_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) moving_step(__ldg(mean + c), __ldg(var + c), rows, momentum, moving_mean + c, moving_var + c);
}

inline bool aligned16(const void *p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace

extern "C" size_t hd_bn_stats_workspace_bytes(long long rows, int C) {
  if (rows < 2 || C <= 0 || C % 4 != 0) return 0;
  const Geometry g = geometry(rows, C);
  return (size_t)g.chunks * (size_t)C * sizeof(double2);
}

extern "C" int hd_bn_batch_stats(const float *x, long long rows, int C, long long ld, const float *gamma, const float *beta, float eps,
                                 float *scale, float *shift, float *mean, float *var, float *moving_mean, float *moving_var, double decay,
                                 void *workspace, size_t workspace_bytes, void *stream) {
  HD_REQUIRE(x && gamma && beta && scale && shift && workspace, "hd_bn_batch_stats: null pointer");
  HD_REQUIRE(rows >= 2 && C > 0 && C % 4 == 0 && ld >= C && ld % 4 == 0 && eps >= 0.f,
             "hd_bn_batch_stats: need rows >= 2, C % 4 == 0, ld >= C with ld % 4 == 0, eps >= 0");
  HD_REQUIRE(aligned16(x) && aligned16(workspace), "hd_bn_batch_stats: x and workspace must be 16-byte aligned");
  HD_REQUIRE((moving_mean == nullptr) == (moving_var == nullptr) && (!moving_mean || (decay >= 0. && decay <= 1.)),
             "hd_bn_batch_stats: moving_mean and moving_variance go together, with 0 <= decay <= 1");
  HD_REQUIRE(workspace_bytes >= hd_bn_stats_workspace_bytes(rows, C), "hd_bn_batch_stats: workspace too small");
  const Geometry g = geometry(rows, C);
  cudaStream_t st = (cudaStream_t)stream;
  bn_partial_kernel<<<dim3(g.chunks, g.groups), kThreads, 0, st>>>(x, rows, ld, g.C4, g.cw, g.rl, g.chunk_rows,
                                                                   reinterpret_cast<double2 *>(workspace));
  int rc = hd::check_launch("bn_partial_kernel");
  if (rc) return rc;
  bn_finish_kernel<<<hd::ceil_div(C, 32), 32 * kFinishLanes, 0, st>>>(x, rows, C, g.chunks, reinterpret_cast<const double2 *>(workspace),
                                                                      gamma, beta, eps, scale, shift, mean, var, moving_mean, moving_var,
                                                                      (float)(1.0 - decay));
  return hd::check_launch("bn_finish_kernel");
}

extern "C" int hd_bn_moving_update(const float *mean, const float *var, long long rows, int C, double decay, float *moving_mean,
                                   float *moving_var, void *stream) {
  HD_REQUIRE(mean && var && moving_mean && moving_var && rows >= 2 && C > 0 && decay >= 0. && decay <= 1.,
             "hd_bn_moving_update: bad arguments (rows >= 2, 0 <= decay <= 1)");
  bn_moving_update_kernel<<<hd::ceil_div(C, 256), 256, 0, (cudaStream_t)stream>>>(mean, var, rows, C, (float)(1.0 - decay), moving_mean,
                                                                                  moving_var);
  return hd::check_launch("bn_moving_update_kernel");
}
