// Backward of the trainable layers of HMMR (f_movie, the IEF heads, fc2_res) for sm_90a: the operands the tensor-core GEMM
// (hd_conv_gemm, 3xTF32) needs for dX and dW, and the non-GEMM parts of the backward.
//
// Every reduction here is owned by one thread or one warp and runs in a fixed order; nothing uses a floating-point atomic.  Row
// (clip) r of an input gradient depends only on row (clip) r, so input gradients are bit-identical across launches, batch splits and
// permutations of the clips; weight gradients are reductions over the batch and depend on it by definition.
#include <cuda_fp16.h>
#include "conv_common.cuh"

namespace {

// Round to the nearest TF32 value (low 13 mantissa bits zero); oracle/pack_ref.py:tf32_split restates it in numpy.
__device__ __forceinline__ float rn_tf32(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}

// One element of a split operand: mode 0 = plain fp32 (hi only), 1 = TF32 head / remainder (fp32 storage), 2 = fp16 head /
// 2^11-scaled remainder (round-to-nearest-even conversions; oracle/pack_ref.py:f16_split restates it in numpy).
__device__ __forceinline__ void store_split(float v, int mode, void *hi, void *lo, size_t o) {
  if (mode == 2) {
    const __half h = __float2half_rn(v);
    reinterpret_cast<__half *>(hi)[o] = h;
    reinterpret_cast<__half *>(lo)[o] = __float2half_rn(__fmul_rn(__fsub_rn(v, __half2float(h)), 2048.0f));
  } else if (mode == 1) {
    const float h = rn_tf32(v);
    reinterpret_cast<float *>(hi)[o] = h;
    if (lo) reinterpret_cast<float *>(lo)[o] = rn_tf32(__fsub_rn(v, h));         // lo NULL: the head alone (1xTF32)
  } else {
    reinterpret_cast<float *>(hi)[o] = v;
  }
}

// dst[r, k] = src[k, r] (r < cols, k < rows), zero in the padding [cols, out_rows) x [rows, out_cols).  32 x 32 tiles through shared
// memory, so both the read (along r) and the write (along k) are coalesced.
__global__ void __launch_bounds__(256) transpose_split_kernel(const float *__restrict__ src, long long rows, int cols, long long ld, int mode,
                                                              void *hi, void *lo, long long out_ld, int out_rows, long long out_cols) {
  __shared__ float tile[32][33];
  const long long k0 = (long long)blockIdx.x * 32;
  const int r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    const long long k = k0 + i;
    const int r = r0 + tx;
    tile[i][tx] = (k < rows && r < cols) ? __ldg(src + k * ld + r) : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i;
    const long long k = k0 + tx;
    if (r < out_rows && k < out_cols) store_split(tile[tx][i], mode, hi, lo, (size_t)r * out_ld + k);
  }
}

// Backward-data packing of a KH x 1 conv (FC: KH = 1): W'[k', co, ci] = W[KH-1-k', ci, co] as the K-major B operand
// dst[ci, k' * Cout + co].  Each tap is a plain row-major [Cin, Cout] block of W, so the copy is coalesced without a transpose.
__global__ void pack_bwd_data_kernel(const float *__restrict__ w, int KH, int Cin, int Cout, int mode, void *hi, void *lo, int rows,
                                     int k_pad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * k_pad) return;
  const int ci = (int)(i / k_pad), k = (int)(i % k_pad);
  float v = 0.f;
  if (ci < Cin && k < KH * Cout) {
    const int kp = k / Cout, co = k - kp * Cout;
    v = __ldg(w + ((size_t)(KH - 1 - kp) * Cin + ci) * Cout + co);
  }
  store_split(v, mode, hi, lo, (size_t)i);
}

// Transposing im2col of a [B, T, C] sequence for the weight gradient of a KH x 1 SAME conv over T:
//   out[(kh * C + c) * out_ld + b * T + t] = a[b, t + kh - pad, c]   (0 outside the clip), columns [B*T, out_cols) = 0,
//   a = x, or relu(x * gain[b, c] + offset[b, c]) when gain / offset are given (the GroupNorm + ReLU of the forward, recomputed).
// Tile = 32 channels x 32 (clip, frame) columns per tap, through shared memory.
__global__ void __launch_bounds__(256) im2col_t_kernel(const float *__restrict__ x, int B, int T, int C, int KH, int pad,
                                                       const float *__restrict__ gain, const float *__restrict__ offset, int relu,
                                                       float *__restrict__ out, long long out_ld, long long out_cols) {
  __shared__ float tile[32][33];
  const long long col0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32, kh = blockIdx.z;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const long long BT = (long long)B * T;
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    const long long col = col0 + i;
    const int c = c0 + tx;
    float v = 0.f;
    if (col < BT && c < C) {
      const int b = (int)(col / T), t = (int)(col % T);
      const int ts = t + kh - pad;
      if (ts >= 0 && ts < T) {
        v = __ldg(x + ((size_t)b * T + ts) * C + c);
        if (gain) v = v * __ldg(gain + (size_t)b * C + c) + __ldg(offset + (size_t)b * C + c);
        if (relu) v = fmaxf(v, 0.f);
      }
    }
    tile[i][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i;
    const long long col = col0 + tx;
    if (c < C && col < out_cols) out[((size_t)kh * C + c) * out_ld + col] = tile[tx][i];
  }
}

// GroupNorm (+ ReLU) backward, one warp per (clip, group).  The statistics are recomputed with the arithmetic of
// groupnorm_stats_kernel / groupnorm_relu_split_kernel (same lane-strided order, same butterfly), so the ReLU mask z > 0 is the
// forward's.  With g = dy * (z > 0), x^ = (x - mean) * rstd, g^ = g * gamma (biased variance over n = T * C/groups elements):
//   dx = rstd * (g^ - mean(g^) - x^ * mean(g^ x^)) + addend;   dbeta_part[b, c] = sum_t g;  dgamma_part[b, c] = sum_t g x^.
// A lane owns channels lane, lane + 32, ... of the group and walks t in order, so every sum has a fixed order; any T works.
__global__ void __launch_bounds__(128) groupnorm_relu_backward_kernel(const float *__restrict__ x, const float *__restrict__ gamma,
                                                                      const float *__restrict__ beta, const float *__restrict__ dy,
                                                                      const float *__restrict__ addend, float *__restrict__ dx,
                                                                      float *__restrict__ dgamma_part, float *__restrict__ dbeta_part,
                                                                      int B, int T, int C, int groups, float eps, int relu) {
  const int lane = threadIdx.x & 31;
  const int wg = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wg >= B * groups) return;
  const int b = wg / groups, g = wg % groups;
  const int cg = C / groups;
  const float *base = x + (size_t)b * T * C + (size_t)g * cg;
  const int cnt = T * cg;
  float s = 0.f;
  for (int i = lane; i < cnt; i += 32) s += __ldg(base + (size_t)(i / cg) * C + (i % cg));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)cnt;
  float v = 0.f;
  for (int i = lane; i < cnt; i += 32) {
    const float d = __ldg(base + (size_t)(i / cg) * C + (i % cg)) - mean;
    v += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const float rstd = rsqrtf(v / (float)cnt + eps);
  const size_t off0 = (size_t)b * T * C + (size_t)g * cg;
  float s1 = 0.f, s2 = 0.f;
  for (int c = lane; c < cg; c += 32) {
    const int ch = g * cg + c;
    const float gm = __ldg(gamma + ch);
    const float gn = rstd * gm;
    const float off = __ldg(beta + ch) - mean * gn;
    float db = 0.f, dg = 0.f;
    for (int t = 0; t < T; ++t) {
      const size_t idx = off0 + (size_t)t * C + c;
      const float xv = __ldg(x + idx);
      const float z = xv * gn + off;
      const float gp = (!relu || z > 0.f) ? __ldg(dy + idx) : 0.f;
      const float xh = (xv - mean) * rstd;
      db += gp;
      dg += gp * xh;
    }
    dbeta_part[(size_t)b * C + ch] = db;
    dgamma_part[(size_t)b * C + ch] = dg;
    s1 += db * gm;
    s2 += dg * gm;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  const float m1 = s1 / (float)cnt, m2 = s2 / (float)cnt;
  for (int c = lane; c < cg; c += 32) {
    const int ch = g * cg + c;
    const float gm = __ldg(gamma + ch);
    const float gn = rstd * gm;
    const float off = __ldg(beta + ch) - mean * gn;
    for (int t = 0; t < T; ++t) {
      const size_t idx = off0 + (size_t)t * C + c;
      const float xv = __ldg(x + idx);
      const float z = xv * gn + off;
      const float gp = (!relu || z > 0.f) ? __ldg(dy + idx) : 0.f;
      const float xh = (xv - mean) * rstd;
      dx[idx] = rstd * (gp * gm - m1 - xh * m2) + (addend ? __ldg(addend + idx) : 0.f);
    }
  }
}

// out[c] = sum_r x[r * ld + c]: 8 row slices per column (rows r = slice, slice + 8, ...), then the 8 partials in slice order.
__global__ void __launch_bounds__(256) col_sum_kernel(const float *__restrict__ x, long long rows, int cols, long long ld,
                                                      float *__restrict__ out) {
  __shared__ float part[8][33];
  const int lane = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  float s = 0.f;
  if (c < cols)
    for (long long r = sl; r < rows; r += 8) s += __ldg(x + r * ld + c);
  part[sl][lane] = s;
  __syncthreads();
  if (sl == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += part[k][lane];
    out[c] = t;
  }
}

// dx = dy * (y > 0) (TF ReluGrad: 0 at 0); y is the ReLU's output (or input).  p < 1: y is the output of a dropout after the ReLU
// (y > 0 <=> kept and positive) and dx = y > 0 ? dy / p : 0, TF's gradient through the dropout's Mul by the 0 / 1 mask, then its
// RealDiv by keep_prob.
__global__ void relu_backward_kernel(const float *__restrict__ y, const float *dy, float *dx, long long n, float p) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  dx[i] = __ldg(y + i) > 0.f ? (p < 1.f ? __fdiv_rn(dy[i], p) : dy[i]) : 0.f;
}

// out[n, k] = (mask[n, k] > 0) * sum_{j < D} g[n, j] * Wt[j, k]    (Wt [D, K] row-major, D <= 96, mask nullable).
// The K = 85 / 72 input-gradient product of the IEF fc3 (dh2 = dtheta . W3^T): too short for the tensor-core tile.  A block takes 8
// rows and all K columns (thread = 4 columns); j runs in order, so each output has a fixed summation order.  p < 1: mask is the output
// of a dropout after the ReLU and a kept element's gradient is divided by p (relu_backward_kernel).
__global__ void __launch_bounds__(256) fc_small_dgrad_kernel(const float *__restrict__ g, int g_ld, const float *__restrict__ Wt, int K,
                                                             int D, const float *__restrict__ mask, float *__restrict__ out, int N, float p) {
  __shared__ float gs[8][96];
  const int r0 = blockIdx.x * 8;
  for (int i = threadIdx.x; i < 8 * 96; i += 256) {
    const int r = i / 96, j = i - r * 96;
    gs[r][j] = (r0 + r < N && j < D) ? __ldg(g + (size_t)(r0 + r) * g_ld + j) : 0.f;
  }
  __syncthreads();
  for (int c = threadIdx.x * 4; c < K; c += 1024) {
    float acc[8][4];
#pragma unroll
    for (int r = 0; r < 8; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;
    for (int j = 0; j < D; ++j) {
      const float4 w = __ldg(reinterpret_cast<const float4 *>(Wt + (size_t)j * K + c));
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float t = gs[r][j];
        acc[r][0] += t * w.x; acc[r][1] += t * w.y; acc[r][2] += t * w.z; acc[r][3] += t * w.w;
      }
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      if (r0 + r >= N) break;
      const size_t o = (size_t)(r0 + r) * K + c;
      float4 y = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
      if (mask) {
        const float4 m = __ldg(reinterpret_cast<const float4 *>(mask + o));
        y.x = m.x > 0.f ? y.x : 0.f; y.y = m.y > 0.f ? y.y : 0.f; y.z = m.z > 0.f ? y.z : 0.f; y.w = m.w > 0.f ? y.w : 0.f;
        if (p < 1.f) { y.x = __fdiv_rn(y.x, p); y.y = __fdiv_rn(y.y, p); y.z = __fdiv_rn(y.z, p); y.w = __fdiv_rn(y.w, p); }
      }
      *reinterpret_cast<float4 *>(out + o) = y;
    }
  }
}

// out[r, c] = a[r, c] + b[r, c] at independent row strides (out may alias a or b).
__global__ void add_strided_kernel(const float *a, long long lda, const float *b, long long ldb, float *out, long long ldo, int rows, int cols) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * cols) return;
  const long long r = i / cols, c = i % cols;
  out[r * ldo + c] = a[r * lda + c] + b[r * ldb + c];
}

}  // namespace

extern "C" {

int hd_transpose_split(const float *x, long long rows, int cols, long long ld, int mode, void *hi, void *lo, long long out_ld, int out_rows,
                       long long out_cols, void *stream) {
  HD_REQUIRE(x && hi && rows > 0 && cols > 0 && ld >= cols && (mode == 0 || mode == 1 || mode == 2) && (mode == 0 ? lo == nullptr : (mode == 1 || lo != nullptr)) &&
                 out_rows >= cols && out_cols >= rows && out_ld >= out_cols,
             "hd_transpose_split: bad arguments (mode 0 = fp32 with lo NULL, 1 = tf32 pair or head, 2 = fp16 pair; out_rows >= cols, out_cols >= rows)");
  dim3 grid((unsigned)hd::ceil_div(out_cols, 32), (unsigned)hd::ceil_div(out_rows, 32));
  HD_REQUIRE(grid.y <= 65535u, "hd_transpose_split: out_rows too large");
  transpose_split_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, rows, cols, ld, mode, hi, lo, out_ld, out_rows, out_cols);
  return hd::check_launch("transpose_split_kernel");
}

int hd_pack_weight(const float *w, int KH, int Cin, int Cout, int mode, int elem_bytes, void *hi, void *lo, int rows, int k_pad, void *stream) {
  HD_REQUIRE(w && hi && lo && KH > 0 && Cin > 0 && Cout > 0 && (mode == HD_PACK_FORWARD || mode == HD_PACK_BACKWARD_DATA) &&
                 (elem_bytes == 2 || elem_bytes == 4) && rows > 0 && rows % 64 == 0 && k_pad > 0 && k_pad % (128 / elem_bytes) == 0 &&
                 hd::aligned16(hi) && hd::aligned16(lo),
             "hd_pack_weight: bad arguments (rows % 64 == 0, k_pad % 32 (tf32) / % 64 (fp16) == 0, aligned outputs)");
  const int n_out = mode == HD_PACK_FORWARD ? Cout : Cin;
  const long long k = (long long)KH * (mode == HD_PACK_FORWARD ? Cin : Cout);
  HD_REQUIRE(rows >= n_out && k_pad >= k, "hd_pack_weight: rows / k_pad smaller than the packed matrix");
  const int sm = elem_bytes == 2 ? 2 : 1;
  if (mode == HD_PACK_FORWARD) return hd_transpose_split(w, k, Cout, Cout, sm, hi, lo, k_pad, rows, k_pad, stream);
  const long long total = (long long)rows * k_pad;
  pack_bwd_data_kernel<<<hd::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(w, KH, Cin, Cout, sm, hi, lo, rows, k_pad);
  return hd::check_launch("pack_bwd_data_kernel");
}

int hd_im2col_t(const float *x, int B, int T, int C, int KH, int pad, const float *gain, const float *offset, int relu, float *out,
                long long out_ld, long long out_cols, void *stream) {
  HD_REQUIRE(x && out && B > 0 && T > 0 && C > 0 && KH > 0 && KH <= 65535 && pad >= 0 && pad < KH && ((gain == nullptr) == (offset == nullptr)) &&
                 out_cols >= (long long)B * T && out_ld >= out_cols,
             "hd_im2col_t: bad arguments");
  dim3 grid((unsigned)hd::ceil_div(out_cols, 32), (unsigned)hd::ceil_div(C, 32), (unsigned)KH);
  HD_REQUIRE(grid.y <= 65535u, "hd_im2col_t: C too large");
  im2col_t_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, B, T, C, KH, pad, gain, offset, relu, out, out_ld, out_cols);
  return hd::check_launch("im2col_t_kernel");
}

int hd_groupnorm_relu_backward(const float *x, const float *gamma, const float *beta, const float *dy, const float *addend, float *dx,
                               float *dgamma_part, float *dbeta_part, int B, int T, int C, int groups, float eps, int relu, void *stream) {
  HD_REQUIRE(x && gamma && beta && dy && dx && dgamma_part && dbeta_part && B > 0 && T > 0 && C > 0 && groups > 0 && C % groups == 0 &&
                 dx != x && dx != dy,
             "hd_groupnorm_relu_backward: bad arguments");
  groupnorm_relu_backward_kernel<<<hd::ceil_div((long long)B * groups, 4), 128, 0, (cudaStream_t)stream>>>(
      x, gamma, beta, dy, addend, dx, dgamma_part, dbeta_part, B, T, C, groups, eps, relu);
  return hd::check_launch("groupnorm_relu_backward_kernel");
}

int hd_col_sum(const float *x, long long rows, int cols, long long ld, float *out, void *stream) {
  HD_REQUIRE(x && out && rows > 0 && cols > 0 && ld >= cols, "hd_col_sum: bad arguments");
  col_sum_kernel<<<hd::ceil_div(cols, 32), 256, 0, (cudaStream_t)stream>>>(x, rows, cols, ld, out);
  return hd::check_launch("col_sum_kernel");
}

int hd_relu_backward(const float *y, const float *dy, float *dx, long long n, void *stream) {
  HD_REQUIRE(y && dy && dx && n > 0, "hd_relu_backward: bad arguments");
  relu_backward_kernel<<<hd::ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(y, dy, dx, n, 1.f);
  return hd::check_launch("relu_backward_kernel");
}

int hd_relu_dropout_backward(const float *y, const float *dy, float *dx, long long n, float p, void *stream) {
  HD_REQUIRE(y && dy && dx && n > 0 && p > 0.f && p <= 1.f, "hd_relu_dropout_backward: bad arguments (0 < p <= 1)");
  relu_backward_kernel<<<hd::ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(y, dy, dx, n, p);
  return hd::check_launch("relu_backward_kernel");
}

int hd_fc_small_dgrad(const float *g, int g_ld, const float *Wt, int K, int D, const float *mask, float *out, int N, void *stream) {
  HD_REQUIRE(g && Wt && out && N > 0 && D > 0 && D <= 96 && g_ld >= D && K > 0 && K % 4 == 0 && hd::aligned16(Wt) && hd::aligned16(out) &&
                 (!mask || hd::aligned16(mask)),
             "hd_fc_small_dgrad: bad arguments (D <= 96, K % 4 == 0, 16-byte aligned Wt / mask / out)");
  fc_small_dgrad_kernel<<<hd::ceil_div(N, 8), 256, 0, (cudaStream_t)stream>>>(g, g_ld, Wt, K, D, mask, out, N, 1.f);
  return hd::check_launch("fc_small_dgrad_kernel");
}

int hd_fc_small_dgrad_dropout(const float *g, int g_ld, const float *Wt, int K, int D, const float *mask, float p, float *out, int N,
                              void *stream) {
  HD_REQUIRE(g && Wt && mask && out && N > 0 && D > 0 && D <= 96 && g_ld >= D && K > 0 && K % 4 == 0 && p > 0.f && p <= 1.f &&
                 hd::aligned16(Wt) && hd::aligned16(out) && hd::aligned16(mask),
             "hd_fc_small_dgrad_dropout: bad arguments (D <= 96, K % 4 == 0, 0 < p <= 1, 16-byte aligned Wt / mask / out)");
  fc_small_dgrad_kernel<<<hd::ceil_div(N, 8), 256, 0, (cudaStream_t)stream>>>(g, g_ld, Wt, K, D, mask, out, N, p);
  return hd::check_launch("fc_small_dgrad_kernel");
}

int hd_add_strided(const float *a, long long lda, const float *b, long long ldb, float *out, long long ldo, int rows, int cols, void *stream) {
  HD_REQUIRE(a && b && out && rows > 0 && cols > 0 && lda >= cols && ldb >= cols && ldo >= cols, "hd_add_strided: bad arguments");
  add_strided_kernel<<<hd::ceil_div((long long)rows * cols, 256), 256, 0, (cudaStream_t)stream>>>(a, lda, b, ldb, out, ldo, rows, cols);
  return hd::check_launch("add_strided_kernel");
}

}  // extern "C"
