// Small non-GEMM pieces of the network path: ResNet root/tail, GroupNorm statistics, IEF glue.
#include <cuda_fp16.h>
#include "conv_common.cuh"
#include "dropout.cuh"

namespace {

// pool1 (slim.max_pool2d 3x3/2 'SAME'): padded cells are ignored.
__global__ void maxpool3x3s2_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, int N, int H, int W, int C4,
                                    int Ho, int Wo, int pt, int pl, const float4 *__restrict__ scale,
                                    const float4 *__restrict__ shift, uint2 *__restrict__ out_hi, uint2 *__restrict__ out_lo) {
  const long long total = (long long)N * Ho * Wo * C4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C4);
  long long r = i / C4;
  const int ox = (int)(r % Wo); r /= Wo;
  const int oy = (int)(r % Ho);
  const int n = (int)(r / Ho);
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = oy * 2 - pt + ky;
    if (iy < 0 || iy >= H) continue;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int ix = ox * 2 - pl + kx;
      if (ix < 0 || ix >= W) continue;
      const float4 v = __ldg(in + ((size_t)((size_t)n * H + iy) * W + ix) * C4 + c);
      m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
    }
  }
  if (out) out[i] = m;
  if (out_hi) {        // relu(bn(x)) of the first bottleneck unit, as an fp16 head/remainder pair
    const float4 sc = __ldg(scale + c), sh = __ldg(shift + c);
    const float y[4] = {fmaxf(m.x * sc.x + sh.x, 0.f), fmaxf(m.y * sc.y + sh.y, 0.f), fmaxf(m.z * sc.z + sh.z, 0.f),
                        fmaxf(m.w * sc.w + sh.w, 0.f)};
    uint32_t hp[2], lp[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) hd::split_f16x2(y[2 * e], y[2 * e + 1], hp[e], lp[e]);
    out_hi[i] = make_uint2(hp[0], hp[1]);
    if (out_lo) out_lo[i] = make_uint2(lp[0], lp[1]);
  }
}

// postnorm BN + ReLU + mean over HW.  One thread per (n, c); consecutive threads -> consecutive channels.
__global__ void bnrelu_avgpool_kernel(const float *__restrict__ in, const float *__restrict__ scale,
                                      const float *__restrict__ shift, float *__restrict__ out, int N, int HW, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * C) return;
  const int c = (int)(i % C);
  const long long n = i / C;
  const float s = __ldg(scale + c), b = __ldg(shift + c);
  const float *p = in + (size_t)n * HW * C + c;
  float acc = 0.f;
  for (int k = 0; k < HW; ++k) acc += fmaxf(__ldg(p + (size_t)k * C) * s + b, 0.f);
  out[i] = acc / (float)HW;
}

// One warp per (clip, group): two-pass mean / biased variance over T x (C/groups) elements, then the
// per-channel affine that the conv prologue applies: y = x*gain + offset.
__global__ void __launch_bounds__(128) groupnorm_stats_kernel(const float *__restrict__ x, const float *__restrict__ gamma,
                                                              const float *__restrict__ beta, float *__restrict__ gain,
                                                              float *__restrict__ offset, int B, int T, int C, int groups,
                                                              float eps) {
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
  for (int c = lane; c < cg; c += 32) {
    const int ch = g * cg + c;
    const float gn = rstd * __ldg(gamma + ch);
    gain[(size_t)b * C + ch] = gn;
    offset[(size_t)b * C + ch] = __ldg(beta + ch) - mean * gn;
  }
}

// process_image (src/evaluation/run_video.py:56-107): one thread per output pixel of the S x S crop.
//   crop(y,x) = padded_scaled[y0 + y + S][x0 + x + S], padded = edge-replicated => clamp the scaled-image coordinates;
//   scaled = cv2.resize(2*(u8/255 - 0.5), (Ws,Hs)) bilinear: source coordinate (d + 0.5)*scale - 0.5, floor, weights (1-f, f),
//   neighbours clamped to the image (cv2's xofs/yofs clipping).
__global__ void process_image_kernel(const uint8_t *__restrict__ frames, int N, int H, int W, const int4 *__restrict__ geom,
                                     float *__restrict__ out, int S, uint2 *__restrict__ plane_hi, uint2 *__restrict__ plane_lo, int WP) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * S * S) return;
  const int x = (int)(i % S);
  const int y = (int)((i / S) % S);
  const int n = (int)(i / ((long long)S * S));
  const int4 g = __ldg(geom + n);              // Hs, Ws, x0, y0
  const int Hs = g.x, Ws = g.y;
  const int xs = min(max(g.z + x, 0), Ws - 1), ys = min(max(g.w + y, 0), Hs - 1);
  const double scale_x = 1.0 / ((double)Ws / (double)W), scale_y = 1.0 / ((double)Hs / (double)H);     // cv2: scale = 1. / inv_scale
  // the reference resizes the float64 image: cv2 (4.x) keeps source coordinates and weights in double on that path -- probed with a
  // ramp image, tests/test_preprocess.py -- so the fraction is taken in double and only then narrowed
  const double cxd = (xs + 0.5) * scale_x - 0.5, cyd = (ys + 0.5) * scale_y - 0.5;
  int sx = (int)floor(cxd), sy = (int)floor(cyd);
  float fx = (float)(cxd - (double)sx), fy = (float)(cyd - (double)sy);
  if (sx < 0) { fx = 0.f; sx = 0; }
  if (sx >= W - 1) { fx = 0.f; sx = W - 1; }
  const int sx1 = min(sx + 1, W - 1);
  const int sy0 = min(max(sy, 0), H - 1), sy1 = min(max(sy + 1, 0), H - 1);
  const uint8_t *f = frames + (size_t)n * H * W * 3;
  const uint8_t *r0 = f + (size_t)sy0 * W * 3, *r1 = f + (size_t)sy1 * W * 3;
  const float a0 = 1.f - fx, a1 = fx, b0 = 1.f - fy, b1 = fy;
  float v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float p00 = ((float)r0[sx * 3 + c] / 255.f - 0.5f) * 2.f, p01 = ((float)r0[sx1 * 3 + c] / 255.f - 0.5f) * 2.f;
    const float p10 = ((float)r1[sx * 3 + c] / 255.f - 0.5f) * 2.f, p11 = ((float)r1[sx1 * 3 + c] / 255.f - 0.5f) * 2.f;
    v[c] = (p00 * a0 + p01 * a1) * b0 + (p10 * a0 + p11 * a1) * b1;
  }
  if (out) {
    float *o = out + (size_t)i * 3;
    o[0] = v[0]; o[1] = v[1]; o[2] = v[2];
  }
  if (plane_hi) {        // the tensor-core conv1's input format (see pack_conv1_planes_kernel): the fp32 crop need not exist at all
    uint32_t h0, l0, h1, l1;
    hd::split_f16x2(v[0], v[1], h0, l0);
    hd::split_f16x2(v[2], 0.f, h1, l1);
    const size_t po = ((size_t)n * (S + 6) + y + 3) * WP + x + 3;
    plane_hi[po] = make_uint2(h0, h1);
    if (plane_lo) plane_lo[po] = make_uint2(l0, l1);
  }
}

// fp32 NHWC image -> padded RGBX fp16 head / remainder planes (the A operand of the tensor-core conv1).  One thread per pixel.
__global__ void pack_conv1_planes_kernel(const float *__restrict__ img, uint2 *__restrict__ hi, uint2 *__restrict__ lo, int N, int H, int W,
                                         int WP) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * H * W) return;
  const int x = (int)(i % W);
  const int y = (int)((i / W) % H);
  const int n = (int)(i / ((long long)W * H));
  const float *s = img + (size_t)i * 3;
  uint32_t h0, l0, h1, l1;
  hd::split_f16x2(__ldg(s), __ldg(s + 1), h0, l0);
  hd::split_f16x2(__ldg(s + 2), 0.f, h1, l1);
  const size_t o = ((size_t)n * (H + 6) + y + 3) * WP + x + 3;
  hi[o] = make_uint2(h0, h1);
  if (lo) lo[o] = make_uint2(l0, l1);
}

// max_pool2d(1x1, stride s) = spatial subsampling: the identity shortcut of a strided bottleneck unit (A.4).
// One warp per 4 consecutive output pixels: lanes stride over the channels, the 4 pixels' loads are independent, so a thread has
// 4 (C = 128) to 8 (C >= 256, loop unrolled twice) 16-byte loads in flight -- the kernel is a pure strided copy and lives on that.
__global__ void __launch_bounds__(256) subsample_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, int N, int H, int W, int C4,
                                                        int Ho, int Wo, int s) {
  constexpr int PPW = 4;
  const long long total = (long long)N * Ho * Wo;
  const long long pix0 = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * PPW;
  if (pix0 >= total) return;
  const int lane = threadIdx.x & 31;
  const float4 *src[PPW];
#pragma unroll
  for (int u = 0; u < PPW; ++u) {
    const long long pix = pix0 + u < total ? pix0 + u : total - 1;      // tail: duplicates of the last pixel, never stored
    const int ox = (int)(pix % Wo);
    const int oy = (int)((pix / Wo) % Ho);
    const int n = (int)(pix / ((long long)Wo * Ho));
    src[u] = in + ((size_t)((size_t)n * H + (size_t)oy * s) * W + (size_t)ox * s) * C4;
  }
  float4 *dst = out + (size_t)pix0 * C4;
#pragma unroll 2
  for (int c = lane; c < C4; c += 32) {
    float4 v[PPW];
#pragma unroll
    for (int u = 0; u < PPW; ++u) v[u] = __ldg(src[u] + c);
#pragma unroll
    for (int u = 0; u < PPW; ++u)
      if (pix0 + u < total) dst[(size_t)u * C4 + c] = v[u];
  }
}

// GroupNorm + ReLU + fp16 split in one pass (f_movie pre-activations, src/models.py:155-171,188-204): one warp per (clip, group).
// Same statistics and the same affine as groupnorm_stats_kernel + the conv prologue it replaces (y = relu(x*gain + offset), gain =
// rstd*gamma, offset = beta - mean*gain; identical summation order), but the result leaves as the pre-split A operand of the
// tensor-core conv, so the temporal convs take the cp.async producer instead of the register-staged one.  T*cg <= 40*32 elements.
__global__ void __launch_bounds__(128) groupnorm_relu_split_kernel(const float *__restrict__ x, const float *__restrict__ gamma,
                                                                   const float *__restrict__ beta, __half *__restrict__ out_hi,
                                                                   __half *__restrict__ out_lo, int B, int T, int C, int groups, float eps) {
  const int lane = threadIdx.x & 31;
  const int wg = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wg >= B * groups) return;
  const int b = wg / groups, g = wg % groups;
  const int cg = C / groups;
  const size_t base = (size_t)b * T * C + (size_t)g * cg;
  const int cnt = T * cg;
  constexpr int MAXE = 40;
  float v[MAXE];
  float s = 0.f;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) {
    const int i = lane + 32 * e;
    // element i of the group = (row i / cg, channel i % cg); cg == 64 (f_movie: 2048 / 32) makes that (e >> 1, lane + 32 (e & 1))
    const size_t off = cg == 64 ? (size_t)(e >> 1) * C + (lane + 32 * (e & 1)) : (size_t)(i / cg) * C + (i % cg);
    v[e] = i < cnt ? __ldg(x + base + off) : 0.f;
    if (i < cnt) s += v[e];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)cnt;
  float q = 0.f;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) {
    const int i = lane + 32 * e;
    if (i < cnt) { const float d = v[e] - mean; q += d * d; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)cnt + eps);
#pragma unroll
  for (int e = 0; e < MAXE; ++e) {
    const int i = lane + 32 * e;
    if (i >= cnt) continue;
    const int cin = cg == 64 ? lane + 32 * (e & 1) : i % cg;
    const int ch = g * cg + cin;
    const float gn = rstd * __ldg(gamma + ch);
    const float off = __ldg(beta + ch) - mean * gn;
    const float y = fmaxf(v[e] * gn + off, 0.f);
    uint32_t h, l;
    hd::split_f16x2(y, 0.f, h, l);
    const size_t o = base + (cg == 64 ? (size_t)(e >> 1) * C : (size_t)(i / cg) * C) + cin;
    out_hi[o] = __ushort_as_half((unsigned short)(h & 0xffffu));
    if (out_lo) out_lo[o] = __ushort_as_half((unsigned short)(l & 0xffffu));
  }
}

// fp32 -> fp16 head / remainder pair (the A operand format of the tensor-core GEMM), 4 elements per thread.
__global__ void split_f16_kernel(const float4 *__restrict__ x, uint2 *__restrict__ hi, uint2 *__restrict__ lo, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = __ldg(x + i);
  uint32_t h0, l0, h1, l1;
  hd::split_f16x2(v.x, v.y, h0, l0);
  hd::split_f16x2(v.z, v.w, h1, l1);
  hi[i] = make_uint2(h0, h1);
  if (lo) lo[i] = make_uint2(l0, l1);
}

// IEF fc1, theta part (src/models.py:402,102: state = concat[phi, theta] -> fc1): h1 = relu(P + theta . W1[2048:]) with P = phi . W1[:2048]
// + b1 hoisted out of the stage loop.  K = 85 / 72 is far too short for the tensor-core tile; here a block takes 8 rows and all C
// columns (thread = 4 columns), theta rows sit in smem, W streams from L2 (348 KB, read once per block).  Output = the pre-split
// fp16 pair fc2's cp.async producer loads (and optionally fp32).  drop.p < 1: the dropout1 mask (dropout.cuh) is applied to h1 before
// either is written.
__global__ void __launch_bounds__(256) ief_fc1_theta_kernel(const float *__restrict__ P, const float *__restrict__ theta, int theta_ld,
                                                            const float *__restrict__ W, int K, int Cc, __half *__restrict__ out_hi,
                                                            __half *__restrict__ out_lo, float *__restrict__ out_f32, int N,
                                                            const hd::DropoutSite drop) {
  __shared__ float th[8][96];
  const int r0 = blockIdx.x * 8;
  for (int i = threadIdx.x; i < 8 * 96; i += 256) {
    const int r = i / 96, k = i - r * 96;
    th[r][k] = (r0 + r < N && k < K) ? __ldg(theta + (size_t)(r0 + r) * theta_ld + k) : 0.f;
  }
  __syncthreads();
  for (int c = threadIdx.x * 4; c < Cc; c += 1024) {
    float acc[8][4];
#pragma unroll
    for (int r = 0; r < 8; ++r) { acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f; }
    for (int k0 = 0; k0 < K; k0 += 8) {          // 8 weight rows in flight: the loop is L2-latency-, not FMA-bound otherwise
      float4 w[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        w[u] = (k0 + u < K) ? __ldg(reinterpret_cast<const float4 *>(W + (size_t)(k0 + u) * Cc + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const float t = th[r][k0 + u];           // zero beyond K (th is 96 wide, K <= 96)
          acc[r][0] += t * w[u].x; acc[r][1] += t * w[u].y; acc[r][2] += t * w[u].z; acc[r][3] += t * w[u].w;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      if (r0 + r >= N) break;
      const size_t o = (size_t)(r0 + r) * Cc + c;
      const float4 p = __ldg(reinterpret_cast<const float4 *>(P + o));
      float y0 = fmaxf(acc[r][0] + p.x, 0.f), y1 = fmaxf(acc[r][1] + p.y, 0.f), y2 = fmaxf(acc[r][2] + p.z, 0.f),
            y3 = fmaxf(acc[r][3] + p.w, 0.f);
      if (drop.p < 1.f) {            // Cc % 4 == 0: columns c .. c+3 are the four words of one Philox call
        const float4 m = hd::dropout_apply4(drop, o >> 2, make_float4(y0, y1, y2, y3));
        y0 = m.x; y1 = m.y; y2 = m.z; y3 = m.w;
      }
      if (out_f32) *reinterpret_cast<float4 *>(out_f32 + o) = make_float4(y0, y1, y2, y3);
      if (out_hi) {
        uint32_t h0, l0, h1, l1;
        hd::split_f16x2(y0, y1, h0, l0);
        hd::split_f16x2(y2, y3, h1, l1);
        *reinterpret_cast<uint2 *>(out_hi + o) = make_uint2(h0, h1);
        if (out_lo) *reinterpret_cast<uint2 *>(out_lo + o) = make_uint2(l0, l1);
      }
    }
  }
}

// IEF fc3 + update (models.py:113,410): theta_out = theta_prev + h2 . W3 + b3, W3 [K, D] with D = 85 / 72: one tensor-core tile
// would serialise K = 1024 on 5 CTAs.  Block = 8 rows x 8 warps; warp w sums k in [w*K/8, (w+1)*K/8) for the block's rows (lane = output
// column, 3 per lane), partial sums meet in smem in warp order: fixed summation order, bit-reproducible.  drop.p < 1: h2 is read
// through the dropout2 mask (dropout.cuh) and the masked rows are written back over it (fc3's weight gradient reads them); the sums
// are the same code.
__global__ void __launch_bounds__(256) ief_fc3_kernel(const float *h2, const float *__restrict__ W, const float *__restrict__ bias,
                                                      const float *__restrict__ prev, int prev_ld, float *__restrict__ out, int out_ld, int N,
                                                      int K, int D, const hd::DropoutSite drop, float *h2_masked) {
  extern __shared__ float sm[];
  float *hs = sm;                         // [8][K]
  float *part = sm + 8 * K;               // [8 warps][8 rows][96]
  const int r0 = blockIdx.x * 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (drop.p < 1.f) {
    for (int i = threadIdx.x * 4; i < 8 * K; i += 1024) {        // K % 64 == 0: four columns of one row, one Philox call
      const int r = i / K, k = i - r * K;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r0 + r < N) {
        const size_t o = (size_t)(r0 + r) * K + k;
        v = hd::dropout_apply4(drop, o >> 2, *reinterpret_cast<const float4 *>(h2 + o));
        *reinterpret_cast<float4 *>(h2_masked + o) = v;
      }
      *reinterpret_cast<float4 *>(hs + i) = v;
    }
  } else {
    for (int i = threadIdx.x; i < 8 * K; i += 256) {
      const int r = i / K, k = i - r * K;
      hs[i] = (r0 + r < N) ? __ldg(h2 + (size_t)(r0 + r) * K + k) : 0.f;
    }
  }
  __syncthreads();
  float acc[8][3];
#pragma unroll
  for (int r = 0; r < 8; ++r) acc[r][0] = acc[r][1] = acc[r][2] = 0.f;
  const int kper = K / 8;
  const bool c0 = lane < D, c1 = lane + 32 < D, c2 = lane + 64 < D;     // D < 32: no column of W past D is read
  for (int k0 = warp * kper; k0 < (warp + 1) * kper; k0 += 8) {       // (kper % 8 == 0 is required by the host entry)
    float w0[8], w1[8], w2[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float *wr = W + (size_t)(k0 + u) * D;
      w0[u] = c0 ? __ldg(wr + lane) : 0.f; w1[u] = c1 ? __ldg(wr + lane + 32) : 0.f; w2[u] = c2 ? __ldg(wr + lane + 64) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float h = hs[r * K + k0 + u];
        acc[r][0] += h * w0[u]; acc[r][1] += h * w1[u]; acc[r][2] += h * w2[u];
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    float *pp = part + (warp * 8 + r) * 96;
    pp[lane] = acc[r][0]; pp[lane + 32] = acc[r][1]; pp[lane + 64] = acc[r][2];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 8 * D; i += 256) {
    const int r = i / D, j = i - r * D;
    if (r0 + r >= N) continue;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += part[(w * 8 + r) * 96 + j];
    out[(size_t)(r0 + r) * out_ld + j] = (s + __ldg(bias + j)) + prev[(size_t)(r0 + r) * prev_ld + j];
  }
}

__global__ void ief_delta_init_kernel(const float *__restrict__ theta, float *__restrict__ dst, int dst_ld, int N) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * 85) return;
  const int c = i % 85, n = i / 85;
  dst[(size_t)n * dst_ld + c] = c == 0 ? 1.0f : (c < 3 ? 0.0f : theta[i]);
}

}  // namespace

extern "C" {

int hd_conv1_7x7s2(const float *in, const float *w, const float *bias, float *out, int N, int H, int W, void *stream) {
  HD_REQUIRE(in && w && bias && out && N > 0 && H > 0 && W > 0 && (H % 2 == 0) && (W % 2 == 0), "hd_conv1_7x7s2: bad arguments");
  hd_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.in = in; d.in_ld = 3; d.n_img = N; d.H = H; d.W = W; d.Cin = 3;
  d.Ho = H / 2; d.Wo = W / 2; d.KH = 7; d.KW = 7; d.stride = 2; d.pad_t = 3; d.pad_l = 3;   // conv2d_same: explicit pad 3+3
  d.w_kn = w; d.Cout = 64; d.post_shift = bias; d.out = out; d.out_ld = 64; d.impl = HD_IMPL_SIMT;
  hd::ConvParams p;
  int rc = hd::fill_params(&d, p);
  if (rc) return rc;
  return hd::launch_conv_simt(p, (cudaStream_t)stream);
}

int hd_maxpool3x3s2_same(const float *in, float *out, int N, int H, int W, int C, const float *scale, const float *shift,
                         void *out_hi, void *out_lo, void *stream) {
  HD_REQUIRE(in && (out || out_hi) && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "hd_maxpool3x3s2_same: bad arguments");
  HD_REQUIRE((out_hi || !out_lo) && (!out_hi || (scale && shift)), "hd_maxpool3x3s2_same: split output needs scale, shift and out_hi");
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const int pth = (Ho - 1) * 2 + 3 - H, ptw = (Wo - 1) * 2 + 3 - W;
  const int pt = (pth > 0 ? pth : 0) / 2, pl = (ptw > 0 ? ptw : 0) / 2;
  const long long total = (long long)N * Ho * Wo * (C / 4);
  maxpool3x3s2_kernel<<<hd::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4 *>(in), reinterpret_cast<float4 *>(out), N, H, W, C / 4, Ho, Wo, pt, pl,
      reinterpret_cast<const float4 *>(scale), reinterpret_cast<const float4 *>(shift), reinterpret_cast<uint2 *>(out_hi),
      reinterpret_cast<uint2 *>(out_lo));
  return hd::check_launch("maxpool3x3s2_kernel");
}

int hd_bnrelu_avgpool(const float *in, const float *scale, const float *shift, float *out, int N, int HW, int C, void *stream) {
  HD_REQUIRE(in && scale && shift && out && N > 0 && HW > 0 && C > 0, "hd_bnrelu_avgpool: bad arguments");
  bnrelu_avgpool_kernel<<<hd::ceil_div((long long)N * C, 256), 256, 0, (cudaStream_t)stream>>>(in, scale, shift, out, N, HW, C);
  return hd::check_launch("bnrelu_avgpool_kernel");
}

int hd_groupnorm_stats(const float *x, const float *gamma, const float *beta, float *gain, float *offset, int B, int T,
                       int C, int groups, float eps, void *stream) {
  HD_REQUIRE(x && gamma && beta && gain && offset && B > 0 && T > 0 && C > 0 && groups > 0 && C % groups == 0,
             "hd_groupnorm_stats: bad arguments");
  groupnorm_stats_kernel<<<hd::ceil_div((long long)B * groups, 4), 128, 0, (cudaStream_t)stream>>>(x, gamma, beta, gain, offset,
                                                                                                 B, T, C, groups, eps);
  return hd::check_launch("groupnorm_stats_kernel");
}

int hd_ief_delta_init(const float *theta, float *dst, int dst_ld, int N, void *stream) {
  HD_REQUIRE(theta && dst && N > 0 && dst_ld >= 85, "hd_ief_delta_init: bad arguments");
  ief_delta_init_kernel<<<hd::ceil_div((long long)N * 85, 256), 256, 0, (cudaStream_t)stream>>>(theta, dst, dst_ld, N);
  return hd::check_launch("ief_delta_init_kernel");
}

}  // extern "C"

extern "C" int hd_process_image(const unsigned char *frames, int N, int H, int W, const int *geom, float *out, int S, void *plane_hi,
                                void *plane_lo, int WP, void *stream) {
  HD_REQUIRE(frames && geom && (out || plane_hi) && N > 0 && H > 0 && W > 0 && S > 0 && ((uintptr_t)geom & 15u) == 0 &&
                 (plane_hi || !plane_lo) && (!plane_hi || (WP >= S + 8 && WP % 2 == 0 && hd::aligned16(plane_hi) && hd::aligned16(plane_lo))),
             "hd_process_image: bad arguments");
  const long long total = (long long)N * S * S;
  process_image_kernel<<<hd::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(frames, N, H, W, reinterpret_cast<const int4 *>(geom), out, S,
                                                                                 reinterpret_cast<uint2 *>(plane_hi),
                                                                                 reinterpret_cast<uint2 *>(plane_lo), WP);
  return hd::check_launch("process_image_kernel");
}

extern "C" int hd_pack_conv1_planes(const float *img, void *plane_hi, void *plane_lo, int N, int H, int W, int WP, void *stream) {
  HD_REQUIRE(img && plane_hi && N > 0 && H > 0 && W > 0 && WP >= W + 8 && WP % 2 == 0 && hd::aligned16(plane_hi) &&
                 hd::aligned16(plane_lo),
             "hd_pack_conv1_planes: bad arguments");
  const long long total = (long long)N * H * W;
  pack_conv1_planes_kernel<<<hd::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(img, reinterpret_cast<uint2 *>(plane_hi),
                                                                                     reinterpret_cast<uint2 *>(plane_lo), N, H, W, WP);
  return hd::check_launch("pack_conv1_planes_kernel");
}

extern "C" int hd_subsample(const float *in, float *out, int N, int H, int W, int C, int stride, void *stream) {
  HD_REQUIRE(in && out && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && stride >= 1 && hd::aligned16(in) && hd::aligned16(out),
             "hd_subsample: bad arguments");
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long total = (long long)N * Ho * Wo;            // one warp per 4 output pixels, 8 warps per block
  subsample_kernel<<<hd::ceil_div(total, 32), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4 *>(in), reinterpret_cast<float4 *>(out), N,
                                                                             H, W, C / 4, Ho, Wo, stride);
  return hd::check_launch("subsample_kernel");
}

extern "C" int hd_groupnorm_relu_split(const float *x, const float *gamma, const float *beta, void *out_hi, void *out_lo, int B, int T, int C,
                                       int groups, float eps, void *stream) {
  HD_REQUIRE(x && gamma && beta && out_hi && B > 0 && T > 0 && C > 0 && groups > 0 && C % groups == 0 && T * (C / groups) <= 40 * 32,
             "hd_groupnorm_relu_split: bad arguments (T * C/groups must be <= 1280)");
  groupnorm_relu_split_kernel<<<hd::ceil_div((long long)B * groups, 4), 128, 0, (cudaStream_t)stream>>>(
      x, gamma, beta, reinterpret_cast<__half *>(out_hi), reinterpret_cast<__half *>(out_lo), B, T, C, groups, eps);
  return hd::check_launch("groupnorm_relu_split_kernel");
}

extern "C" int hd_split_f16(const float *x, void *hi, void *lo, long long n, void *stream) {
  HD_REQUIRE(x && hi && n > 0 && n % 4 == 0 && hd::aligned16(x) && hd::aligned16(hi) && hd::aligned16(lo), "hd_split_f16: bad arguments");
  split_f16_kernel<<<hd::ceil_div(n / 4, 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4 *>(x), reinterpret_cast<uint2 *>(hi),
                                                                              reinterpret_cast<uint2 *>(lo), n / 4);
  return hd::check_launch("split_f16_kernel");
}

extern "C" int hd_ief_fc1_theta(const float *P, const float *theta, int theta_ld, const float *W, int K, int C, void *out_hi, void *out_lo,
                                float *out_f32, int N, void *stream) {
  HD_REQUIRE(P && theta && W && (out_hi || out_f32) && (out_hi || !out_lo) && N > 0 && K > 0 && K <= 96 && theta_ld >= K &&
                 C > 0 && C % 4 == 0 && hd::aligned16(P) && hd::aligned16(W) && (!out_hi || (hd::aligned16(out_hi) && hd::aligned16(out_lo))) &&
                 (!out_f32 || hd::aligned16(out_f32)),
             "hd_ief_fc1_theta: bad arguments");
  ief_fc1_theta_kernel<<<hd::ceil_div(N, 8), 256, 0, (cudaStream_t)stream>>>(P, theta, theta_ld, W, K, C, reinterpret_cast<__half *>(out_hi),
                                                                            reinterpret_cast<__half *>(out_lo), out_f32, N,
                                                                            hd::DropoutSite{0, 0, 0, 1.f});
  return hd::check_launch("ief_fc1_theta_kernel");
}

extern "C" int hd_ief_fc1_theta_dropout(const float *P, const float *theta, int theta_ld, const float *W, int K, int C, void *out_hi,
                                        void *out_lo, float *out_f32, int N, unsigned long long seed, unsigned long long step, int site,
                                        float p, void *stream) {
  HD_REQUIRE(P && theta && W && (out_hi || out_f32) && (out_hi || !out_lo) && N > 0 && K > 0 && K <= 96 && theta_ld >= K &&
                 C > 0 && C % 4 == 0 && (long long)N * C <= (1ll << 34) && site >= 0 && p > 0.f && p <= 1.f && hd::aligned16(P) &&
                 hd::aligned16(W) && (!out_hi || (hd::aligned16(out_hi) && hd::aligned16(out_lo))) && (!out_f32 || hd::aligned16(out_f32)),
             "hd_ief_fc1_theta_dropout: bad arguments (0 < p <= 1, site >= 0, N*C <= 2^34)");
  ief_fc1_theta_kernel<<<hd::ceil_div(N, 8), 256, 0, (cudaStream_t)stream>>>(P, theta, theta_ld, W, K, C, reinterpret_cast<__half *>(out_hi),
                                                                            reinterpret_cast<__half *>(out_lo), out_f32, N,
                                                                            hd::DropoutSite{seed, step, (unsigned)site, p});
  return hd::check_launch("ief_fc1_theta_kernel");
}

namespace {

int launch_ief_fc3(const float *h2, const float *W, const float *bias, const float *prev, int prev_ld, float *out, int out_ld, int N, int K,
                   int D, const hd::DropoutSite &drop, float *h2_masked, void *stream) {
  const size_t smem = (size_t)(8 * K + 8 * 8 * 96) * sizeof(float);
  static bool configured[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && !configured[dev] && smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(ief_fc3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    if (e != cudaSuccess) { hd::set_last_error("ief_fc3 attr", e); return HD_ERR_CUDA; }
    configured[dev] = true;
  }
  HD_REQUIRE(smem <= 100 * 1024, "hd_ief_fc3: K too large");
  ief_fc3_kernel<<<hd::ceil_div(N, 8), 256, smem, (cudaStream_t)stream>>>(h2, W, bias, prev, prev_ld, out, out_ld, N, K, D, drop, h2_masked);
  return hd::check_launch("ief_fc3_kernel");
}

// One thread per group of 4 elements (one Philox call): out[w] = keep of element w, for w < N*C.
__global__ void dropout_mask_kernel(const hd::DropoutSite d, long long total, uint8_t *__restrict__ out) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g * 4 >= total) return;
  const uint4 w = hd::dropout_words(d, (unsigned long long)g);
  const uint32_t words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int e = 0; e < 4; ++e)
    if (g * 4 + e < total) out[g * 4 + e] = hd::dropout_keep(words[e], d.p) ? 1 : 0;
}

}  // namespace

extern "C" int hd_ief_fc3(const float *h2, const float *W, const float *bias, const float *prev, int prev_ld, float *out, int out_ld, int N,
                          int K, int D, void *stream) {
  HD_REQUIRE(h2 && W && bias && prev && out && N > 0 && K > 0 && K % 64 == 0 && D > 0 && D <= 96 && prev_ld >= D && out_ld >= D,
             "hd_ief_fc3: bad arguments (K % 64 == 0, D <= 96)");
  return launch_ief_fc3(h2, W, bias, prev, prev_ld, out, out_ld, N, K, D, hd::DropoutSite{0, 0, 0, 1.f}, nullptr, stream);
}

extern "C" int hd_ief_fc3_dropout(float *h2, const float *W, const float *bias, const float *prev, int prev_ld, float *out, int out_ld, int N,
                                  int K, int D, unsigned long long seed, unsigned long long step, int site, float p, void *stream) {
  HD_REQUIRE(h2 && W && bias && prev && out && N > 0 && K > 0 && K % 64 == 0 && D > 0 && D <= 96 && prev_ld >= D && out_ld >= D &&
                 (long long)N * K <= (1ll << 34) && site >= 0 && p > 0.f && p <= 1.f && hd::aligned16(h2),
             "hd_ief_fc3_dropout: bad arguments (K % 64 == 0, D <= 96, 0 < p <= 1, site >= 0, h2 16-byte aligned)");
  return launch_ief_fc3(h2, W, bias, prev, prev_ld, out, out_ld, N, K, D, hd::DropoutSite{seed, step, (unsigned)site, p}, h2, stream);
}

extern "C" int hd_dropout_mask(unsigned long long seed, unsigned long long step, int site, int N, int C, float p, unsigned char *out,
                               void *stream) {
  HD_REQUIRE(out && N > 0 && C > 0 && (long long)N * C <= (1ll << 34) && site >= 0 && p > 0.f && p <= 1.f,
             "hd_dropout_mask: bad arguments (N, C > 0, N*C <= 2^34, site >= 0, 0 < p <= 1)");
  const long long total = (long long)N * C;
  dropout_mask_kernel<<<hd::ceil_div((total + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(hd::DropoutSite{seed, step, (unsigned)site, p},
                                                                                          total, out);
  return hd::check_launch("dropout_mask_kernel");
}
