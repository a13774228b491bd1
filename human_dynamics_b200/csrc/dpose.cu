// The adversarial pose prior D_pose (reference src/discriminators.py) for sm_90a: the kernels around its two 1024-wide FC layers,
// which run on hd_conv_gemm.  Forward of one batch of N poses (23 rotation matrices each):
//   trunk:  h1 = relu(x W1 + b1), h2 = relu(h1 W2 + b2) over the N*23 joint rows (the two 1x1 convs), logits[:, j] = h2[:, j] . wj[j] + bj[j]
//   fc1 / fc2 (hd_conv_gemm) on flatten(h2) = h2 viewed as [N, 736], then  out: logits[:, 23] = relu(fc2) . w_out + b_out.
// Backward: the fc layers' dX / dW are hd_conv_gemm again; the trunk backward here takes d flatten(h2) (fc1's dX) plus the heads' terms.
//
// Lane c of a warp owns channel c of one joint row, so every per-row sum (over the 9 inputs, the 32 channels, the 1024 features) runs in
// a fixed order inside one warp: a row's logits and input gradient depend on that row only, and are bit-identical across launches,
// batch splits and permutations.  Weight gradients use a fixed partition (64 poses per block, fixed warp order), partials written to a
// workspace, and a fixed-order second stage; nothing uses a floating-point atomic.
#include "conv_common.cuh"

namespace {

constexpr int J = HD_DPOSE_JOINTS;       // 23
constexpr int CH = 32;                   // channels of D_conv1 / D_conv2
constexpr int FLAT = J * CH;             // 736: fc1's input width
constexpr int HID = 1024;                // fc1 / fc2 width
constexpr int CHUNK = 64;                // poses per block of the backward (the fixed partition of the weight-gradient sums)
constexpr int BWD_WARPS = 4;
// one (chunk, joint) slot of the trunk partials: dW1 [9][32] | db1 [32] | dW2 [32][32] | db2 [32]
constexpr int SLOT_A = 9 * CH + CH + CH * CH + CH;          // 1376
constexpr int SLOT_B = J * CH + J;                          // 759: dwj [23][32] | dbj [23] per chunk
constexpr int SLOT_C = HID + 1;                             // 1025: dw_out [1024] | db_out per chunk
static_assert(SLOT_A + SLOT_B + SLOT_C == HD_DPOSE_GRAD_FLOATS, "packed gradient layout");

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One warp per joint row (n, j), lane = channel; 8 rows per warp.
__global__ void __launch_bounds__(256, 1) dpose_trunk_forward_kernel(const float *__restrict__ x, const float *__restrict__ W1,
                                                                  const float *__restrict__ b1, const float *__restrict__ W2,
                                                                  const float *__restrict__ b2, const float *__restrict__ wj,
                                                                  const float *__restrict__ bj, float *__restrict__ h1,
                                                                  float *__restrict__ h2, float *__restrict__ logits, long long rows) {
  const int c = threadIdx.x & 31;
  float w1[9], w2[CH];
#pragma unroll
  for (int i = 0; i < 9; ++i) w1[i] = __ldg(W1 + i * CH + c);
#pragma unroll
  for (int k = 0; k < CH; ++k) w2[k] = __ldg(W2 + k * CH + c);
  const float bb1 = __ldg(b1 + c), bb2 = __ldg(b2 + c);
  const long long r0 = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * 8;
  for (long long row = r0; row < r0 + 8 && row < rows; ++row) {
    const int j = (int)(row % J);
    const float xv = c < 9 ? __ldg(x + row * 9 + c) : 0.f;
    float a = 0.f;
#pragma unroll
    for (int i = 0; i < 9; ++i) a = fmaf(__shfl_sync(0xffffffffu, xv, i), w1[i], a);
    const float v1 = fmaxf(a + bb1, 0.f);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < CH; ++k) s = fmaf(__shfl_sync(0xffffffffu, v1, k), w2[k], s);
    const float v2 = fmaxf(s + bb2, 0.f);
    h1[row * CH + c] = v1;
    h2[row * CH + c] = v2;
    const float l = warp_sum(v2 * __ldg(wj + j * CH + c));
    if (c == 0) logits[(row / J) * (J + 1) + j] = l + __ldg(bj + j);
  }
}

// logits[n, 23] = h[n] . w + b: one warp per pose, lane-strided float4s, butterfly sum.
__global__ void __launch_bounds__(256) dpose_out_forward_kernel(const float *__restrict__ h, const float *__restrict__ w,
                                                                const float *__restrict__ b, float *__restrict__ logits, int N) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (n >= N) return;
  const float4 *hr = reinterpret_cast<const float4 *>(h + (size_t)n * HID);
  const float4 *wr = reinterpret_cast<const float4 *>(w);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < HID / 128; ++i) {
    const float4 a = __ldg(hr + i * 32 + lane), q = __ldg(wr + i * 32 + lane);
    s = fmaf(a.x, q.x, s); s = fmaf(a.y, q.y, s); s = fmaf(a.z, q.z, s); s = fmaf(a.w, q.w, s);
  }
  s = warp_sum(s);
  if (lane == 0) logits[(size_t)n * (J + 1) + J] = s + __ldg(b);
}

// Trunk backward.  Block (chunk, j), j < 23: poses [chunk*64, chunk*64 + 64) of joint j, warp w taking poses w, w + 4, ...; per row
//   d = dflat[n, j*32 + c] + g[n, j] * wj[j, c],  dp2 = d * (h2 > 0),  dp1 = (dp2 . W2^T) * (h1 > 0),  dx[n, j, :] = dp1 . W1^T
// and, with `part`, the block's sums of the trunk and head weight gradients.  Block (chunk, 23): the out layer's dw / db partials
// sum_n g[n, 23] * hf[n, :], sum_n g[n, 23] over the chunk.
__global__ void __launch_bounds__(BWD_WARPS * 32) dpose_trunk_backward_kernel(
    const float *__restrict__ x, const float *__restrict__ h1, const float *__restrict__ h2, const float *__restrict__ dflat,
    const float *__restrict__ g, const float *__restrict__ hf, const float *__restrict__ W1, const float *__restrict__ W2,
    const float *__restrict__ wj, float *__restrict__ dx, float *__restrict__ part, int N, int chunks) {
  __shared__ float w1s[9][33];
  __shared__ float red[BWD_WARPS][SLOT_A + CH + 1];
  const int chunk = blockIdx.x, j = blockIdx.y;
  const int n0 = chunk * CHUNK, n1 = min(N, n0 + CHUNK);
  if (j == J) {     // out layer partials (launched only with part)
    float *pc = part + (size_t)chunks * J * SLOT_A + (size_t)chunks * SLOT_B + (size_t)chunk * SLOT_C;
    for (int col = threadIdx.x; col < HID; col += blockDim.x) {
      float s = 0.f;
      for (int n = n0; n < n1; ++n) s = fmaf(__ldg(g + (size_t)n * (J + 1) + J), __ldg(hf + (size_t)n * HID + col), s);
      pc[col] = s;
    }
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int n = n0; n < n1; ++n) s += __ldg(g + (size_t)n * (J + 1) + J);
      pc[HID] = s;
    }
    return;
  }
  const int c = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (dx)
    for (int i = threadIdx.x; i < 9 * CH; i += blockDim.x) w1s[i / CH][i % CH] = __ldg(W1 + i);
  __syncthreads();
  float w2r[CH];                                           // row c of W2: dh1[c] = sum_k dp2[k] * W2[c, k]
#pragma unroll
  for (int k = 0; k < CH; ++k) w2r[k] = __ldg(W2 + c * CH + k);
  const float wjc = __ldg(wj + j * CH + c);
  float a2[CH], a1[9], sb1 = 0.f, sb2 = 0.f, sw = 0.f, sbj = 0.f;
#pragma unroll
  for (int k = 0; k < CH; ++k) a2[k] = 0.f;
#pragma unroll
  for (int i = 0; i < 9; ++i) a1[i] = 0.f;
  for (int n = n0 + wid; n < n1; n += BWD_WARPS) {
    const long long row = (long long)n * J + j;
    const float gj = __ldg(g + (size_t)n * (J + 1) + j);
    const float v2 = __ldg(h2 + row * CH + c), v1 = __ldg(h1 + row * CH + c);
    const float d = fmaf(gj, wjc, __ldg(dflat + (size_t)n * FLAT + j * CH + c));
    const float dp2 = v2 > 0.f ? d : 0.f;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < CH; ++k) s = fmaf(__shfl_sync(0xffffffffu, dp2, k), w2r[k], s);
    const float dp1 = v1 > 0.f ? s : 0.f;
    if (dx) {
      float t = 0.f;
      const int i = c < 9 ? c : 0;
#pragma unroll
      for (int k = 0; k < CH; ++k) t = fmaf(__shfl_sync(0xffffffffu, dp1, k), w1s[i][k], t);
      if (c < 9) dx[row * 9 + c] = t;
    }
    if (part) {
      const float xv = c < 9 ? __ldg(x + row * 9 + c) : 0.f;
#pragma unroll
      for (int k = 0; k < CH; ++k) a2[k] = fmaf(__shfl_sync(0xffffffffu, v1, k), dp2, a2[k]);
#pragma unroll
      for (int i = 0; i < 9; ++i) a1[i] = fmaf(__shfl_sync(0xffffffffu, xv, i), dp1, a1[i]);
      sb1 += dp1;
      sb2 += dp2;
      sw = fmaf(gj, v2, sw);
      sbj += gj;
    }
  }
  if (!part) return;
  float *r = red[wid];
#pragma unroll
  for (int i = 0; i < 9; ++i) r[i * CH + c] = a1[i];
  r[9 * CH + c] = sb1;
#pragma unroll
  for (int k = 0; k < CH; ++k) r[10 * CH + k * CH + c] = a2[k];
  r[10 * CH + CH * CH + c] = sb2;
  r[SLOT_A + c] = sw;
  if (c == 0) r[SLOT_A + CH] = sbj;
  __syncthreads();
  float *pa = part + ((size_t)chunk * J + j) * SLOT_A;
  float *pb = part + (size_t)chunks * J * SLOT_A + (size_t)chunk * SLOT_B;
  for (int i = threadIdx.x; i < SLOT_A + CH + 1; i += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < BWD_WARPS; ++w) s += red[w][i];
    if (i < SLOT_A) pa[i] = s;
    else if (i < SLOT_A + CH) pb[j * CH + (i - SLOT_A)] = s;
    else pb[J * CH + j] = s;
  }
}

// Second stage: column sums of the three partial tables in a fixed order (8 row slices per column, then the slices in order), written
// to the packed gradient [A | B | C].  Block b < 43: table A (rows chunks*23), < 67: B (rows chunks), else C (rows chunks).
__global__ void __launch_bounds__(256) dpose_grad_reduce_kernel(const float *__restrict__ part, int chunks, float *__restrict__ grad) {
  __shared__ float ps[8][33];
  constexpr int BA = (SLOT_A + 31) / 32, BB = (SLOT_B + 31) / 32;
  const int lane = threadIdx.x & 31, sl = threadIdx.x >> 5;
  int blk = blockIdx.x, cols, out_off;
  long long rows;
  const float *src;
  if (blk < BA) {
    src = part, rows = (long long)chunks * J, cols = SLOT_A, out_off = 0;
  } else if (blk < BA + BB) {
    blk -= BA;
    src = part + (size_t)chunks * J * SLOT_A, rows = chunks, cols = SLOT_B, out_off = SLOT_A;
  } else {
    blk -= BA + BB;
    src = part + (size_t)chunks * J * SLOT_A + (size_t)chunks * SLOT_B, rows = chunks, cols = SLOT_C, out_off = SLOT_A + SLOT_B;
  }
  const int col = blk * 32 + lane;
  float s = 0.f;
  if (col < cols)
    for (long long r = sl; r < rows; r += 8) s += __ldg(src + r * cols + col);
  ps[sl][lane] = s;
  __syncthreads();
  if (sl == 0 && col < cols) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += ps[k][lane];
    grad[out_off + col] = t;
  }
}

inline int dpose_chunks(int N) { return hd::ceil_div(N, CHUNK); }

}  // namespace

extern "C" {

size_t hd_dpose_workspace_bytes(int N) {
  if (N <= 0) return 0;
  const size_t S = (size_t)dpose_chunks(N);
  return (S * J * SLOT_A + S * SLOT_B + S * SLOT_C) * sizeof(float);
}

int hd_dpose_trunk_forward(const float *x, const float *W1, const float *b1, const float *W2, const float *b2, const float *wj,
                           const float *bj, float *h1, float *h2, float *logits, int N, void *stream) {
  HD_REQUIRE(x && W1 && b1 && W2 && b2 && wj && bj && h1 && h2 && logits && N > 0, "hd_dpose_trunk_forward: null pointer or N <= 0");
  const long long rows = (long long)N * J;
  dpose_trunk_forward_kernel<<<hd::ceil_div(rows, 64), 256, 0, (cudaStream_t)stream>>>(x, W1, b1, W2, b2, wj, bj, h1, h2, logits, rows);
  return hd::check_launch("dpose_trunk_forward_kernel");
}

int hd_dpose_out_forward(const float *h, const float *w, const float *b, float *logits, int N, void *stream) {
  HD_REQUIRE(h && w && b && logits && N > 0 && hd::aligned16(h) && hd::aligned16(w),
             "hd_dpose_out_forward: null pointer, N <= 0 or h / w not 16-byte aligned");
  dpose_out_forward_kernel<<<hd::ceil_div(N, 8), 256, 0, (cudaStream_t)stream>>>(h, w, b, logits, N);
  return hd::check_launch("dpose_out_forward_kernel");
}

int hd_dpose_trunk_backward(const float *x, const float *h1, const float *h2, const float *dflat, const float *g, const float *hf,
                            const float *W1, const float *W2, const float *wj, float *dx, void *ws, size_t ws_bytes, int N, void *stream) {
  HD_REQUIRE(h1 && h2 && dflat && g && W2 && wj && N > 0 && (dx || ws) && (!dx || W1) && (!ws || (x && hf)),
             "hd_dpose_trunk_backward: null pointer, N <= 0 or neither dx nor ws (ws needs x and hf, dx needs W1)");
  HD_REQUIRE(!ws || ws_bytes >= hd_dpose_workspace_bytes(N), "hd_dpose_trunk_backward: workspace smaller than hd_dpose_workspace_bytes(N)");
  const int S = dpose_chunks(N);
  dim3 grid((unsigned)S, ws ? J + 1 : J);
  dpose_trunk_backward_kernel<<<grid, BWD_WARPS * 32, 0, (cudaStream_t)stream>>>(x, h1, h2, dflat, g, hf, W1, W2, wj, dx, (float *)ws, N, S);
  return hd::check_launch("dpose_trunk_backward_kernel");
}

int hd_dpose_grad_reduce(const void *ws, size_t ws_bytes, int N, float *grad, void *stream) {
  HD_REQUIRE(ws && grad && N > 0 && ws_bytes >= hd_dpose_workspace_bytes(N), "hd_dpose_grad_reduce: null pointer, N <= 0 or workspace too small");
  const int blocks = (SLOT_A + 31) / 32 + (SLOT_B + 31) / 32 + (SLOT_C + 31) / 32;
  dpose_grad_reduce_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const float *)ws, dpose_chunks(N), grad);
  return hd::check_launch("dpose_grad_reduce_kernel");
}

}  // extern "C"
