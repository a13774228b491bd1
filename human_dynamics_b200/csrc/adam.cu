// TensorFlow 1.8's ApplyAdam (training_ops.cc / training_ops_gpu.cu.cc, use_nesterov=False) over a list of fp32 tensors for sm_90a,
// one launch per HD_ADAM_MAX_TENSORS tensors plus one for the beta powers (include/hd_b200.h, hd_adam_tf).
//   adam_tf_kernel: CTA c takes chunk c of CHUNK elements; a prefix of the tensors' chunk counts (chunk0) maps it to (tensor, offset).
//                   Each element is read once (p, g, m, v) and written once (p, m, v); the gradient with a streaming hint.
//   adam_powers_kernel: TF's _finish, beta1_power *= beta1 and beta2_power *= beta2, after every tensor of the step.
// Built with -fmad=false (Makefile): every operation is rounded once, in the order below, so a float32 numpy restatement in the same
// order (oracle/adam_ref.py) is bit-identical.  The table travels by value as a __grid_constant__ parameter, as in losses.cu.
#include <climits>
#include <cmath>

#include "common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int VEC_PER_THREAD = 4;                            // float4 per thread per chunk
constexpr int CHUNK = THREADS * VEC_PER_THREAD * 4;          // 4096 elements per CTA

struct Params {
  hd_adam_tensor t[HD_ADAM_MAX_TENSORS];
  int chunk0[HD_ADAM_MAX_TENSORS + 1];                       // first chunk of each tensor; chunk0[n] = grid size
  int n;
  float lr, one_minus_beta1, one_minus_beta2, epsilon;
  const float *powers;
};
static_assert(sizeof(Params) < 32000, "kernel parameter limit");

__device__ __forceinline__ void update(float &p, float g, float &m, float &v, float alpha, float c1, float c2, float eps) {
  m = m + c1 * (g - m);
  v = v + c2 * (g * g - v);
  p = p - (alpha * m) / (eps + sqrtf(v));
}

__global__ void __launch_bounds__(THREADS) adam_tf_kernel(const __grid_constant__ Params P) {
  const int c = (int)blockIdx.x;
  int lo = 0, hi = P.n - 1;                                  // the last tensor whose first chunk is <= c
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (P.chunk0[mid] <= c) lo = mid;
    else hi = mid - 1;
  }
  const hd_adam_tensor &T = P.t[lo];
  // alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power), from the powers before this step's _finish
  const float b1p = P.powers[0], b2p = P.powers[1];
  const float alpha = (P.lr * sqrtf(1.f - b2p)) / (1.f - b1p);
  const float c1 = P.one_minus_beta1, c2 = P.one_minus_beta2, eps = P.epsilon;
  const long long s = (long long)(c - P.chunk0[lo]) * CHUNK;
  const long long e = min(T.numel, s + CHUNK);
  float *__restrict__ pp = T.param;
  const float *__restrict__ gp = T.grad;
  float *__restrict__ mp = T.m;
  float *__restrict__ vp = T.v;
  const bool aligned = ((reinterpret_cast<uintptr_t>(pp) | reinterpret_cast<uintptr_t>(gp) | reinterpret_cast<uintptr_t>(mp) |
                         reinterpret_cast<uintptr_t>(vp)) & 15) == 0;
  if (aligned) {
    const long long nv = (e - s) >> 2;                       // whole float4 of the chunk (s is a multiple of 4)
    float4 P4[VEC_PER_THREAD], G4[VEC_PER_THREAD], M4[VEC_PER_THREAD], V4[VEC_PER_THREAD];
#pragma unroll
    for (int k = 0; k < VEC_PER_THREAD; ++k) {
      const long long i = k * THREADS + threadIdx.x;
      if (i < nv) {
        const long long o = s + 4 * i;
        P4[k] = *reinterpret_cast<const float4 *>(pp + o);
        G4[k] = __ldcs(reinterpret_cast<const float4 *>(gp + o));
        M4[k] = *reinterpret_cast<const float4 *>(mp + o);
        V4[k] = *reinterpret_cast<const float4 *>(vp + o);
      }
    }
#pragma unroll
    for (int k = 0; k < VEC_PER_THREAD; ++k) {
      const long long i = k * THREADS + threadIdx.x;
      if (i < nv) {
        const long long o = s + 4 * i;
        update(P4[k].x, G4[k].x, M4[k].x, V4[k].x, alpha, c1, c2, eps);
        update(P4[k].y, G4[k].y, M4[k].y, V4[k].y, alpha, c1, c2, eps);
        update(P4[k].z, G4[k].z, M4[k].z, V4[k].z, alpha, c1, c2, eps);
        update(P4[k].w, G4[k].w, M4[k].w, V4[k].w, alpha, c1, c2, eps);
        *reinterpret_cast<float4 *>(pp + o) = P4[k];
        *reinterpret_cast<float4 *>(mp + o) = M4[k];
        *reinterpret_cast<float4 *>(vp + o) = V4[k];
      }
    }
    const long long tail = s + 4 * nv + threadIdx.x;         // the last numel % 4 elements of the tensor
    if (tail < e) {
      float p = pp[tail], m = mp[tail], v = vp[tail];
      update(p, __ldcs(gp + tail), m, v, alpha, c1, c2, eps);
      pp[tail] = p, mp[tail] = m, vp[tail] = v;
    }
    return;
  }
  for (long long i = s + threadIdx.x; i < e; i += THREADS) {
    float p = pp[i], m = mp[i], v = vp[i];
    update(p, __ldcs(gp + i), m, v, alpha, c1, c2, eps);
    pp[i] = p, mp[i] = m, vp[i] = v;
  }
}

__global__ void adam_powers_kernel(float *powers, float beta1, float beta2) {
  powers[0] = powers[0] * beta1;
  powers[1] = powers[1] * beta2;
}

}  // namespace

extern "C" {

int hd_adam_tf(const hd_adam_tensor *t, int n, float lr, float beta1, float beta2, float epsilon, float *powers, void *stream) {
  HD_REQUIRE(n >= 0 && (n == 0 || t), "hd_adam_tf: n < 0, or a NULL tensor table");
  HD_REQUIRE(powers, "hd_adam_tf: powers (device [2]: beta1_power, beta2_power) is NULL");
  HD_REQUIRE(std::isfinite(lr) && std::isfinite(beta1) && std::isfinite(beta2) && std::isfinite(epsilon),
             "hd_adam_tf: lr, beta1, beta2 and epsilon must be finite");
  for (int i = 0; i < n; ++i) {
    HD_REQUIRE(t[i].param && t[i].grad && t[i].m && t[i].v, "hd_adam_tf: a NULL param / grad / m / v pointer");
    HD_REQUIRE(t[i].numel >= 0, "hd_adam_tf: numel < 0");
  }
  for (int g0 = 0; g0 < n; g0 += HD_ADAM_MAX_TENSORS) {      // every group is checked before the first launch
    long long chunks = 0;
    for (int i = g0; i < n && i < g0 + HD_ADAM_MAX_TENSORS; ++i) chunks += (t[i].numel + CHUNK - 1) / CHUNK;
    HD_REQUIRE(chunks <= INT_MAX, "hd_adam_tf: more than 2^31 - 1 chunks in one launch");
  }
  static thread_local Params P;
  const cudaStream_t st = (cudaStream_t)stream;
  P.lr = lr, P.one_minus_beta1 = 1.f - beta1, P.one_minus_beta2 = 1.f - beta2, P.epsilon = epsilon, P.powers = powers;
  for (int g0 = 0; g0 < n; g0 += HD_ADAM_MAX_TENSORS) {
    const int m = n - g0 < HD_ADAM_MAX_TENSORS ? n - g0 : HD_ADAM_MAX_TENSORS;
    P.n = m;
    long long c = 0;
    for (int i = 0; i < m; ++i) {
      P.t[i] = t[g0 + i];
      P.chunk0[i] = (int)c;
      c += (t[g0 + i].numel + CHUNK - 1) / CHUNK;
    }
    P.chunk0[m] = (int)c;
    if (c == 0) continue;
    adam_tf_kernel<<<(unsigned)c, THREADS, 0, st>>>(P);
    const int e = hd::check_launch("adam_tf_kernel");
    if (e != HD_OK) return e;
  }
  adam_powers_kernel<<<1, 1, 0, st>>>(powers, beta1, beta2);
  return hd::check_launch("adam_powers_kernel");
}

}  // extern "C"
