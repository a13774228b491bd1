// Batched SMPL forward for sm_90a: Rodrigues + 24-joint FK (warp-shuffle tree walk), fused
// shape/pose blend + linear-blend skinning, keypoint regression + orthographic projection.
//
// Replaces src/tf_smpl/batch_smpl.py:89-162, batch_lbs.py:15-60,133-194, projection.py:16-29 of the
// reference (one TF op + HBM round trip per line there; three kernels and no materialised W/T here).
#include "conv_common.cuh"
#include "smpl_common.cuh"

namespace {

using hd_smpl::Tree;
using hd_smpl::build_tree;
using hd_smpl::rodrigues;
using hd_smpl::fk_chain;

// One warp per pose.  Writes Rs [N,24,9], Jtr [N,24,3] (optional), A12 [N,24,12] (rows of [R | t - R J]).
__global__ void __launch_bounds__(128) smpl_pose_kernel(Tree tree, const float *__restrict__ beta, int beta_ld,
                                                        const float *__restrict__ theta, int theta_ld,
                                                        const float *__restrict__ J_template,
                                                        const float *__restrict__ J_shapedirs, float *__restrict__ Rs,
                                                        float *__restrict__ Rs_out, float *__restrict__ Jtr,
                                                        float *__restrict__ A12, int N, int out_mul, int out_off,
                                                        float *__restrict__ coef, int coef_ld, __half *__restrict__ coef_hi,
                                                        __half *__restrict__ coef_lo, __half *__restrict__ a12t_hi,
                                                        __half *__restrict__ a12t_lo) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  const int j = lane < 24 ? lane : 23;
  float J[3], R[9];
#pragma unroll
  for (int c = 0; c < 3; ++c) J[c] = 0.f;
#pragma unroll
  for (int b = 0; b < 10; ++b) {                       // J = (beta . shapedirs + v_template) . J_regressor
    const float bb = __ldg(beta + (size_t)n * beta_ld + b);
#pragma unroll
    for (int c = 0; c < 3; ++c) J[c] += bb * __ldg(J_shapedirs + b * 72 + j * 3 + c);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) J[c] += __ldg(J_template + j * 3 + c);
  const float *th = theta + (size_t)n * theta_ld + j * 3;
  rodrigues(__ldg(th), __ldg(th + 1), __ldg(th + 2), R);
  float Rw[9], tw[3];
  fk_chain(tree, lane, R, J, Rw, tw);
  if (lane < 24) {
    const size_t no = (size_t)n * out_mul + out_off;
    {
      float *o = Rs + ((size_t)n * 24 + lane) * 9;
#pragma unroll
      for (int i = 0; i < 9; ++i) o[i] = R[i];
    }
    if (Rs_out) {
      float *o = Rs_out + (no * 24 + lane) * 9;
#pragma unroll
      for (int i = 0; i < 9; ++i) o[i] = R[i];
    }
    if (Jtr) {
      float *o = Jtr + (no * 24 + lane) * 3;
      o[0] = tw[0]; o[1] = tw[1]; o[2] = tw[2];
    }
    if (coef) {        // blend-GEMM operand row: [beta(10) | (R_j - I), j = 1..23 (207) | 0 ...]  (batch_smpl.py:110,127-128)
      float *cr = coef + (size_t)n * coef_ld;
      if (lane == 0) {
#pragma unroll
        for (int b = 0; b < 10; ++b) cr[b] = __ldg(beta + (size_t)n * beta_ld + b);
        for (int k = 217; k < coef_ld; ++k) cr[k] = 0.f;
      } else {
#pragma unroll
        for (int i = 0; i < 9; ++i) cr[10 + (lane - 1) * 9 + i] = R[i] - ((i == 0 || i == 4 || i == 8) ? 1.0f : 0.0f);
      }
    }
    if (coef_hi) {     // the same operand row, pre-split into the fp16 head / 2^11-scaled remainder pair the tensor-core kernel loads
      __half *ch = coef_hi + (size_t)n * coef_ld, *cl = coef_lo + (size_t)n * coef_ld;
      auto put = [&](int k, float x) {
        uint32_t h, l;
        hd::split_f16x2(x, 0.f, h, l);
        ch[k] = __ushort_as_half((unsigned short)(h & 0xffffu));
        cl[k] = __ushort_as_half((unsigned short)(l & 0xffffu));
      };
      if (lane == 0) {
#pragma unroll
        for (int b = 0; b < 10; ++b) put(b, __ldg(beta + (size_t)n * beta_ld + b));
        for (int k = 217; k < coef_ld; ++k) put(k, 0.f);
      } else {
#pragma unroll
        for (int i = 0; i < 9; ++i) put(10 + (lane - 1) * 9 + i, R[i] - ((i == 0 || i == 4 || i == 8) ? 1.0f : 0.0f));
      }
    }
    float4 *a = reinterpret_cast<float4 *>(A12 + ((size_t)n * 24 + lane) * 12);
    float av[12];
#pragma unroll
    for (int r = 0; r < 3; ++r) {                      // A = results - pad(results . [J;0]), batch_lbs.py:188-192
      const float ib = Rw[r * 3 + 0] * J[0] + Rw[r * 3 + 1] * J[1] + Rw[r * 3 + 2] * J[2];
      a[r] = make_float4(Rw[r * 3 + 0], Rw[r * 3 + 1], Rw[r * 3 + 2], tw[r] - ib);
      av[r * 4 + 0] = Rw[r * 3 + 0]; av[r * 4 + 1] = Rw[r * 3 + 1]; av[r * 4 + 2] = Rw[r * 3 + 2]; av[r * 4 + 3] = tw[r] - ib;
    }
    if (a12t_hi) {     // B operand of the tensor-core skinning GEMM (smpl_lbs_tc.cu): [n][entry i][joint k, 32 wide] as an UNSCALED fp16
                       // head / remainder pair (entries are O(1): the remainder stays far above the fp16 subnormal floor in absolute terms)
#pragma unroll
      for (int i = 0; i < 12; ++i) {
        const __half h = __float2half_rn(av[i]);
        a12t_hi[((size_t)n * 12 + i) * 32 + lane] = h;
        a12t_lo[((size_t)n * 12 + i) * 32 + lane] = __float2half_rn(av[i] - __half2float(h));
      }
    }
  } else if (a12t_hi) {                                // joints 24..31: the zero padding of K
#pragma unroll
    for (int i = 0; i < 12; ++i) {
      a12t_hi[((size_t)n * 12 + i) * 32 + lane] = __float2half_rn(0.f);
      a12t_lo[((size_t)n * 12 + i) * 32 + lane] = __float2half_rn(0.f);
    }
  }
}

constexpr int kNumDirs = 217;  // 10 shape + 207 pose basis rows

// Fused blend + skinning.  CTA = 128 vertices x PT poses; one vertex per thread, PT poses in registers.
//   v_posed = v_template + beta.shapedirs + (Rs[1:]-I).posedirs      (batch_smpl.py:110-112,127-133)
//   verts   = (sum_k w_k A_k) [v_posed;1]                             (batch_smpl.py:141-151)
template <int PT, int NNZ>
__global__ void __launch_bounds__(128) smpl_skin_kernel(const float *__restrict__ v_template,
                                                        const float *__restrict__ dirs,
                                                        const int *__restrict__ lbs_idx,
                                                        const float *__restrict__ lbs_w, int nnz_rt,
                                                        const float *__restrict__ beta, int beta_ld, const float *__restrict__ Rs,
                                                        const float *__restrict__ A12, float *__restrict__ verts,
                                                        int N, int V, int out_mul, int out_off) {
  extern __shared__ __align__(16) float smem[];
  float *coef = smem;                        // [kNumDirs][PT]
  float *As = smem + kNumDirs * PT;          // [PT][24*12]
  const int p0 = blockIdx.x * PT;
  const int tid = threadIdx.x;
  for (int i = tid; i < kNumDirs * PT; i += 128) {
    const int k = i / PT, p = i % PT;
    const int n = p0 + p;
    float c = 0.f;
    if (n < N) {
      if (k < 10) c = __ldg(beta + (size_t)n * beta_ld + k);
      else {
        const int q = k - 10;                 // pose_feature index: joint 1+q/9, entry q%9
        const int e = q % 9;
        c = __ldg(Rs + (size_t)n * 216 + 9 + q) - ((e == 0 || e == 4 || e == 8) ? 1.0f : 0.0f);
      }
    }
    coef[k * PT + p] = c;
  }
  for (int i = tid; i < PT * 288; i += 128) {
    const int p = i / 288;
    As[i] = (p0 + p < N) ? __ldg(A12 + (size_t)p0 * 288 + i) : 0.f;
  }
  __syncthreads();

  const int v = blockIdx.y * 128 + tid;
  const int vc = v < V ? v : V - 1;
  float acc[PT][3];
  {
    const float t0 = __ldg(v_template + vc * 3 + 0), t1 = __ldg(v_template + vc * 3 + 1), t2 = __ldg(v_template + vc * 3 + 2);
#pragma unroll
    for (int p = 0; p < PT; ++p) { acc[p][0] = t0; acc[p][1] = t1; acc[p][2] = t2; }
  }
  const float *dptr = dirs + (size_t)vc * 3;
  const size_t dstride = (size_t)V * 3;
#pragma unroll 4
  for (int k = 0; k < kNumDirs; ++k) {
    const float d0 = __ldg(dptr + k * dstride), d1 = __ldg(dptr + k * dstride + 1), d2 = __ldg(dptr + k * dstride + 2);
    const float4 *c4 = reinterpret_cast<const float4 *>(coef + k * PT);
#pragma unroll
    for (int q = 0; q < PT / 4; ++q) {
      const float4 c = c4[q];
      acc[4 * q + 0][0] += c.x * d0; acc[4 * q + 0][1] += c.x * d1; acc[4 * q + 0][2] += c.x * d2;
      acc[4 * q + 1][0] += c.y * d0; acc[4 * q + 1][1] += c.y * d1; acc[4 * q + 1][2] += c.y * d2;
      acc[4 * q + 2][0] += c.z * d0; acc[4 * q + 2][1] += c.z * d1; acc[4 * q + 2][2] += c.z * d2;
      acc[4 * q + 3][0] += c.w * d0; acc[4 * q + 3][1] += c.w * d1; acc[4 * q + 3][2] += c.w * d2;
    }
  }

  int jid[NNZ > 0 ? NNZ : 1];
  float jw[NNZ > 0 ? NNZ : 1];
  const int nnz = NNZ > 0 ? NNZ : nnz_rt;
  if (NNZ > 0) {
#pragma unroll
    for (int e = 0; e < NNZ; ++e) { jid[e] = __ldg(lbs_idx + (size_t)vc * NNZ + e) * 12; jw[e] = __ldg(lbs_w + (size_t)vc * NNZ + e); }
  }
#pragma unroll
  for (int p = 0; p < PT; ++p) {
    float T[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) T[i] = 0.f;
    const float *Ap = As + p * 288;
    if (NNZ > 0) {
#pragma unroll
      for (int e = 0; e < (NNZ > 0 ? NNZ : 1); ++e) {
        const float4 *a = reinterpret_cast<const float4 *>(Ap + jid[e]);
        const float w = jw[e];
        const float4 a0 = a[0], a1 = a[1], a2 = a[2];
        T[0] += w * a0.x; T[1] += w * a0.y; T[2] += w * a0.z; T[3] += w * a0.w;
        T[4] += w * a1.x; T[5] += w * a1.y; T[6] += w * a1.z; T[7] += w * a1.w;
        T[8] += w * a2.x; T[9] += w * a2.y; T[10] += w * a2.z; T[11] += w * a2.w;
      }
    } else {
      for (int e = 0; e < nnz; ++e) {
        const int jj = __ldg(lbs_idx + (size_t)vc * nnz + e) * 12;
        const float w = __ldg(lbs_w + (size_t)vc * nnz + e);
        const float4 *a = reinterpret_cast<const float4 *>(Ap + jj);
        const float4 a0 = a[0], a1 = a[1], a2 = a[2];
        T[0] += w * a0.x; T[1] += w * a0.y; T[2] += w * a0.z; T[3] += w * a0.w;
        T[4] += w * a1.x; T[5] += w * a1.y; T[6] += w * a1.z; T[7] += w * a1.w;
        T[8] += w * a2.x; T[9] += w * a2.y; T[10] += w * a2.z; T[11] += w * a2.w;
      }
    }
    const float x = acc[p][0], y = acc[p][1], z = acc[p][2];
    const int n = p0 + p;
    if (n < N && v < V) {
      float *o = verts + (((size_t)n * out_mul + out_off) * V + v) * 3;
      o[0] = T[0] * x + T[1] * y + T[2] * z + T[3];
      o[1] = T[4] * x + T[5] * y + T[6] * z + T[7];
      o[2] = T[8] * x + T[9] * y + T[10] * z + T[11];
    }
  }
}

// Skinning only: verts = (sum_k w_k A_k) [v_posed;1] with v_posed already blended (tensor-core GEMM).  HBM-bound:
// reads v_posed, writes verts.  CTA = 128 vertices x PT poses; A of the PT poses in smem.
template <int PT, int NNZ>
__global__ void __launch_bounds__(128) smpl_lbs_kernel(const float *__restrict__ v_posed, long long vp_ld,
                                                       const int *__restrict__ lbs_idx, const float *__restrict__ lbs_w,
                                                       int nnz_rt, const float *__restrict__ A12, float *__restrict__ verts,
                                                       int N, int V, int out_mul, int out_off) {
  __shared__ __align__(16) float As[PT * 288];
  const int p0 = blockIdx.x * PT;
  const int tid = threadIdx.x;
  for (int i = tid; i < PT * 288; i += 128) As[i] = (p0 + i / 288 < N) ? __ldg(A12 + (size_t)p0 * 288 + i) : 0.f;
  __syncthreads();
  const int v = blockIdx.y * 128 + tid;
  if (v >= V) return;
  const int nnz = NNZ > 0 ? NNZ : nnz_rt;
  int jid[NNZ > 0 ? NNZ : 1];
  float jw[NNZ > 0 ? NNZ : 1];
  if (NNZ > 0) {
#pragma unroll
    for (int e = 0; e < NNZ; ++e) { jid[e] = __ldg(lbs_idx + (size_t)v * NNZ + e) * 12; jw[e] = __ldg(lbs_w + (size_t)v * NNZ + e); }
  }
#pragma unroll 4
  for (int p = 0; p < PT; ++p) {
    const int n = p0 + p;
    if (n >= N) break;
    const float *vp = v_posed + (size_t)n * vp_ld + (size_t)v * 3;
    const float x = __ldg(vp), y = __ldg(vp + 1), z = __ldg(vp + 2);
    float T[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) T[i] = 0.f;
    const float *Ap = As + p * 288;
    for (int e = 0; e < nnz; ++e) {
      const int jj = NNZ > 0 ? jid[e < (NNZ > 0 ? NNZ : 1) ? e : 0] : __ldg(lbs_idx + (size_t)v * nnz + e) * 12;
      const float w = NNZ > 0 ? jw[e < (NNZ > 0 ? NNZ : 1) ? e : 0] : __ldg(lbs_w + (size_t)v * nnz + e);
      const float4 *a = reinterpret_cast<const float4 *>(Ap + jj);
      const float4 a0 = a[0], a1 = a[1], a2 = a[2];
      T[0] += w * a0.x; T[1] += w * a0.y; T[2] += w * a0.z; T[3] += w * a0.w;
      T[4] += w * a1.x; T[5] += w * a1.y; T[6] += w * a1.z; T[7] += w * a1.w;
      T[8] += w * a2.x; T[9] += w * a2.y; T[10] += w * a2.z; T[11] += w * a2.w;
    }
    float *o = verts + (((size_t)n * out_mul + out_off) * V + v) * 3;
    o[0] = T[0] * x + T[1] * y + T[2] * z + T[3];
    o[1] = T[4] * x + T[5] * y + T[6] * z + T[7];
    o[2] = T[8] * x + T[9] * y + T[10] * z + T[11];
  }
}

// joints = verts . joint_regressor (batch_smpl.py:154-157) + projection s*(xy + t) (projection.py:25-29).
// One CTA per pose; a warp walks the non-zeros of one keypoint column at a time (deterministic order).
__global__ void __launch_bounds__(128) smpl_joints_kernel(const float *__restrict__ verts, const int *__restrict__ kp_ptr,
                                                          const int *__restrict__ kp_vidx, const float *__restrict__ kp_w,
                                                          const float *__restrict__ cam, int cam_ld, float *__restrict__ joints,
                                                          float *__restrict__ kps, int V, int K, int out_mul, int out_off) {
  const int n = blockIdx.x;
  const size_t no = (size_t)n * out_mul + out_off;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float *vp = verts + no * V * 3;
  for (int k = warp; k < K; k += 4) {
    const int b = __ldg(kp_ptr + k), e = __ldg(kp_ptr + k + 1);
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int i = b + lane; i < e; i += 32) {
      const int vi = __ldg(kp_vidx + i);
      const float w = __ldg(kp_w + i);
      sx += w * vp[vi * 3 + 0]; sy += w * vp[vi * 3 + 1]; sz += w * vp[vi * 3 + 2];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sx += __shfl_xor_sync(0xffffffffu, sx, o);
      sy += __shfl_xor_sync(0xffffffffu, sy, o);
      sz += __shfl_xor_sync(0xffffffffu, sz, o);
    }
    if (lane == 0) {
      if (joints) {
        float *o = joints + (no * K + k) * 3;
        o[0] = sx; o[1] = sy; o[2] = sz;
      }
      if (kps) {
        const float s = __ldg(cam + (size_t)n * cam_ld), tx = __ldg(cam + (size_t)n * cam_ld + 1), ty = __ldg(cam + (size_t)n * cam_ld + 2);
        kps[(no * K + k) * 2 + 0] = s * (sx + tx);
        kps[(no * K + k) * 2 + 1] = s * (sy + ty);
      }
    }
  }
}

__global__ void rodrigues_kernel(const float *__restrict__ theta, float *__restrict__ R, int M) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  float r[9];
  rodrigues(theta[(size_t)i * 3], theta[(size_t)i * 3 + 1], theta[(size_t)i * 3 + 2], r);
#pragma unroll
  for (int k = 0; k < 9; ++k) R[(size_t)i * 9 + k] = r[k];
}

// batch_global_rigid_transformation with explicit Rs / Js inputs; A written as full 4x4.
__global__ void __launch_bounds__(128) global_rigid_kernel(Tree tree, const float *__restrict__ Rs,
                                                           const float *__restrict__ Js, float *__restrict__ new_J,
                                                           float *__restrict__ A44, int N, int rotate_base) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  const int j = lane < 24 ? lane : 23;
  float R[9], J[3];
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = __ldg(Rs + ((size_t)n * 24 + j) * 9 + i);
#pragma unroll
  for (int i = 0; i < 3; ++i) J[i] = __ldg(Js + ((size_t)n * 24 + j) * 3 + i);
  if (rotate_base && lane == 0) {          // Rs[:,0] . diag(1,-1,-1), batch_lbs.py:151-156
#pragma unroll
    for (int r = 0; r < 3; ++r) { R[r * 3 + 1] = -R[r * 3 + 1]; R[r * 3 + 2] = -R[r * 3 + 2]; }
  }
  float Rw[9], tw[3];
  fk_chain(tree, lane, R, J, Rw, tw);
  if (lane < 24) {
    float *nj = new_J + ((size_t)n * 24 + lane) * 3;
    nj[0] = tw[0]; nj[1] = tw[1]; nj[2] = tw[2];
    float4 *a = reinterpret_cast<float4 *>(A44 + ((size_t)n * 24 + lane) * 16);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float ib = Rw[r * 3 + 0] * J[0] + Rw[r * 3 + 1] * J[1] + Rw[r * 3 + 2] * J[2];
      a[r] = make_float4(Rw[r * 3 + 0], Rw[r * 3 + 1], Rw[r * 3 + 2], tw[r] - ib);
    }
    a[3] = make_float4(0.f, 0.f, 0.f, 1.f);
  }
}

// batch_rot2aa (src/tf_smpl/batch_lbs.py:63-105), one thread per matrix (hd_smpl::rot2aa).
__global__ void rot2aa_kernel(const float *__restrict__ Rs, float *__restrict__ aa, int M) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  hd_smpl::rot2aa(Rs + (size_t)i * 9, aa + (size_t)i * 3);
}

__global__ void orth_proj_kernel(const float *__restrict__ X, const float *__restrict__ cam, float *__restrict__ out,
                                 long long total, int P) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // over N*P points
  if (i >= total) return;
  const long long n = i / P;
  const float s = cam[n * 3], tx = cam[n * 3 + 1], ty = cam[n * 3 + 2];
  out[i * 2 + 0] = s * (X[i * 3 + 0] + tx);
  out[i * 2 + 1] = s * (X[i * 3 + 1] + ty);
}

constexpr int kMaxDevices = 64;

template <int PT, int NNZ>
int launch_skin(const hd_smpl_consts *c, const float *beta, int beta_ld, const float *Rs, const float *A12, float *verts, int N,
                int out_mul, int out_off, cudaStream_t st) {
  const size_t smem = (size_t)(kNumDirs * PT + PT * 288) * sizeof(float);
  // function attributes are per device: a process may drive several GPUs through this library
  static bool configured[kMaxDevices] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) { hd::set_last_error_text("smpl_skin: device ordinal out of range"); return HD_ERR_UNSUPPORTED; }
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(smpl_skin_kernel<PT, NNZ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { hd::set_last_error("smpl_skin attr", e); return HD_ERR_CUDA; }
    configured[dev] = true;
  }
  dim3 grid(hd::ceil_div(N, PT), hd::ceil_div(c->num_verts, 128));
  smpl_skin_kernel<PT, NNZ><<<grid, 128, smem, st>>>(c->v_template, c->dirs, c->lbs_idx, c->lbs_w, c->lbs_nnz, beta, beta_ld, Rs,
                                                     A12, verts, N, c->num_verts, out_mul, out_off);
  return hd::check_launch("smpl_skin_kernel");
}

}  // namespace

extern "C" {

size_t hd_smpl_workspace_bytes(int N) {
  return (size_t)N * 24 * (12 + 9) * sizeof(float) + 256;
}

int hd_smpl_forward(const hd_smpl_consts *c, const float *beta, int beta_ld, const float *theta, int theta_ld, int N,
                    float *verts, float *joints, float *Rs, float *Jtr, const float *cam, int cam_ld, float *kps,
                    int out_mul, int out_off, void *ws, size_t ws_bytes, void *stream) {
  HD_REQUIRE(c && beta && theta && verts && ws, "hd_smpl_forward: null pointer");
  HD_REQUIRE(N >= 0 && beta_ld >= 10 && theta_ld >= 72 && (!cam || cam_ld >= 3) && out_mul >= 1 && out_off >= 0 && out_off < out_mul,
             "hd_smpl_forward: bad N / leading dimensions / output interleave");
  HD_REQUIRE((cam == nullptr) == (kps == nullptr), "hd_smpl_forward: cam and kps must be given together");
  HD_REQUIRE(c->lbs_nnz >= 1 && c->lbs_nnz <= 24 && c->num_verts > 0 && c->num_kps >= 0, "hd_smpl_forward: bad consts");
  if (N == 0) return HD_OK;
  if (ws_bytes < hd_smpl_workspace_bytes(N)) return HD_ERR_WORKSPACE;
  Tree tree;
  if (!build_tree(c->parents, tree)) { hd::set_last_error_text("hd_smpl_forward: parents must satisfy parent[i] < i"); return HD_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  float *A12 = reinterpret_cast<float *>(ws);
  float *Rs_w = A12 + (size_t)N * 288;
  smpl_pose_kernel<<<hd::ceil_div(N, 4), 128, 0, st>>>(tree, beta, beta_ld, theta, theta_ld, c->J_template, c->J_shapedirs, Rs_w, Rs, Jtr, A12, N, out_mul, out_off, nullptr, 0, nullptr, nullptr, nullptr, nullptr);
  int rc = hd::check_launch("smpl_pose_kernel");
  if (rc) return rc;
  const bool big = N >= 32 * 132;        // enough 32-pose blocks to fill the 132 SMs of an H100
  if (c->lbs_nnz == 4) rc = big ? launch_skin<32, 4>(c, beta, beta_ld, Rs_w, A12, verts, N, out_mul, out_off, st) : launch_skin<8, 4>(c, beta, beta_ld, Rs_w, A12, verts, N, out_mul, out_off, st);
  else rc = big ? launch_skin<32, 0>(c, beta, beta_ld, Rs_w, A12, verts, N, out_mul, out_off, st) : launch_skin<8, 0>(c, beta, beta_ld, Rs_w, A12, verts, N, out_mul, out_off, st);
  if (rc) return rc;
  if ((joints || kps) && c->num_kps > 0) {
    smpl_joints_kernel<<<N, 128, 0, st>>>(verts, c->kp_ptr, c->kp_vidx, c->kp_w, cam, cam_ld, joints, kps, c->num_verts, c->num_kps, out_mul, out_off);
    rc = hd::check_launch("smpl_joints_kernel");
  }
  return rc;
}

// ---- staged SMPL (tensor-core blend): pose -> [hd_conv_gemm: v_posed = coef . dirs + v_template] -> lbs -> joints ----
int hd_smpl_pose(const hd_smpl_consts *c, const float *beta, int beta_ld, const float *theta, int theta_ld, int N, float *Rs,
                 float *Jtr, float *A12, float *coef, int coef_ld, void *coef_hi, void *coef_lo, void *a12t_hi, void *a12t_lo, int out_mul,
                 int out_off, void *ws, size_t ws_bytes, void *stream) {
  HD_REQUIRE(c && beta && theta && A12 && ws && N > 0 && beta_ld >= 10 && theta_ld >= 72 && out_mul >= 1 && out_off >= 0 &&
                 out_off < out_mul && ((!coef && !coef_hi) || coef_ld >= 217) && ((coef_hi == nullptr) == (coef_lo == nullptr)) &&
                 ((a12t_hi == nullptr) == (a12t_lo == nullptr)),
             "hd_smpl_pose: bad arguments");
  if (ws_bytes < (size_t)N * 216 * sizeof(float)) return HD_ERR_WORKSPACE;
  Tree tree;
  if (!build_tree(c->parents, tree)) { hd::set_last_error_text("hd_smpl_pose: parents must satisfy parent[i] < i"); return HD_ERR_INVALID; }
  smpl_pose_kernel<<<hd::ceil_div(N, 4), 128, 0, (cudaStream_t)stream>>>(tree, beta, beta_ld, theta, theta_ld, c->J_template,
                                                                          c->J_shapedirs, reinterpret_cast<float *>(ws), Rs, Jtr,
                                                                          A12, N, out_mul, out_off, coef, coef_ld,
                                                                          reinterpret_cast<__half *>(coef_hi), reinterpret_cast<__half *>(coef_lo),
                                                                          reinterpret_cast<__half *>(a12t_hi), reinterpret_cast<__half *>(a12t_lo));
  return hd::check_launch("smpl_pose_kernel");
}

int hd_smpl_lbs(const hd_smpl_consts *c, const float *v_posed, long long vp_ld, const float *A12, float *verts, int N, int out_mul,
                int out_off, void *stream) {
  HD_REQUIRE(c && v_posed && A12 && verts && N > 0 && vp_ld >= (long long)c->num_verts * 3 && out_mul >= 1 && out_off >= 0 &&
                 out_off < out_mul,
             "hd_smpl_lbs: bad arguments");
  dim3 grid(hd::ceil_div(N, 16), hd::ceil_div(c->num_verts, 128));
  if (c->lbs_nnz == 4)
    smpl_lbs_kernel<16, 4><<<grid, 128, 0, (cudaStream_t)stream>>>(v_posed, vp_ld, c->lbs_idx, c->lbs_w, 4, A12, verts, N, c->num_verts, out_mul, out_off);
  else
    smpl_lbs_kernel<16, 0><<<grid, 128, 0, (cudaStream_t)stream>>>(v_posed, vp_ld, c->lbs_idx, c->lbs_w, c->lbs_nnz, A12, verts, N, c->num_verts, out_mul, out_off);
  return hd::check_launch("smpl_lbs_kernel");
}

int hd_smpl_joints(const hd_smpl_consts *c, const float *verts, const float *cam, int cam_ld, float *joints, float *kps, int N,
                   int out_mul, int out_off, void *stream) {
  HD_REQUIRE(c && verts && N > 0 && (joints || kps) && (!kps || (cam && cam_ld >= 3)) && out_mul >= 1 && out_off >= 0 && out_off < out_mul,
             "hd_smpl_joints: bad arguments");
  if (c->num_kps == 0) return HD_OK;
  smpl_joints_kernel<<<N, 128, 0, (cudaStream_t)stream>>>(verts, c->kp_ptr, c->kp_vidx, c->kp_w, cam, cam_ld, joints, kps, c->num_verts,
                                                         c->num_kps, out_mul, out_off);
  return hd::check_launch("smpl_joints_kernel");
}

int hd_rodrigues(const float *theta, float *R, int M, void *stream) {
  HD_REQUIRE(theta && R && M >= 0, "hd_rodrigues: bad arguments");
  if (M == 0) return HD_OK;
  rodrigues_kernel<<<hd::ceil_div(M, 256), 256, 0, (cudaStream_t)stream>>>(theta, R, M);
  return hd::check_launch("rodrigues_kernel");
}

int hd_rot2aa(const float *Rs, float *aa, int M, void *stream) {
  HD_REQUIRE(Rs && aa && M >= 0, "hd_rot2aa: bad arguments");
  if (M == 0) return HD_OK;
  rot2aa_kernel<<<hd::ceil_div(M, 256), 256, 0, (cudaStream_t)stream>>>(Rs, aa, M);
  return hd::check_launch("rot2aa_kernel");
}

int hd_global_rigid(const float *Rs, const float *Js, const int *parents_host, float *new_J, float *A44, int N,
                    int rotate_base, void *stream) {
  HD_REQUIRE(Rs && Js && parents_host && new_J && A44 && N >= 0, "hd_global_rigid: bad arguments");
  if (N == 0) return HD_OK;
  Tree tree;
  if (!build_tree(parents_host, tree)) { hd::set_last_error_text("hd_global_rigid: parents must satisfy parent[i] < i"); return HD_ERR_INVALID; }
  global_rigid_kernel<<<hd::ceil_div(N, 4), 128, 0, (cudaStream_t)stream>>>(tree, Rs, Js, new_J, A44, N, rotate_base);
  return hd::check_launch("global_rigid_kernel");
}

int hd_orth_proj(const float *X, const float *cam, float *out, int N, int P, void *stream) {
  HD_REQUIRE(X && cam && out && N >= 0 && P >= 0, "hd_orth_proj: bad arguments");
  const long long total = (long long)N * P;
  if (total == 0) return HD_OK;
  orth_proj_kernel<<<hd::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(X, cam, out, total, P);
  return hd::check_launch("orth_proj_kernel");
}

}  // extern "C"
