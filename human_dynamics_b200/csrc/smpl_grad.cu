// Batched SMPL backward for sm_90a: skinning + keypoint backward, FK + Rodrigues backward, and the backward of the standalone
// helpers (batch_rodrigues, batch_global_rigid_transformation, batch_orth_proj_idrot).
//
// Reverse mode of src/tf_smpl/batch_smpl.py:89-162, batch_lbs.py:42-60,133-194 and projection.py:16-29.  Nothing here uses a
// floating-point atomic: each reduction is owned by one thread or one warp and runs in a fixed order, so the gradients of pose n
// depend only on pose n and are bit-identical across launches, batch sizes and permutations.
#include "smpl_common.cuh"

using hd_smpl::Tree;
using hd_smpl::build_tree;
using hd_smpl::rodrigues;
using hd_smpl::fk_chain;

namespace {

constexpr int kTile = HD_SMPL_GRAD_TILE;   // vertices per tile of the skinning backward
constexpr int kLbsPT = 4;                  // poses per CTA of the skinning backward
constexpr int kMaxKps = 64;
constexpr int kLbsThreads = 288;           // one thread per (joint, entry of A) in the reduction; the first kTile also own a vertex

// Skinning + keypoint backward.  CTA = kLbsPT poses walking every vertex tile; threads < kTile own one vertex in the vertex phase.
//   g_v       = dverts_v + sum_k Kreg[k,v] djoints_k                 (vertex-major regressor, fixed order)
//   dv_posed  = (sum_k w_vk R_k)^T g_v
//   dA_k(r,c) += sum_{v in tile} w_vk g_v[r] [v_posed_v; 1][c]      (joint-major tile lists; thread (k, r, c) walks joint k's list
//                                                                    once for all kLbsPT poses)
template <int NNZ>
__global__ void __launch_bounds__(kLbsThreads) smpl_lbs_backward_kernel(
    const float *__restrict__ v_posed, long long vp_ld, const float *__restrict__ A12, const float *__restrict__ dverts,
    const float *__restrict__ djoints, const int *__restrict__ lbs_idx, const float *__restrict__ lbs_w, int nnz_rt,
    const int *__restrict__ kpv_ptr, const int *__restrict__ kpv_kidx, const float *__restrict__ kpv_w, int K,
    const int *__restrict__ lbt_ptr, const int *__restrict__ lbt_v, const float *__restrict__ lbt_w, int num_tiles,
    float *__restrict__ dv_posed, float *__restrict__ dA12, int N, int V) {
  extern __shared__ __align__(16) float smem[];
  float *As = smem;                          // [PT][288]
  float *gAs = As + kLbsPT * 288;            // [PT][288]
  float *P = gAs + kLbsPT * 288;             // [PT][12][kTile]
  float *gJ = P + kLbsPT * 12 * kTile;       // [PT][K*3]
  const int tid = threadIdx.x;
  const int p0 = blockIdx.x * kLbsPT;
  for (int i = tid; i < kLbsPT * 288; i += kLbsThreads) {
    const int p = i / 288;
    As[i] = (p0 + p < N) ? __ldg(A12 + (size_t)p0 * 288 + i) : 0.f;
    gAs[i] = 0.f;
  }
  for (int i = tid; i < kLbsPT * K * 3; i += kLbsThreads) {
    const int p = i / (K * 3);
    gJ[i] = (djoints && p0 + p < N) ? __ldg(djoints + (size_t)p0 * K * 3 + i) : 0.f;
  }
  // padding columns of dv_posed are the zero K-tail of the dc GEMM
  for (int p = 0; p < kLbsPT; ++p) {
    const int n = p0 + p;
    if (n >= N) break;
    for (long long k = (long long)V * 3 + tid; k < vp_ld; k += kLbsThreads) dv_posed[(size_t)n * vp_ld + k] = 0.f;
  }
  __syncthreads();
  const int nnz = NNZ > 0 ? NNZ : nnz_rt;
  for (int t = 0; t < num_tiles; ++t) {
    const int v = t * kTile + tid;
    if (tid < kTile && v < V) {
      int jid[NNZ > 0 ? NNZ : 1];
      float jw[NNZ > 0 ? NNZ : 1];
      if (NNZ > 0) {
#pragma unroll
        for (int e = 0; e < (NNZ > 0 ? NNZ : 1); ++e) { jid[e] = __ldg(lbs_idx + (size_t)v * NNZ + e) * 12; jw[e] = __ldg(lbs_w + (size_t)v * NNZ + e); }
      }
      const int kb = __ldg(kpv_ptr + v), ke = __ldg(kpv_ptr + v + 1);
#pragma unroll 1
      for (int p = 0; p < kLbsPT; ++p) {
        const int n = p0 + p;
        float *Pp = P + p * 12 * kTile + tid;
        if (n >= N) {
#pragma unroll
          for (int i = 0; i < 12; ++i) Pp[i * kTile] = 0.f;
          continue;
        }
        const float *dv = dverts + ((size_t)n * V + v) * 3;
        float g0 = __ldg(dv), g1 = __ldg(dv + 1), g2 = __ldg(dv + 2);
        const float *gj = gJ + p * K * 3;
        for (int e = kb; e < ke; ++e) {
          const int k = __ldg(kpv_kidx + e) * 3;
          const float w = __ldg(kpv_w + e);
          g0 += w * gj[k]; g1 += w * gj[k + 1]; g2 += w * gj[k + 2];
        }
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
        const float *vp = v_posed + (size_t)n * vp_ld + (size_t)v * 3;
        const float x = __ldg(vp), y = __ldg(vp + 1), z = __ldg(vp + 2);
        float *o = dv_posed + (size_t)n * vp_ld + (size_t)v * 3;
        o[0] = T[0] * g0 + T[4] * g1 + T[8] * g2;
        o[1] = T[1] * g0 + T[5] * g1 + T[9] * g2;
        o[2] = T[2] * g0 + T[6] * g1 + T[10] * g2;
        const float g[3] = {g0, g1, g2};
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          Pp[(r * 4 + 0) * kTile] = g[r] * x;
          Pp[(r * 4 + 1) * kTile] = g[r] * y;
          Pp[(r * 4 + 2) * kTile] = g[r] * z;
          Pp[(r * 4 + 3) * kTile] = g[r];
        }
      }
    }
    __syncthreads();
    {
      const int k = tid / 12, i = tid % 12;
      const float *Pi = P + i * kTile - t * kTile;
      const int eb = __ldg(lbt_ptr + t * 24 + k), ee = __ldg(lbt_ptr + t * 24 + k + 1);
      float acc[kLbsPT];
#pragma unroll
      for (int p = 0; p < kLbsPT; ++p) acc[p] = 0.f;
#pragma unroll 2
      for (int e = eb; e < ee; ++e) {
        const float w = __ldg(lbt_w + e);
        const int vv = __ldg(lbt_v + e);
#pragma unroll
        for (int p = 0; p < kLbsPT; ++p) acc[p] += w * Pi[p * 12 * kTile + vv];
      }
#pragma unroll
      for (int p = 0; p < kLbsPT; ++p) gAs[p * 288 + tid] += acc[p];
    }
    __syncthreads();
  }
  for (int i = tid; i < kLbsPT * 288; i += kLbsThreads) {
    const int p = i / 288;
    if (p0 + p < N) dA12[(size_t)p0 * 288 + i] = gAs[i];
  }
}

// d/dtheta of R = rodrigues(theta) (batch_lbs.py:42-60) in fp64, the reference's expression including the +1e-8 shift:
//   angle = |theta + eps|, r = theta / angle, R = cos I + (1 - cos) r r^T + sin [r]x.
// At theta = 0 it is finite and gives dR = [dtheta]x up to O(eps).
__device__ __forceinline__ void rodrigues_backward(float tx, float ty, float tz, const float *G, float *gth) {
  const double th[3] = {(double)tx, (double)ty, (double)tz};
  const double eps = 1e-8;
  const double s[3] = {th[0] + eps, th[1] + eps, th[2] + eps};
  const double angle = sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
  const double r[3] = {th[0] / angle, th[1] / angle, th[2] / angle};
  double sn, c;
  sincos(angle, &sn, &c);
  double g[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) g[i] = (double)G[i];
  double gc = g[0] + g[4] + g[8];                       // d/dcos of cos I + (1 - cos) r r^T
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) gc -= g[a * 3 + b] * r[a] * r[b];
  const double w[3] = {g[7] - g[5], g[2] - g[6], g[3] - g[1]};   // sum_ij G_ij d[r]x_ij / dr
  const double gsn = r[0] * w[0] + r[1] * w[1] + r[2] * w[2];
  double gr[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double acc = 0.0;
#pragma unroll
    for (int b = 0; b < 3; ++b) acc += (g[a * 3 + b] + g[b * 3 + a]) * r[b];
    gr[a] = (1.0 - c) * acc + sn * w[a];
  }
  const double inv = 1.0 / angle;
  const double gangle = -sn * gc + c * gsn - (gr[0] * th[0] + gr[1] * th[1] + gr[2] * th[2]) * inv * inv;
#pragma unroll
  for (int a = 0; a < 3; ++a) gth[a] = (float)(gr[a] * inv + gangle * s[a] * inv);
}

// Reverse of fk_chain + the A = [Rw | tw - Rw J] construction (batch_lbs.py:160-194), one lane per joint.
// In: local rotation Rl, rest joint J, dA (rows of [R | t], 12), dtw (gradient on the joint's world position, new_J / J_transformed).
// Out: dRl (gradient on the local rotation), dJ (gradient on J).  Children are added to their parent in ascending joint order.
__device__ __forceinline__ void fk_backward(const Tree &tree, int lane, const float *Rl, const float *J, const float *dA,
                                            const float *dtw_in, float *dRl, float *dJ) {
  const bool active = lane < 24;
  const int par = active ? tree.parent[lane] : 0;
  const int dep = active ? tree.depth[lane] : -1;
  float Rw[9], tw[3], tl[3];
  fk_chain(tree, lane, Rl, J, Rw, tw);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float jp = __shfl_sync(0xffffffffu, J[c], par);
    tl[c] = (dep == 0) ? J[c] : J[c] - jp;
  }
  float gRw[9], gtw[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float gt = active ? dA[r * 4 + 3] : 0.f;
    gtw[r] = gt + (active ? dtw_in[r] : 0.f);
#pragma unroll
    for (int c = 0; c < 3; ++c) gRw[r * 3 + c] = active ? dA[r * 4 + c] - gt * J[c] : 0.f;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    dJ[c] = active ? -(Rw[0 * 3 + c] * dA[3] + Rw[1 * 3 + c] * dA[7] + Rw[2 * 3 + c] * dA[11]) : 0.f;
  }
#pragma unroll
  for (int i = 0; i < 9; ++i) dRl[i] = 0.f;
  for (int level = tree.maxdepth; level >= 1; --level) {
    float pR[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) pR[i] = __shfl_sync(0xffffffffu, Rw[i], par);
    float cR[9], ct[3], cJ[3];                       // this joint's contributions to its parent
#pragma unroll
    for (int i = 0; i < 9; ++i) cR[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) { ct[i] = 0.f; cJ[i] = 0.f; }
    if (dep == level) {
      // Rw = pR Rl:  dRl += pR^T dRw;  dpR += dRw Rl^T.   tw = pR tl + pt:  dpR += dtw tl^T;  dtl = pR^T dtw;  dpt += dtw
#pragma unroll
      for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          dRl[a * 3 + c] += pR[0 * 3 + a] * gRw[0 * 3 + c] + pR[1 * 3 + a] * gRw[1 * 3 + c] + pR[2 * 3 + a] * gRw[2 * 3 + c];
      }
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int a = 0; a < 3; ++a)
          cR[r * 3 + a] = gRw[r * 3 + 0] * Rl[a * 3 + 0] + gRw[r * 3 + 1] * Rl[a * 3 + 1] + gRw[r * 3 + 2] * Rl[a * 3 + 2] + gtw[r] * tl[a];
        ct[r] = gtw[r];
      }
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float gtl = pR[0 * 3 + a] * gtw[0] + pR[1 * 3 + a] * gtw[1] + pR[2 * 3 + a] * gtw[2];
        dJ[a] += gtl;                                  // tl = J - J_parent
        cJ[a] = -gtl;
      }
    }
    for (int src = 1; src < 24; ++src) {              // warp-uniform: the tree is a kernel parameter
      if (tree.depth[src] != level) continue;
      const bool mine = tree.parent[src] == lane;
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        const float x = __shfl_sync(0xffffffffu, cR[i], src);
        if (mine) gRw[i] += x;
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const float x = __shfl_sync(0xffffffffu, ct[i], src);
        const float y = __shfl_sync(0xffffffffu, cJ[i], src);
        if (mine) { gtw[i] += x; dJ[i] += y; }
      }
    }
  }
  if (dep == 0) {                                      // root: Rw = Rl, tw = J
#pragma unroll
    for (int i = 0; i < 9; ++i) dRl[i] += gRw[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) dJ[i] += gtw[i];
  }
}

// One warp per pose.  Recomputes J and R as smpl_pose_kernel does, then FK backward, the Rs / pose-blend gradients, Rodrigues
// backward and the beta reduction (butterfly over the lanes: fixed order).
__global__ void __launch_bounds__(128) smpl_pose_backward_kernel(Tree tree, const float *__restrict__ beta, int beta_ld,
                                                                 const float *__restrict__ theta, int theta_ld,
                                                                 const float *__restrict__ J_template,
                                                                 const float *__restrict__ J_shapedirs, const float *__restrict__ dA12,
                                                                 const float *__restrict__ dc, int dc_ld, const float *__restrict__ dRs,
                                                                 const float *__restrict__ dJtr, float *__restrict__ dbeta, int dbeta_ld,
                                                                 float *__restrict__ dtheta, int dtheta_ld, int N) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  const int j = lane < 24 ? lane : 23;
  float J[3], R[9];
#pragma unroll
  for (int c = 0; c < 3; ++c) J[c] = 0.f;
#pragma unroll
  for (int b = 0; b < 10; ++b) {
    const float bb = __ldg(beta + (size_t)n * beta_ld + b);
#pragma unroll
    for (int c = 0; c < 3; ++c) J[c] += bb * __ldg(J_shapedirs + b * 72 + j * 3 + c);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) J[c] += __ldg(J_template + j * 3 + c);
  const float *th = theta + (size_t)n * theta_ld + j * 3;
  const float t0 = __ldg(th), t1 = __ldg(th + 1), t2 = __ldg(th + 2);
  rodrigues(t0, t1, t2, R);
  float gA[12], gt[3];
#pragma unroll
  for (int i = 0; i < 12; ++i) gA[i] = dA12 ? __ldg(dA12 + ((size_t)n * 24 + j) * 12 + i) : 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) gt[i] = dJtr ? __ldg(dJtr + ((size_t)n * 24 + j) * 3 + i) : 0.f;
  float gR[9], gJ[3];
  fk_backward(tree, lane, R, J, gA, gt, gR, gJ);
  if (dRs) {
#pragma unroll
    for (int i = 0; i < 9; ++i) gR[i] += __ldg(dRs + ((size_t)n * 24 + j) * 9 + i);
  }
  if (dc && lane >= 1 && lane < 24) {                  // pose_feature = vec(R_j - I), j = 1..23 (batch_smpl.py:127-128)
#pragma unroll
    for (int i = 0; i < 9; ++i) gR[i] += __ldg(dc + (size_t)n * dc_ld + 10 + (lane - 1) * 9 + i);
  }
  if (lane < 24) {
    float gth[3];
    rodrigues_backward(t0, t1, t2, gR, gth);
    float *o = dtheta + (size_t)n * dtheta_ld + lane * 3;
    o[0] = gth[0]; o[1] = gth[1]; o[2] = gth[2];
  }
#pragma unroll
  for (int b = 0; b < 10; ++b) {
    float v = lane < 24 ? gJ[0] * __ldg(J_shapedirs + b * 72 + j * 3 + 0) + gJ[1] * __ldg(J_shapedirs + b * 72 + j * 3 + 1) +
                              gJ[2] * __ldg(J_shapedirs + b * 72 + j * 3 + 2)
                        : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == b) dbeta[(size_t)n * dbeta_ld + b] = v + (dc ? __ldg(dc + (size_t)n * dc_ld + b) : 0.f);
  }
}

__global__ void rodrigues_backward_kernel(const float *__restrict__ theta, const float *__restrict__ dR, float *__restrict__ dtheta, int M) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  float G[9], g[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) G[k] = dR[(size_t)i * 9 + k];
  rodrigues_backward(theta[(size_t)i * 3], theta[(size_t)i * 3 + 1], theta[(size_t)i * 3 + 2], G, g);
  dtheta[(size_t)i * 3 + 0] = g[0]; dtheta[(size_t)i * 3 + 1] = g[1]; dtheta[(size_t)i * 3 + 2] = g[2];
}

__global__ void __launch_bounds__(128) global_rigid_backward_kernel(Tree tree, const float *__restrict__ Rs, const float *__restrict__ Js,
                                                                    const float *__restrict__ dnew_J, const float *__restrict__ dA44,
                                                                    float *__restrict__ dRs, float *__restrict__ dJs, int N, int rotate_base) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  const int j = lane < 24 ? lane : 23;
  float R[9], J[3], gA[12], gt[3];
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = __ldg(Rs + ((size_t)n * 24 + j) * 9 + i);
#pragma unroll
  for (int i = 0; i < 3; ++i) J[i] = __ldg(Js + ((size_t)n * 24 + j) * 3 + i);
  const bool flip = rotate_base && lane == 0;           // Rs[:,0] . diag(1,-1,-1), batch_lbs.py:151-156
  if (flip) {
#pragma unroll
    for (int r = 0; r < 3; ++r) { R[r * 3 + 1] = -R[r * 3 + 1]; R[r * 3 + 2] = -R[r * 3 + 2]; }
  }
#pragma unroll
  for (int i = 0; i < 12; ++i) gA[i] = dA44 ? __ldg(dA44 + ((size_t)n * 24 + j) * 16 + i) : 0.f;   // rows 0..2; row 3 is constant
#pragma unroll
  for (int i = 0; i < 3; ++i) gt[i] = dnew_J ? __ldg(dnew_J + ((size_t)n * 24 + j) * 3 + i) : 0.f;
  float gR[9], gJ[3];
  fk_backward(tree, lane, R, J, gA, gt, gR, gJ);
  if (flip) {
#pragma unroll
    for (int r = 0; r < 3; ++r) { gR[r * 3 + 1] = -gR[r * 3 + 1]; gR[r * 3 + 2] = -gR[r * 3 + 2]; }
  }
  if (lane < 24) {
#pragma unroll
    for (int i = 0; i < 9; ++i) dRs[((size_t)n * 24 + lane) * 9 + i] = gR[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) dJs[((size_t)n * 24 + lane) * 3 + i] = gJ[i];
  }
}

// One warp per pose: dX written per point, the camera gradient reduced over the points in a fixed (lane-strided + butterfly) order.
__global__ void __launch_bounds__(128) orth_proj_backward_kernel(const float *__restrict__ X, const float *__restrict__ cam,
                                                                 const float *__restrict__ dout, float *__restrict__ dX,
                                                                 float *__restrict__ dcam, int N, int P) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  const float s = cam[(size_t)n * 3], tx = cam[(size_t)n * 3 + 1], ty = cam[(size_t)n * 3 + 2];
  float gs = 0.f, gx = 0.f, gy = 0.f;
  for (int p = lane; p < P; p += 32) {
    const size_t i = (size_t)n * P + p;
    const float ox = dout[i * 2], oy = dout[i * 2 + 1];
    dX[i * 3 + 0] = s * ox;
    dX[i * 3 + 1] = s * oy;
    dX[i * 3 + 2] = 0.f;
    gs += (X[i * 3 + 0] + tx) * ox + (X[i * 3 + 1] + ty) * oy;
    gx += ox;
    gy += oy;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    gs += __shfl_xor_sync(0xffffffffu, gs, o);
    gx += __shfl_xor_sync(0xffffffffu, gx, o);
    gy += __shfl_xor_sync(0xffffffffu, gy, o);
  }
  if (lane == 0) {
    dcam[(size_t)n * 3 + 0] = gs;
    dcam[(size_t)n * 3 + 1] = s * gx;
    dcam[(size_t)n * 3 + 2] = s * gy;
  }
}

size_t lbs_backward_smem(int K) { return (size_t)(2 * kLbsPT * 288 + kLbsPT * 12 * kTile + kLbsPT * K * 3) * sizeof(float); }

constexpr int kMaxDevices = 64;

template <int NNZ>
int launch_lbs_backward(const hd_smpl_consts *c, const hd_smpl_grad_consts *g, const float *v_posed, long long vp_ld, const float *A12,
                        const float *dverts, const float *djoints, float *dv_posed, float *dA12, int N, cudaStream_t st) {
  const size_t smem = lbs_backward_smem(kMaxKps);
  // function attributes are per device: a process may drive several GPUs through this library
  static bool configured[kMaxDevices] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) { hd::set_last_error_text("smpl_lbs_backward: device ordinal out of range"); return HD_ERR_UNSUPPORTED; }
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(smpl_lbs_backward_kernel<NNZ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { hd::set_last_error("smpl_lbs_backward attr", e); return HD_ERR_CUDA; }
    configured[dev] = true;
  }
  smpl_lbs_backward_kernel<NNZ><<<hd::ceil_div(N, kLbsPT), kLbsThreads, lbs_backward_smem(c->num_kps), st>>>(
      v_posed, vp_ld, A12, dverts, djoints, c->lbs_idx, c->lbs_w, c->lbs_nnz, g->kpv_ptr, g->kpv_kidx, g->kpv_w, c->num_kps, g->lbt_ptr,
      g->lbt_v, g->lbt_w, g->num_tiles, dv_posed, dA12, N, c->num_verts);
  return hd::check_launch("smpl_lbs_backward_kernel");
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

}  // namespace

extern "C" {

size_t hd_smpl_backward_workspace_bytes(int N, int V) {
  if (N <= 0 || V <= 0) return 0;
  const size_t n = (size_t)N, vp_ld = ((size_t)V * 3 + 3) / 4 * 4;
  return align256(n * 288 * 4) * 2 + align256(n * HD_SMPL_GRAD_CLD * 4) + align256(n * 216 * 4) + align256(n * 256 * 2) * 2 +
         align256(n * vp_ld * 4) * 2;
}

int hd_smpl_lbs_backward(const hd_smpl_consts *c, const hd_smpl_grad_consts *g, const float *v_posed, long long vp_ld, const float *A12,
                         const float *dverts, const float *djoints, float *dv_posed, float *dA12, int N, void *stream) {
  HD_REQUIRE(c && g && v_posed && A12 && dverts && dv_posed && dA12 && N >= 0, "hd_smpl_lbs_backward: null pointer or N < 0");
  HD_REQUIRE(c->num_verts > 0 && c->lbs_nnz >= 1 && c->lbs_nnz <= 24 && c->num_kps >= 0 && c->num_kps <= kMaxKps &&
                 g->num_verts == c->num_verts && g->num_kps == c->num_kps && g->tile_verts == kTile &&
                 g->num_tiles == hd::ceil_div(c->num_verts, kTile) && g->kpv_ptr && g->lbt_ptr && g->lbt_v && g->lbt_w,
             "hd_smpl_lbs_backward: consts / grad consts mismatch (num_kps <= 64, tile_verts = HD_SMPL_GRAD_TILE)");
  HD_REQUIRE(vp_ld >= (long long)c->num_verts * 3, "hd_smpl_lbs_backward: vp_ld < 3V");
  if (N == 0) return HD_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (c->lbs_nnz == 4) return launch_lbs_backward<4>(c, g, v_posed, vp_ld, A12, dverts, djoints, dv_posed, dA12, N, st);
  return launch_lbs_backward<0>(c, g, v_posed, vp_ld, A12, dverts, djoints, dv_posed, dA12, N, st);
}

int hd_smpl_pose_backward(const hd_smpl_consts *c, const float *beta, int beta_ld, const float *theta, int theta_ld, int N,
                          const float *dA12, const float *dc, int dc_ld, const float *dRs, const float *dJtr, float *dbeta, int dbeta_ld,
                          float *dtheta, int dtheta_ld, void *stream) {
  HD_REQUIRE(c && beta && theta && dbeta && dtheta && N >= 0 && beta_ld >= 10 && theta_ld >= 72 && dbeta_ld >= 10 && dtheta_ld >= 72 &&
                 (!dc || dc_ld >= 217),
             "hd_smpl_pose_backward: bad arguments");
  if (N == 0) return HD_OK;
  Tree tree;
  if (!build_tree(c->parents, tree)) { hd::set_last_error_text("hd_smpl_pose_backward: parents must satisfy parent[i] < i"); return HD_ERR_INVALID; }
  smpl_pose_backward_kernel<<<hd::ceil_div(N, 4), 128, 0, (cudaStream_t)stream>>>(tree, beta, beta_ld, theta, theta_ld, c->J_template,
                                                                                   c->J_shapedirs, dA12, dc, dc_ld, dRs, dJtr, dbeta,
                                                                                   dbeta_ld, dtheta, dtheta_ld, N);
  return hd::check_launch("smpl_pose_backward_kernel");
}

int hd_rodrigues_backward(const float *theta, const float *dR, float *dtheta, int M, void *stream) {
  HD_REQUIRE(theta && dR && dtheta && M >= 0, "hd_rodrigues_backward: bad arguments");
  if (M == 0) return HD_OK;
  rodrigues_backward_kernel<<<hd::ceil_div(M, 256), 256, 0, (cudaStream_t)stream>>>(theta, dR, dtheta, M);
  return hd::check_launch("rodrigues_backward_kernel");
}

int hd_global_rigid_backward(const float *Rs, const float *Js, const int *parents_host, const float *dnew_J, const float *dA44, float *dRs,
                             float *dJs, int N, int rotate_base, void *stream) {
  HD_REQUIRE(Rs && Js && parents_host && dRs && dJs && N >= 0, "hd_global_rigid_backward: bad arguments");
  if (N == 0) return HD_OK;
  Tree tree;
  if (!build_tree(parents_host, tree)) { hd::set_last_error_text("hd_global_rigid_backward: parents must satisfy parent[i] < i"); return HD_ERR_INVALID; }
  global_rigid_backward_kernel<<<hd::ceil_div(N, 4), 128, 0, (cudaStream_t)stream>>>(tree, Rs, Js, dnew_J, dA44, dRs, dJs, N, rotate_base);
  return hd::check_launch("global_rigid_backward_kernel");
}

int hd_orth_proj_backward(const float *X, const float *cam, const float *dout, float *dX, float *dcam, int N, int P, void *stream) {
  HD_REQUIRE(X && cam && dout && dX && dcam && N >= 0 && P >= 0, "hd_orth_proj_backward: bad arguments");
  if (N == 0) return HD_OK;
  orth_proj_backward_kernel<<<hd::ceil_div(N, 4), 128, 0, (cudaStream_t)stream>>>(X, cam, dout, dX, dcam, N, P);
  return hd::check_launch("orth_proj_backward_kernel");
}

}  // extern "C"
