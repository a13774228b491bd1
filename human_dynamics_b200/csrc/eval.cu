// The per-frame metrics of the reference's evaluation (src/evaluation/eval.py compute_errors_batched over eval_util.py) for sm_90a:
//   eval_frames_kernel   one warp per frame: 2-D keypoint error / optimal-camera error / PCK (lane = keypoint), MPJPE and PA-MPJPE
//                        (lane = joint; the similarity transform through Horn's quaternion eigenproblem, Jacobi in registers), the
//                        prediction's acceleration and the acceleration error inside the frame's tube;
//   mesh_tpose_kernel    one block per frame: the T-pose mesh distance in closed form from the shape blend and the skinning weights;
//   verts_error_kernel   one block per frame: mean vertex distance between two meshes.
// All reductions run in a fixed order (warp butterflies, shared-memory trees): no atomics, bit-identical across launches and batchings.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int FRAMES_PER_BLOCK = 4;      // warps per block of eval_frames_kernel
constexpr int MESH_THREADS = 256;

__device__ __forceinline__ double nan_d() { return __longlong_as_double(0x7ff8000000000000ULL); }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide fixed-order sum; every thread gets the result.
__device__ double block_sum(double v, double *sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
#pragma unroll 1
  for (int s = MESH_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  double r = sh[0];
  __syncthreads();
  return r;
}

// One Jacobi rotation zeroing a[p][q] of the symmetric 4x4 a; v accumulates the eigenvectors as columns.
template <int p, int q>
__device__ __forceinline__ void jacobi_rotate(double (&a)[4][4], double (&v)[4][4]) {
  const double apq = a[p][q];
  if (apq == 0.0) return;
  const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
  double t = fabs(theta) > 1e150 ? 0.5 / theta : copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
  const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
  for (int k = 0; k < 4; ++k) {          // columns p, q of a . J
    const double akp = a[k][p], akq = a[k][q];
    a[k][p] = c * akp - s * akq;
    a[k][q] = s * akp + c * akq;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {          // rows p, q of J^T . (a . J)
    const double apk = a[p][k], aqk = a[q][k];
    a[p][k] = c * apk - s * aqk;
    a[q][k] = s * apk + c * aqk;
  }
  a[p][q] = a[q][p] = 0.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double vkp = v[k][p], vkq = v[k][q];
    v[k][p] = c * vkp - s * vkq;
    v[k][q] = s * vkp + c * vkq;
  }
}

// The rotation R (row-major) that maximises trace(R K) = sum_j y_j . R x_j over proper rotations, K = sum_j x_j y_j^T: the unit
// eigenvector of Horn's symmetric 4x4 matrix with the largest eigenvalue, as a quaternion.  This is the reference's
// R = V diag(1, 1, sign(det(U V^T))) U^T from the SVD K = U S V^T.  K = 0 gives R = I.
__device__ void best_rotation(const double (&K)[3][3], double (&R)[3][3]) {
  const double sxx = K[0][0], sxy = K[0][1], sxz = K[0][2], syx = K[1][0], syy = K[1][1], syz = K[1][2];
  const double szx = K[2][0], szy = K[2][1], szz = K[2][2];
  double a[4][4] = {{sxx + syy + szz, syz - szy, szx - sxz, sxy - syx},
                    {syz - szy, sxx - syy - szz, sxy + syx, szx + sxz},
                    {szx - sxz, sxy + syx, -sxx + syy - szz, syz + szy},
                    {sxy - syx, szx + sxz, syz + szy, -sxx - syy + szz}};
  double v[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
#pragma unroll 1
  for (int sweep = 0; sweep < 32; ++sweep) {
    const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[0][3]) + fabs(a[1][2]) + fabs(a[1][3]) + fabs(a[2][3]);
    const double diag = fabs(a[0][0]) + fabs(a[1][1]) + fabs(a[2][2]) + fabs(a[3][3]);
    if (!(off > 1e-17 * diag)) break;    // also stops on off == 0 and on NaN input
    jacobi_rotate<0, 1>(a, v); jacobi_rotate<0, 2>(a, v); jacobi_rotate<0, 3>(a, v);
    jacobi_rotate<1, 2>(a, v); jacobi_rotate<1, 3>(a, v); jacobi_rotate<2, 3>(a, v);
  }
  double top = a[0][0], w = v[0][0], x = v[1][0], y = v[2][0], z = v[3][0];
#pragma unroll
  for (int i = 1; i < 4; ++i)            // the first largest eigenvalue; compile-time indices keep a and v in registers
    if (a[i][i] > top) top = a[i][i], w = v[0][i], x = v[1][i], y = v[2][i], z = v[3][i];
  const double n = 1.0 / sqrt(w * w + x * x + y * y + z * z);
  w *= n, x *= n, y *= n, z *= n;
  R[0][0] = w * w + x * x - y * y - z * z; R[0][1] = 2 * (x * y - w * z);         R[0][2] = 2 * (x * z + w * y);
  R[1][0] = 2 * (x * y + w * z);         R[1][1] = w * w - x * x + y * y - z * z; R[1][2] = 2 * (y * z - w * x);
  R[2][0] = 2 * (x * z - w * y);         R[2][1] = 2 * (y * z + w * x);         R[2][2] = w * w - x * x - y * y + z * z;
}

// eval.py:145  vis = sum(kps_gt[:, :14, 2]) > min_visible, for one frame (whole warp).
__device__ __forceinline__ bool frame_vis3d(const hd_eval_frames_args &a, long long f, int lane) {
  const int k14 = a.K < 14 ? a.K : 14;
  const double v = lane < k14 ? (double)a.kps_gt[f * a.kps_gt_ld + lane * 3 + 2] : 0.0;
  return warp_sum(v) > (double)a.min_visible;
}

__device__ __forceinline__ void load3(const float *base, long long ld, long long f, int j, double p[3]) {
  const float *r = base + f * ld + j * 3;
  p[0] = r[0], p[1] = r[1], p[2] = r[2];
}

__device__ __forceinline__ double norm3(double x, double y, double z) { return sqrt(x * x + y * y + z * z); }

__global__ void __launch_bounds__(32 * FRAMES_PER_BLOCK) eval_frames_kernel(const __grid_constant__ hd_eval_frames_args a) {
  const int lane = threadIdx.x & 31;
  const long long f = (long long)blockIdx.x * FRAMES_PER_BLOCK + (threadIdx.x >> 5);
  if (f >= a.N) return;                  // whole warps leave together
  double *row = a.out + f * HD_EVAL_COLS;
  double res[HD_EVAL_COLS];

  // ---- the frame's tube: the last s with seq_start[s] <= f
  int lo = 0, hi = a.n_seq - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.seq_start[mid] <= f) lo = mid; else hi = mid - 1;
  }
  const long long end = a.seq_start[lo + 1];

  // ---- 2-D keypoints (eval_util.py:97-137, compute_opt_cam_with_vis :235-260)
  {
    const bool on = lane < a.K;
    double gx = 0, gy = 0, px = 0, py = 0;
    bool vis = false;
    if (on) {
      const float *g = a.kps_gt + f * a.kps_gt_ld + lane * 3;
      const float *p = a.kps_pred + f * a.kps_pred_ld + lane * 2;
      gx = g[0], gy = g[1];
      vis = g[2] != 0.f;
      // eval.py:131 in float32: ((k + 1) * 0.5) * img_size, one rounding per operation
      px = __fmul_rn(__fmul_rn(__fadd_rn(p[0], 1.f), 0.5f), a.img_size);
      py = __fmul_rn(__fmul_rn(__fadd_rn(p[1], 1.f), 0.5f), a.img_size);
    }
    const int nvis = __popc(__ballot_sync(0xffffffffu, vis));
    if (nvis == 0 || nvis < a.min_visible) {
      res[HD_EVAL_KP] = res[HD_EVAL_KP_PA] = res[HD_EVAL_KP_PCK] = nan_d();
    } else {
      const double n = nvis;
      if (!vis) gx = gy = px = py = 0.0;  // the reference zeroes the hidden points (eval_util.py:242-245)
      res[HD_EVAL_KP] = warp_sum(vis ? norm3(gx - px, gy - py, 0.0) : 0.0) / n;
      const double m1x = warp_sum(px) / n, m1y = warp_sum(py) / n;
      const double m2x = warp_sum(gx) / n, m2y = warp_sum(gy) / n;
      const double x0 = vis ? px - m1x : 0.0, x1 = vis ? py - m1y : 0.0, y0 = vis ? gx - m2x : 0.0, y1 = vis ? gy - m2y : 0.0;
      const double a00 = warp_sum(x0 * x0) + 1e-6, a01 = warp_sum(x0 * x1), a11 = warp_sum(x1 * x1) + 1e-6;
      const double b00 = warp_sum(x0 * y0), b01 = warp_sum(x0 * y1), b10 = warp_sum(x1 * y0), b11 = warp_sum(x1 * y1);
      const double det = a00 * a11 - a01 * a01;
      const double i00 = a11 / det, i01 = -a01 / det, i11 = a00 / det;
      const double scale = (i00 * b00 + i01 * b10 + i01 * b01 + i11 * b11) / 2.0;
      const double tx = m2x / scale - m1x, ty = m2y / scale - m1y;
      const double d = norm3(gx - scale * (px + tx), gy - scale * (py + ty), 0.0);
      const double alpha = 0.05 * (double)a.img_size;
      res[HD_EVAL_KP_PA] = warp_sum(vis ? d : 0.0) / n;
      res[HD_EVAL_KP_PCK] = (double)__popc(__ballot_sync(0xffffffffu, vis && d < alpha)) / n;
    }
  }

  // ---- acceleration of the prediction (eval_util.py:14-27), inside the tube
  const bool on = lane < a.J;
  const bool triple = f + 2 < end;
  double p0[3] = {0, 0, 0};
  if (on) load3(a.joints_pred, a.joints_pred_ld, f, lane, p0);
  double p1[3] = {0, 0, 0}, p2[3] = {0, 0, 0};
  if (triple && on) {
    load3(a.joints_pred, a.joints_pred_ld, f + 1, lane, p1);
    load3(a.joints_pred, a.joints_pred_ld, f + 2, lane, p2);
  }
  if (triple) {
    double acc = 0;
    if (on) acc = norm3((p2[0] - p1[0]) - (p1[0] - p0[0]), (p2[1] - p1[1]) - (p1[1] - p0[1]), (p2[2] - p1[2]) - (p1[2] - p0[2]));
    res[HD_EVAL_ACCEL] = warp_sum(acc) / a.J;
  } else {
    res[HD_EVAL_ACCEL] = nan_d();
  }

  // ---- 3-D joints (eval_util.py:30-94, :156-233)
  if (a.joints_gt == nullptr) {
    res[HD_EVAL_JOINTS] = res[HD_EVAL_JOINTS_PA] = res[HD_EVAL_ACCEL_ERROR] = nan_d();
    res[HD_EVAL_VIS3D] = 0.0;
  } else {
    const bool v0 = frame_vis3d(a, f, lane);
    res[HD_EVAL_VIS3D] = v0 ? 1.0 : 0.0;
    double g0[3] = {0, 0, 0};
    if (on) load3(a.joints_gt, a.joints_gt_ld, f, lane, g0);

    // acceleration error: every frame of the triple VIS3D (eval_util.py:85-94)
    if (triple && v0 && frame_vis3d(a, f + 1, lane) && frame_vis3d(a, f + 2, lane)) {
      double e = 0;
      if (on) {
        double g1[3], g2[3], dd[3];
        load3(a.joints_gt, a.joints_gt_ld, f + 1, lane, g1);
        load3(a.joints_gt, a.joints_gt_ld, f + 2, lane, g2);
#pragma unroll
        for (int c = 0; c < 3; ++c) dd[c] = (p0[c] - 2 * p1[c] + p2[c]) - (g0[c] - 2 * g1[c] + g2[c]);
        e = norm3(dd[0], dd[1], dd[2]);
      }
      res[HD_EVAL_ACCEL_ERROR] = warp_sum(e) / a.J;
    } else {
      res[HD_EVAL_ACCEL_ERROR] = nan_d();
    }

    // pelvis alignment (LSP hips 2 and 3), then MPJPE
    double gp[3], pp[3], g[3], p[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      gp[c] = (__shfl_sync(0xffffffffu, g0[c], 3) + __shfl_sync(0xffffffffu, g0[c], 2)) / 2.0;
      pp[c] = (__shfl_sync(0xffffffffu, p0[c], 3) + __shfl_sync(0xffffffffu, p0[c], 2)) / 2.0;
      g[c] = g0[c] - gp[c];
      p[c] = p0[c] - pp[c];
    }
    const double wj = on ? 1.0 : 0.0;
    const double J = a.J;
    res[HD_EVAL_JOINTS] = warp_sum(wj * norm3(g[0] - p[0], g[1] - p[1], g[2] - p[2])) / J;

    // similarity transform of the prediction onto the ground truth
    double mu1[3], mu2[3], x[3], y[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      mu1[c] = warp_sum(wj * p[c]) / J;
      mu2[c] = warp_sum(wj * g[c]) / J;
      x[c] = wj * (p[c] - mu1[c]);
      y[c] = wj * (g[c] - mu2[c]);
    }
    const double var1 = warp_sum(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    double K[3][3], R[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) K[r][c] = warp_sum(x[r] * y[c]);
    best_rotation(K, R);
    double tr = 0;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) tr += R[r][c] * K[c][r];
    const double scale = tr / var1;
    double e = 0;
    if (on) {
      double d[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const double rp = R[r][0] * p[0] + R[r][1] * p[1] + R[r][2] * p[2];
        const double rm = R[r][0] * mu1[0] + R[r][1] * mu1[1] + R[r][2] * mu1[2];
        d[r] = g[r] - (scale * rp + (mu2[r] - scale * rm));
      }
      e = norm3(d[0], d[1], d[2]);
    }
    res[HD_EVAL_JOINTS_PA] = warp_sum(e) / J;
  }

  if (lane < HD_EVAL_COLS) {
    double v = res[0];
#pragma unroll
    for (int c = 1; c < HD_EVAL_COLS; ++c)
      if (lane == c) v = res[c];
    row[lane] = v;
  }
}

__global__ void __launch_bounds__(MESH_THREADS) verts_error_kernel(const float *__restrict__ a, long long a_ld, const float *__restrict__ b,
                                                                  long long b_ld, int V, double *__restrict__ out) {
  __shared__ double sh[MESH_THREADS];
  const long long f = blockIdx.x;
  const float *ra = a + f * a_ld, *rb = b + f * b_ld;
  double s = 0;
  for (int v = threadIdx.x; v < V; v += MESH_THREADS)
    s += norm3((double)ra[v * 3] - rb[v * 3], (double)ra[v * 3 + 1] - rb[v * 3 + 1], (double)ra[v * 3 + 2] - rb[v * 3 + 2]);
  s = block_sum(s, sh);
  if (threadIdx.x == 0) out[f] = s / V;
}

__global__ void __launch_bounds__(MESH_THREADS) mesh_tpose_kernel(const float *__restrict__ dirs, const float *__restrict__ lbs_w, int nnz,
                                                                 int V, const float *__restrict__ beta_gt, int gt_ld,
                                                                 const float *__restrict__ beta_pred, int pred_ld, double *__restrict__ out) {
  __shared__ double sh[MESH_THREADS];
  const long long f = blockIdx.x;
  double db[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) db[i] = (double)beta_gt[f * gt_ld + i] - (double)beta_pred[f * pred_ld + i];
  const long long V3 = 3LL * V;
  double s = 0;
  for (int v = threadIdx.x; v < V; v += MESH_THREADS) {
    double wsum = 0;
    for (int i = 0; i < nnz; ++i) wsum += lbs_w[(long long)v * nnz + i];
    double d[3] = {0, 0, 0};
#pragma unroll
    for (int i = 0; i < 10; ++i)
#pragma unroll
      for (int c = 0; c < 3; ++c) d[c] += (double)dirs[i * V3 + v * 3 + c] * db[i];
    s += fabs(wsum) * norm3(d[0], d[1], d[2]);
  }
  s = block_sum(s, sh);
  if (threadIdx.x == 0) out[f] = s / V;
}

}  // namespace

extern "C" {

int hd_eval_frames(const hd_eval_frames_args *a, void *stream) {
  HD_REQUIRE(a, "hd_eval_frames: null arguments");
  HD_REQUIRE(a->seq_start && a->kps_gt && a->kps_pred && a->joints_pred && a->out, "hd_eval_frames: null pointer");
  HD_REQUIRE(a->N >= 0 && a->n_seq >= 1, "hd_eval_frames: N < 0 or n_seq < 1");
  HD_REQUIRE(a->K >= 1 && a->K <= 32 && a->J >= 4 && a->J <= 32, "hd_eval_frames: K outside [1, 32] or J outside [4, 32]");
  HD_REQUIRE(a->kps_gt_ld >= 3LL * a->K && a->kps_pred_ld >= 2LL * a->K && a->joints_pred_ld >= 3LL * a->J &&
                 (!a->joints_gt || a->joints_gt_ld >= 3LL * a->J),
             "hd_eval_frames: a row stride is shorter than its row");
  HD_REQUIRE(a->img_size > 0.f && a->min_visible >= 0, "hd_eval_frames: img_size <= 0 or min_visible < 0");
  if (a->N == 0) return HD_OK;
  eval_frames_kernel<<<hd::ceil_div(a->N, FRAMES_PER_BLOCK), 32 * FRAMES_PER_BLOCK, 0, (cudaStream_t)stream>>>(*a);
  return hd::check_launch("eval_frames_kernel");
}

int hd_eval_mesh_tpose(const hd_smpl_consts *c, const float *beta_gt, int beta_gt_ld, const float *beta_pred, int beta_pred_ld, int N,
                       double *out, void *stream) {
  HD_REQUIRE(c && beta_gt && beta_pred && out && c->dirs && c->lbs_w, "hd_eval_mesh_tpose: null pointer");
  HD_REQUIRE(N >= 0 && beta_gt_ld >= 10 && beta_pred_ld >= 10, "hd_eval_mesh_tpose: N < 0 or a beta stride < 10");
  HD_REQUIRE(c->num_verts > 0 && c->lbs_nnz >= 1 && c->lbs_nnz <= 24, "hd_eval_mesh_tpose: bad consts");
  if (N == 0) return HD_OK;
  mesh_tpose_kernel<<<N, MESH_THREADS, 0, (cudaStream_t)stream>>>(c->dirs, c->lbs_w, c->lbs_nnz, c->num_verts, beta_gt, beta_gt_ld,
                                                                   beta_pred, beta_pred_ld, out);
  return hd::check_launch("mesh_tpose_kernel");
}

int hd_eval_verts_error(const float *a, long long a_ld, const float *b, long long b_ld, int N, int V, double *out, void *stream) {
  HD_REQUIRE(a && b && out, "hd_eval_verts_error: null pointer");
  HD_REQUIRE(N >= 0 && V > 0 && a_ld >= 3LL * V && b_ld >= 3LL * V, "hd_eval_verts_error: N < 0, V <= 0 or a stride < 3V");
  if (N == 0) return HD_OK;
  verts_error_kernel<<<N, MESH_THREADS, 0, (cudaStream_t)stream>>>(a, a_ld, b, b_ld, V, out);
  return hd::check_launch("verts_error_kernel");
}

}  // extern "C"
