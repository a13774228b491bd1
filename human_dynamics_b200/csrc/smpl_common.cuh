// Device pieces of the SMPL pose chain shared by the forward (smpl.cu) and backward (smpl_grad.cu) kernels:
// the kinematic tree, Rodrigues in the reference's op order and the warp-shuffle forward kinematics.
#pragma once
#include "common.cuh"

namespace hd_smpl {

struct Tree {
  int parent[24];
  int depth[24];
  int maxdepth;
};

inline bool build_tree(const int *parents, Tree &t) {
  t.maxdepth = 0;
  for (int i = 0; i < 24; ++i) {
    int p = parents[i];
    if (i == 0) { t.parent[0] = 0; t.depth[0] = 0; continue; }
    if (p < 0 || p >= i) return false;           // batch_lbs.py:172-177 needs parent[i] < i
    t.parent[i] = p;
    t.depth[i] = t.depth[p] + 1;
    if (t.depth[i] > t.maxdepth) t.maxdepth = t.depth[i];
  }
  return true;
}

// batch_lbs.py:42-60 (+ batch_skew :15-39): same operation order as the reference.
__device__ __forceinline__ void rodrigues(float tx, float ty, float tz, float *R) {
  const float eps = 1e-8f;
  const float sx = tx + eps, sy = ty + eps, sz = tz + eps;
  const float angle = sqrtf(sx * sx + sy * sy + sz * sz);
  const float rx = tx / angle, ry = ty / angle, rz = tz / angle;
  const float c = cosf(angle), s = sinf(angle);
  const float oc = 1.0f - c;
  R[0] = c + oc * (rx * rx);
  R[1] = oc * (rx * ry) + s * (-rz);
  R[2] = oc * (rx * rz) + s * ry;
  R[3] = oc * (ry * rx) + s * rz;
  R[4] = c + oc * (ry * ry);
  R[5] = oc * (ry * rz) + s * (-rx);
  R[6] = oc * (rz * rx) + s * (-ry);
  R[7] = oc * (rz * ry) + s * rx;
  R[8] = c + oc * (rz * rz);
}

// batch_rot2aa (src/tf_smpl/batch_lbs.py:63-105): theta = acos(clip((tr R - 1)/2)), axis = (R21-R12, R02-R20, R10-R01) / norm,
// left un-normalised where |theta| < 1e-5 (tf.where in the reference), result theta * axis.
__device__ __forceinline__ void rot2aa(const float *R, float *aa) {
  float c = 0.5f * ((R[0] + R[4] + R[8]) - 1.0f);
  c = fminf(fmaxf(c, -1.0f), 1.0f);
  const float theta = acosf(c);
  const float m21 = R[7] - R[5], m02 = R[2] - R[6], m10 = R[3] - R[1];
  const float denom = sqrtf(m21 * m21 + m02 * m02 + m10 * m10);
  const bool tiny = fabsf(theta) < 0.00001f;
  aa[0] = theta * (tiny ? m21 : m21 / denom);
  aa[1] = theta * (tiny ? m02 : m02 / denom);
  aa[2] = theta * (tiny ? m10 : m10 / denom);
}

// Forward kinematics over the tree, one lane per joint (lanes >= 24 idle but take part in shuffles).
// In: local rotation Rl, rest joint J (per lane).  Out: world rotation Rw, world translation tw.
__device__ __forceinline__ void fk_chain(const Tree &tree, int lane, const float *Rl, const float *J,
                                         float *Rw, float *tw) {
  const bool active = lane < 24;
  const int par = active ? tree.parent[lane] : 0;
  const int dep = active ? tree.depth[lane] : -1;
  float tl[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float jp = __shfl_sync(0xffffffffu, J[c], par);
    tl[c] = (dep == 0) ? J[c] : J[c] - jp;          // batch_lbs.py:170,173
    tw[c] = tl[c];
  }
#pragma unroll
  for (int i = 0; i < 9; ++i) Rw[i] = Rl[i];
  for (int level = 1; level <= tree.maxdepth; ++level) {
    float pR[9], pt[3];
#pragma unroll
    for (int i = 0; i < 9; ++i) pR[i] = __shfl_sync(0xffffffffu, Rw[i], par);
#pragma unroll
    for (int i = 0; i < 3; ++i) pt[i] = __shfl_sync(0xffffffffu, tw[i], par);
    if (dep == level) {                               // results[parent] x A_here, batch_lbs.py:175
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          Rw[r * 3 + c] = pR[r * 3 + 0] * Rl[0 * 3 + c] + pR[r * 3 + 1] * Rl[1 * 3 + c] + pR[r * 3 + 2] * Rl[2 * 3 + c];
        tw[r] = pR[r * 3 + 0] * tl[0] + pR[r * 3 + 1] * tl[1] + pR[r * 3 + 2] * tl[2] + pt[r];
      }
    }
  }
}

}  // namespace hd_smpl
