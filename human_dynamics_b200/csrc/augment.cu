// Training-time tube augmentation: TubePreprocessor.preprocess_image (src/util/tube_augmentation.py:114-186) for F frames in two
// launches.  tube_geom_kernel does a frame's bookkeeping (geometry row + labels, pose, gt3d, centre), tube_crop_kernel builds every
// output pixel straight from the source frame: the scaled, edge-padded, rotated and mirrored intermediates never exist.
//
// Built with -fmad=false (Makefile): every float expression below is evaluated in the reference's op order with one rounding per op,
// like TF's CPU kernels and the float32 numpy restatement in oracle/tube_ref.py.  cos / sin / 2^x are taken in double and rounded
// once (TF's float32 Eigen versions are not correctly rounded either; see oracle/tube_ref.py).
#include <cuda_fp16.h>
#include <cstdint>
#include "conv_common.cuh"
#include "smpl_common.cuh"

namespace {

constexpr int kKnownFlags = HD_AUG_SRC_U8 | HD_AUG_ROTATE | HD_AUG_FLIP;

// flip_image (data_utils.py:601-636): the 25 keypoints' L/R swap from the reference's two name lists, reflect_pose's joint swap
// (its 72-entry swap_inds is this table expanded to 3 axes; signs (1, -1, -1) per joint) and reflect_joints3d's LSP swap.
__constant__ int kKpSwap[25] = {5, 4, 3, 2, 1, 0, 11, 10, 9, 8, 7, 6, 12, 13, 14, 16, 15, 18, 17, 20, 19, 22, 21, 24, 23};
__constant__ int kPoseJointSwap[24] = {0, 2, 1, 3, 5, 4, 6, 8, 7, 9, 11, 10, 12, 14, 13, 15, 17, 16, 19, 18, 21, 20, 23, 22};
__constant__ int kJ3dSwap[14] = {5, 4, 3, 2, 1, 0, 11, 10, 9, 8, 7, 6, 12, 13};

struct FrameGeom {           // one row of the geometry table, as hd_b200.h lays it out
  int Hs, Ws, cx, cy, x0, y0, flip, unused;
  float a[6];                // contrib.image.rotate's projective transform (a0 a1 a2; a3 a4 a5)
  float sy, sx;              // resize_bilinear's steps H / Hs, W / Ws
};
static_assert(sizeof(FrameGeom) == 64, "geometry row is 16 words");

__global__ void tube_geom_kernel(hd_tube_aug_args a) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= a.F) return;
  const int S = a.S, K = a.K;
  const bool rotate = (a.flags & HD_AUG_ROTATE) != 0;
  const bool flip = (a.flags & HD_AUG_FLIP) && a.flip[f] != 0;

  // jitter_center, jitter_scale (data_utils.py:512-548)
  const int jx = a.centers[2 * f] + a.trans[2 * f], jy = a.centers[2 * f + 1] + a.trans[2 * f + 1];
  const float sf = (float)exp2((double)a.scale[f]);
  const int Hs = max((int)((float)a.H * sf), 1), Ws = max((int)((float)a.W * sf), 1);   // reference: Hs = 0 fails in resize
  const float fy = (float)Hs / (float)a.H, fx = (float)Ws / (float)a.W;
  const int cx = (int)((float)jx * fx), cy = (int)((float)jy * fy);
  // pad_image_edge by ms, slice S x S at start = centre + ms - S/2 (tube_augmentation.py:138-153)
  const int half = S / 2, ms = half + a.trans_max + 50;
  const int sx0 = cx + ms - half, sy0 = cy + ms - half;

  float c = 1.f, s = 0.f;
  FrameGeom g;
  g.Hs = Hs; g.Ws = Ws; g.cx = cx; g.cy = cy; g.x0 = sx0 - ms; g.y0 = sy0 - ms; g.flip = flip ? 1 : 0; g.unused = 0;
  g.a[0] = 1.f; g.a[1] = 0.f; g.a[2] = 0.f; g.a[3] = 0.f; g.a[4] = 1.f; g.a[5] = 0.f;
  if (rotate) {              // angles_to_projective_transforms (tf.contrib.image, TF 1.x)
    const double th = (double)a.rot[f];
    c = (float)cos(th);
    s = (float)sin(th);
    const float w1 = (float)S - 1.f, h1 = (float)S - 1.f;
    g.a[0] = c; g.a[1] = -s; g.a[2] = (w1 - (c * w1 - s * h1)) / 2.0f;
    g.a[3] = s; g.a[4] = c;  g.a[5] = (h1 - (s * w1 + c * h1)) / 2.0f;
  }
  g.sy = (float)a.H / (float)Hs;
  g.sx = (float)a.W / (float)Ws;
  int4 *grow = reinterpret_cast<int4 *>(a.geom) + (size_t)f * 4;
  const int4 *gsrc = reinterpret_cast<const int4 *>(&g);
#pragma unroll
  for (int q = 0; q < 4; ++q) grow[q] = gsrc[q];
  a.centers_out[2 * f] = cx;
  a.centers_out[2 * f + 1] = cy;

  // keypoints: output j is input kKpSwap[j] under flip (gather after the per-keypoint transform)
  const float *lab = a.labels + (size_t)f * 3 * K;
  float *lo = a.labels_out + (size_t)f * 3 * K;
  const float cen = (float)S * 0.5f, Sf = (float)S;
  for (int j = 0; j < K; ++j) {
    const int k = flip ? kKpSwap[j] : j;
    float x = lab[k] * fx, y = lab[K + k] * fy;
    const float vis = lab[2 * K + k];
    x = (x + (float)ms) - (float)sx0;
    y = (y + (float)ms) - (float)sy0;
    if (rotate) {            // rotate_img (data_utils.py:737-746): kp0^T R[:2,:2] about (S/2, S/2)
      const float x0 = x - cen, y0 = y - cen;
      x = (x0 * c + y0 * s) + cen;
      y = (x0 * (-s) + y0 * c) + cen;
    }
    if (flip) x = (Sf - x) - 1.f;
    const float v = vis > 0.f ? 1.f : 0.f;
    lo[j] = (2.0f * (x / Sf) - 1.0f) * v;
    lo[K + j] = (2.0f * (y / Sf) - 1.0f) * v;
    lo[2 * K + j] = v * v;
  }

  // gt3d: rotate about the scalar mean of all 42 entries (data_utils.py:748-751), then reflect_joints3d (:687-699)
  float gj[42];
  const float *g3 = a.gt3ds + (size_t)f * 42;
  for (int i = 0; i < 42; ++i) gj[i] = g3[i];
  if (rotate) {
    float sum = 0.f;
    for (int i = 0; i < 42; ++i) sum += gj[i];
    const float mean = sum / 42.f;
    for (int j = 0; j < 14; ++j) {
      const float p = gj[3 * j] - mean, q = gj[3 * j + 1] - mean, r = gj[3 * j + 2] - mean;
      gj[3 * j] = ((p * c + q * s) + r * 0.f) + mean;
      gj[3 * j + 1] = ((p * (-s) + q * c) + r * 0.f) + mean;
      gj[3 * j + 2] = ((p * 0.f + q * 0.f) + r * 1.f) + mean;
    }
  }
  float *go = a.gt3ds_out + (size_t)f * 42;
  if (flip) {
    float ref[42], m[3] = {0.f, 0.f, 0.f};
    for (int j = 0; j < 14; ++j) {
      const int k = kJ3dSwap[j];
      ref[3 * j] = ((-1.f * gj[3 * k]) + 0.f * gj[3 * k + 1]) + 0.f * gj[3 * k + 2];
      ref[3 * j + 1] = gj[3 * k + 1];
      ref[3 * j + 2] = gj[3 * k + 2];
    }
    for (int j = 0; j < 14; ++j)
      for (int d = 0; d < 3; ++d) m[d] += ref[3 * j + d];
    for (int d = 0; d < 3; ++d) m[d] = m[d] / 14.f;
    for (int i = 0; i < 42; ++i) go[i] = ref[i] - m[i % 3];
  } else {
    for (int i = 0; i < 42; ++i) go[i] = gj[i];
  }

  // pose: pose[:3] <- rot2aa(R^T rodrigues(pose[:3])) (data_utils.py:752-758), then reflect_pose (:639-684)
  const float *pz = a.poses + (size_t)f * 72;
  float aa[3] = {pz[0], pz[1], pz[2]};
  if (rotate) {
    float R0[9], Rn[9];
    hd_smpl::rodrigues(pz[0], pz[1], pz[2], R0);
    const float Rt[9] = {c, s, 0.f, -s, c, 0.f, 0.f, 0.f, 1.f};
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Rn[i * 3 + j] = (Rt[i * 3] * R0[j] + Rt[i * 3 + 1] * R0[3 + j]) + Rt[i * 3 + 2] * R0[6 + j];
    hd_smpl::rot2aa(Rn, aa);
  }
  float *po = a.poses_out + (size_t)f * 72;
  for (int i = 0; i < 72; ++i) {
    const int src = flip ? kPoseJointSwap[i / 3] * 3 + i % 3 : i;
    const float v = src < 3 ? aa[src] : pz[src];
    po[i] = flip ? v * (i % 3 == 0 ? 1.f : -1.f) : v;
  }
}

template <bool U8>
__device__ __forceinline__ float3 load_px(const void *frame, int W, int y, int x) {
  const size_t o = ((size_t)y * W + x) * 3;
  if (U8) {
    const uint8_t *p = static_cast<const uint8_t *>(frame) + o;
    return make_float3((float)__ldg(p) / 255.f, (float)__ldg(p + 1) / 255.f, (float)__ldg(p + 2) / 255.f);
  }
  const float *p = static_cast<const float *>(frame) + o;
  return make_float3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
}

__device__ __forceinline__ float lerp_tf(float a, float b, float t) { return a + (b - a) * t; }

// Pixel (ry, rx) of tf.image.resize_images(frame, [Hs, Ws]) (TF 1.x resize_bilinear, align_corners=False): in = out * (in/out),
// lower = (int)in, upper = min(lower + 1, in - 1), top then bottom then vertical lerp.
template <bool U8>
__device__ __forceinline__ float3 scaled_px(const void *frame, int H, int W, const FrameGeom &g, int ry, int rx) {
  const float iy = (float)ry * g.sy, ix = (float)rx * g.sx;
  const int ylo = (int)iy, xlo = (int)ix;
  const int yhi = min(ylo + 1, H - 1), xhi = min(xlo + 1, W - 1);
  const float yl = iy - (float)ylo, xl = ix - (float)xlo;
  const float3 tl = load_px<U8>(frame, W, ylo, xlo), tr = load_px<U8>(frame, W, ylo, xhi);
  const float3 bl = load_px<U8>(frame, W, yhi, xlo), br = load_px<U8>(frame, W, yhi, xhi);
  float3 t, b, v;
  t.x = lerp_tf(tl.x, tr.x, xl); t.y = lerp_tf(tl.y, tr.y, xl); t.z = lerp_tf(tl.z, tr.z, xl);
  b.x = lerp_tf(bl.x, br.x, xl); b.y = lerp_tf(bl.y, br.y, xl); b.z = lerp_tf(bl.z, br.z, xl);
  v.x = lerp_tf(t.x, b.x, yl); v.y = lerp_tf(t.y, b.y, yl); v.z = lerp_tf(t.z, b.z, yl);
  return v;
}

// Pixel (py, px) of the S x S slice of the edge-padded scaled image: padding by edge replication = clamping into the scaled image.
template <bool U8>
__device__ __forceinline__ float3 crop_px(const void *frame, int H, int W, const FrameGeom &g, int py, int px) {
  return scaled_px<U8>(frame, H, W, g, min(max(g.y0 + py, 0), g.Hs - 1), min(max(g.x0 + px, 0), g.Ws - 1));
}

// contrib.image.rotate's BILINEAR read: 0 outside the S x S crop.
template <bool U8>
__device__ __forceinline__ float3 crop_px_fill(const void *frame, int H, int W, const FrameGeom &g, int S, long long py, long long px) {
  if (py < 0 || py >= S || px < 0 || px >= S) return make_float3(0.f, 0.f, 0.f);
  return crop_px<U8>(frame, H, W, g, (int)py, (int)px);
}

template <bool U8, bool ROT>
__global__ void __launch_bounds__(256) tube_crop_kernel(const void *__restrict__ frames, int F, int H, int W, const int4 *__restrict__ geom,
                                                        int S, float *__restrict__ out, uint2 *__restrict__ plane_hi,
                                                        uint2 *__restrict__ plane_lo, int WP) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * S * S) return;
  const int x = (int)(i % S);
  const int y = (int)((i / S) % S);
  const int f = (int)(i / ((long long)S * S));
  FrameGeom g;
  int4 *gd = reinterpret_cast<int4 *>(&g);
#pragma unroll
  for (int q = 0; q < 4; ++q) gd[q] = __ldg(geom + (size_t)f * 4 + q);
  const void *frame = U8 ? (const void *)(static_cast<const uint8_t *>(frames) + (size_t)f * H * W * 3)
                         : (const void *)(static_cast<const float *>(frames) + (size_t)f * H * W * 3);
  const int ox = g.flip ? S - 1 - x : x;          // flip_image mirrors the (rotated) crop's width last
  float3 v;
  if (!ROT) {
    v = crop_px<U8>(frame, H, W, g, y, ox);
  } else {                                        // ImageProjectiveTransform, BILINEAR (projection = 1 for a rotation)
    const float fx = (float)ox, fy = (float)y;
    const float in_x = (g.a[0] * fx + g.a[1] * fy) + g.a[2];
    const float in_y = (g.a[3] * fx + g.a[4] * fy) + g.a[5];
    const float xf = floorf(in_x), yf = floorf(in_y), xc = xf + 1.f, yc = yf + 1.f;
    const long long ixf = (long long)xf, iyf = (long long)yf, ixc = (long long)xc, iyc = (long long)yc;
    const float3 p00 = crop_px_fill<U8>(frame, H, W, g, S, iyf, ixf), p01 = crop_px_fill<U8>(frame, H, W, g, S, iyf, ixc);
    const float3 p10 = crop_px_fill<U8>(frame, H, W, g, S, iyc, ixf), p11 = crop_px_fill<U8>(frame, H, W, g, S, iyc, ixc);
    const float wx0 = xc - in_x, wx1 = in_x - xf, wy0 = yc - in_y, wy1 = in_y - yf;
    float3 top, bot;
    top.x = wx0 * p00.x + wx1 * p01.x; top.y = wx0 * p00.y + wx1 * p01.y; top.z = wx0 * p00.z + wx1 * p01.z;
    bot.x = wx0 * p10.x + wx1 * p11.x; bot.y = wx0 * p10.y + wx1 * p11.y; bot.z = wx0 * p10.z + wx1 * p11.z;
    v.x = wy0 * top.x + wy1 * bot.x; v.y = wy0 * top.y + wy1 * bot.y; v.z = wy0 * top.z + wy1 * bot.z;
  }
  const float r = (v.x - 0.5f) * 2.0f, gg = (v.y - 0.5f) * 2.0f, b = (v.z - 0.5f) * 2.0f;     // rescale_image
  if (out) {
    float *o = out + (size_t)i * 3;
    o[0] = r; o[1] = gg; o[2] = b;
  }
  if (plane_hi) {                                 // hd_pack_conv1_planes' layout and split
    uint32_t h0, l0, h1, l1;
    hd::split_f16x2(r, gg, h0, l0);
    hd::split_f16x2(b, 0.f, h1, l1);
    const size_t po = ((size_t)f * (S + 6) + y + 3) * WP + x + 3;
    plane_hi[po] = make_uint2(h0, h1);
    plane_lo[po] = make_uint2(l0, l1);
  }
}

template <bool U8, bool ROT>
int launch_crop(const hd_tube_aug_args *a, cudaStream_t st) {
  const long long total = (long long)a->F * a->S * a->S;
  tube_crop_kernel<U8, ROT><<<hd::ceil_div(total, 256), 256, 0, st>>>(a->frames, a->F, a->H, a->W, reinterpret_cast<const int4 *>(a->geom),
                                                                      a->S, a->crops, reinterpret_cast<uint2 *>(a->plane_hi),
                                                                      reinterpret_cast<uint2 *>(a->plane_lo), a->WP);
  return hd::check_launch("tube_crop_kernel");
}

}  // namespace

extern "C" int hd_tube_augment(const hd_tube_aug_args *a, void *stream) {
  HD_REQUIRE(a, "hd_tube_augment: null argument block");
  HD_REQUIRE(a->frames && a->trans && a->scale && a->labels && a->centers && a->poses && a->gt3ds && a->geom && a->labels_out &&
                 a->centers_out && a->poses_out && a->gt3ds_out,
             "hd_tube_augment: null pointer");
  HD_REQUIRE(!(a->flags & HD_AUG_ROTATE) || a->rot, "hd_tube_augment: HD_AUG_ROTATE needs rot");
  HD_REQUIRE(!(a->flags & HD_AUG_FLIP) || a->flip, "hd_tube_augment: HD_AUG_FLIP needs flip");
  HD_REQUIRE(a->crops || a->plane_hi, "hd_tube_augment: no output (crops or planes)");
  HD_REQUIRE((a->plane_hi == nullptr) == (a->plane_lo == nullptr), "hd_tube_augment: plane_hi and plane_lo go together");
  HD_REQUIRE(a->F > 0 && a->H > 0 && a->W > 0 && a->K > 0 && a->S > 0 && a->trans_max >= 0, "hd_tube_augment: bad sizes");
  HD_REQUIRE(a->S % 2 == 0, "hd_tube_augment: S must be even");
  HD_REQUIRE((a->flags & ~kKnownFlags) == 0, "hd_tube_augment: unknown flag");
  HD_REQUIRE(!(a->flags & HD_AUG_FLIP) || a->K == 25, "hd_tube_augment: flipping needs the 25 keypoints flip_image swaps");
  HD_REQUIRE(((uintptr_t)a->geom & 15u) == 0, "hd_tube_augment: geom must be 16-byte aligned");
  HD_REQUIRE(!a->plane_hi || (a->WP >= a->S + 8 && a->WP % 2 == 0 && hd::aligned16(a->plane_hi) && hd::aligned16(a->plane_lo)),
             "hd_tube_augment: bad plane layout");
  const cudaStream_t st = (cudaStream_t)stream;
  tube_geom_kernel<<<hd::ceil_div(a->F, 128), 128, 0, st>>>(*a);
  int rc = hd::check_launch("tube_geom_kernel");
  if (rc) return rc;
  const bool u8 = (a->flags & HD_AUG_SRC_U8) != 0, rot = (a->flags & HD_AUG_ROTATE) != 0;
  if (u8) return rot ? launch_crop<true, true>(a, st) : launch_crop<true, false>(a, st);
  return rot ? launch_crop<false, true>(a, st) : launch_crop<false, false>(a, st);
}
