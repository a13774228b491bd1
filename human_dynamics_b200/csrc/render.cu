// Mesh rendering for sm_90a: the orthographic, single-colour, anti-aliased rasterisation that the reference's visualiser
// asks of the Neural Mesh Renderer (src/util/render/nmr_renderer.py:43-240 with nr.Renderer(look_at, perspective=False)).
// The model it implements is stated as R1-R8 in oracle/render_ref.py; this file is one realisation of it:
//
//   render_mean_kernel    (use_rot only) per-frame vertex mean, fixed-order double sum
//   render_clear_kernel   z-buffer [N, 2S, 2S] of 64-bit keys := empty
//   render_raster_kernel  one thread per (frame, face): transform + projection (R1, R2), eye-facing normal and lit colour
//                         (R5, R6), then a scatter atomicMin of key = (float_bits(depth) << 32) | face over the face's samples
//                         (R3, R4).  Faces whose bounding box exceeds kSmallFace samples are swept by the whole warp instead.
//   render_resolve_kernel one thread per output pixel: mean of its 2x2 samples, alpha = covered fraction, composite (R7, R8)
//
// Depth is positive, so the float bits order like the depths and the smallest key is the nearest sample, ties going to the
// lower face index.  atomicMin is order-independent, so the image does not depend on scheduling, batch size or chunking.
#include <algorithm>
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kSmallFace = 24;                       // bbox samples a single thread sweeps on its own
constexpr unsigned long long kEmpty = ~0ull;

struct RenderArgs {
  const float *verts; long long verts_ld; int V;
  const int *faces; int F;
  const float *cam; int cam_ld;
  int N, S;
  float color[3], light[3], ambient, directional, eye_z, near_z, far_z;
  float rot[9]; int use_rot;
};

// Per-frame vertex mean in double: each thread sums a fixed strided subset, then a fixed tree; result depends on V only.
__global__ void __launch_bounds__(kThreads) render_mean_kernel(const float *__restrict__ verts, long long verts_ld, int V,
                                                               double *__restrict__ mean) {
  __shared__ double red[3][kThreads];
  const int n = blockIdx.x;
  const float *v = verts + (long long)n * verts_ld;
  double s[3] = {0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < V; i += kThreads) {
#pragma unroll
    for (int k = 0; k < 3; ++k) s[k] += (double)v[3 * (long long)i + k];
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) red[k][threadIdx.x] = s[k];
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
#pragma unroll
      for (int k = 0; k < 3; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x < 3) mean[4 * n + threadIdx.x] = red[threadIdx.x][0] / (double)V;
}

__global__ void render_clear_kernel(unsigned long long *__restrict__ zbuf, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) zbuf[i] = kEmpty;
}

// Face record in sample space relative to the bbox origin (c0, r0): barycentric weight i at sample (c0 + dc, r0 + dr) is
// w[i] = wc[i] + wa[i]*dc + wb[i]*dr, inverse depth is zc + za*dc + zb*dr.  Coefficients come from double arithmetic, so the
// per-sample float evaluation only sees small, local magnitudes.
struct FaceRec {
  int c0, r0, wc_n, hc_n;                            // bbox origin and extent in samples (extent 0 = nothing to draw)
  float wa[3], wb[3], wc[3], za, zb, zc;
};

__device__ __forceinline__ void raster_sample(unsigned long long *__restrict__ zb, int S2, const FaceRec &f, int dc, int dr,
                                              unsigned int face, float near_z, float far_z) {
  const float fc = (float)dc, fr = (float)dr;
  const float w0 = fmaf(f.wb[0], fr, fmaf(f.wa[0], fc, f.wc[0]));
  const float w1 = fmaf(f.wb[1], fr, fmaf(f.wa[1], fc, f.wc[1]));
  const float w2 = fmaf(f.wb[2], fr, fmaf(f.wa[2], fc, f.wc[2]));
  if (!(w0 > 0.f && w1 > 0.f && w2 > 0.f)) return;                                    // R3
  const float iz = fmaf(f.zb, fr, fmaf(f.za, fc, f.zc));
  if (!(iz > 0.f)) return;
  const float depth = __frcp_rn(iz);                                                    // R4: 1 / sum(w_i / z_i)
  if (!(depth > near_z && depth < far_z)) return;
  const unsigned long long key = ((unsigned long long)__float_as_uint(depth) << 32) | face;
  unsigned long long *p = zb + (long long)(f.r0 + dr) * S2 + (f.c0 + dc);
  if (key < *p) atomicMin(p, key);                   // a stale read is >= the true value, so no winner is ever skipped
}

__global__ void __launch_bounds__(kThreads) render_raster_kernel(RenderArgs a, const double *__restrict__ mean,
                                                                 unsigned long long *__restrict__ zbuf, float4 *__restrict__ colors) {
  const long long gid = blockIdx.x * (long long)kThreads + threadIdx.x;
  const long long total = (long long)a.N * a.F;
  const int S2 = 2 * a.S;
  FaceRec f;
  f.wc_n = 0; f.hc_n = 0; f.c0 = 0; f.r0 = 0;
  unsigned int face = 0;
  int n = 0;
  if (gid < total) {
    n = (int)(gid / a.F);
    face = (unsigned int)(gid - (long long)n * a.F);
    const int i0 = a.faces[3 * face], i1 = a.faces[3 * face + 1], i2 = a.faces[3 * face + 2];
    float4 col = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i0 >= 0 && i0 < a.V && i1 >= 0 && i1 < a.V && i2 >= 0 && i2 < a.V) {           // out-of-range faces are skipped
      const float *vb = a.verts + (long long)n * a.verts_ld;
      const float *cm = a.cam + (long long)n * a.cam_ld;
      const double s = cm[0], tx = cm[1], ty = cm[2];
      const int idx[3] = {i0, i1, i2};
      double P[3][3];                                // R1 coordinates: x, y (negated), z (before the eye shift)
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        double X = vb[3LL * idx[j]], Y = vb[3LL * idx[j] + 1], Z = vb[3LL * idx[j] + 2];
        if (a.use_rot) {                             // rotated(): R (v - mean) + mean
          const double *m = mean + 4 * n;
          const double dx = X - m[0], dy = Y - m[1], dz = Z - m[2];
          X = a.rot[0] * dx + a.rot[1] * dy + a.rot[2] * dz + m[0];
          Y = a.rot[3] * dx + a.rot[4] * dy + a.rot[5] * dz + m[1];
          Z = a.rot[6] * dx + a.rot[7] * dy + a.rot[8] * dz + m[2];
        }
        P[j][0] = s * (X + tx);
        P[j][1] = -(s * (Y + ty));
        P[j][2] = Z;
      }
      // R5 / R6: normal of the eye-facing winding, pointing to -z; colour = c * (ambient + directional * relu(n . d))
      const double e1x = P[0][0] - P[1][0], e1y = P[0][1] - P[1][1], e1z = P[0][2] - P[1][2];
      const double e2x = P[2][0] - P[1][0], e2y = P[2][1] - P[1][1], e2z = P[2][2] - P[1][2];
      double nx = e1y * e2z - e1z * e2y, ny = e1z * e2x - e1x * e2z, nz = e1x * e2y - e1y * e2x;
      if (nz > 0.0) { nx = -nx; ny = -ny; nz = -nz; }
      const double nl = sqrt(nx * nx + ny * ny + nz * nz);
      const double inv = 1.0 / fmax(nl, 1e-12);
      const double dot = (nx * a.light[0] + ny * a.light[1] + nz * a.light[2]) * inv;
      const float shade = a.ambient + a.directional * (float)fmax(dot, 0.0);
      col = make_float4(a.color[0] * shade, a.color[1] * shade, a.color[2] * shade, 0.f);
      // R2: sample (r, c) of the 2S x 2S grid sits at image x = (2c + 1 - 2S) / 2S, image y = -y = (2r + 1 - 2S) / 2S
      double sc[3], sr[3], iz[3];
      bool finite = true;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        sc[j] = P[j][0] * a.S + (a.S - 0.5);
        sr[j] = -P[j][1] * a.S + (a.S - 0.5);
        iz[j] = 1.0 / (P[j][2] - (double)a.eye_z);
        finite = finite && isfinite(sc[j]) && isfinite(sr[j]) && isfinite(iz[j]);
      }
      const double area = (sc[1] - sc[0]) * (sr[2] - sr[0]) - (sr[1] - sr[0]) * (sc[2] - sc[0]);
      if (finite && area != 0.0) {
        const double lo_c = fmax(ceil(fmin(sc[0], fmin(sc[1], sc[2]))), 0.0);
        const double hi_c = fmin(floor(fmax(sc[0], fmax(sc[1], sc[2]))), (double)(S2 - 1));
        const double lo_r = fmax(ceil(fmin(sr[0], fmin(sr[1], sr[2]))), 0.0);
        const double hi_r = fmin(floor(fmax(sr[0], fmax(sr[1], sr[2]))), (double)(S2 - 1));
        if (lo_c <= hi_c && lo_r <= hi_r) {
          f.c0 = (int)lo_c; f.r0 = (int)lo_r;
          f.wc_n = (int)(hi_c - lo_c) + 1; f.hc_n = (int)(hi_r - lo_r) + 1;
          const double ia = 1.0 / area;
          double zc = 0.0, za = 0.0, zb = 0.0;
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            // weight of vertex j = edge function of the opposite edge (k -> l) / area
            const int k = (j + 1) % 3, l = (j + 2) % 3;
            const double ex = sc[l] - sc[k], ey = sr[l] - sr[k];
            const double A = -ey * ia, B = ex * ia;
            const double Cc = (ex * (lo_r - sr[k]) - ey * (lo_c - sc[k])) * ia;
            f.wa[j] = (float)A; f.wb[j] = (float)B; f.wc[j] = (float)Cc;
            za += A * iz[j]; zb += B * iz[j]; zc += Cc * iz[j];
          }
          f.za = (float)za; f.zb = (float)zb; f.zc = (float)zc;
        }
      }
    }
    colors[gid] = col;
  }
  unsigned long long *zb = zbuf + (long long)n * S2 * S2;
  const int area_s = f.wc_n * f.hc_n;
  const bool big = area_s > kSmallFace;
  if (!big) {
    for (int dr = 0; dr < f.hc_n; ++dr)
      for (int dc = 0; dc < f.wc_n; ++dc) raster_sample(zb, S2, f, dc, dr, face, a.near_z, a.far_z);
  }
  // Large faces: the warp sweeps them one at a time, lanes striding over the bbox samples.
  const int lane = threadIdx.x & 31;
  unsigned int todo = __ballot_sync(0xffffffffu, big);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    FaceRec g;
    g.c0 = __shfl_sync(0xffffffffu, f.c0, src); g.r0 = __shfl_sync(0xffffffffu, f.r0, src);
    g.wc_n = __shfl_sync(0xffffffffu, f.wc_n, src); g.hc_n = __shfl_sync(0xffffffffu, f.hc_n, src);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      g.wa[j] = __shfl_sync(0xffffffffu, f.wa[j], src);
      g.wb[j] = __shfl_sync(0xffffffffu, f.wb[j], src);
      g.wc[j] = __shfl_sync(0xffffffffu, f.wc[j], src);
    }
    g.za = __shfl_sync(0xffffffffu, f.za, src); g.zb = __shfl_sync(0xffffffffu, f.zb, src);
    g.zc = __shfl_sync(0xffffffffu, f.zc, src);
    const unsigned int gface = __shfl_sync(0xffffffffu, face, src);
    const int gn = __shfl_sync(0xffffffffu, n, src);
    unsigned long long *gz = zbuf + (long long)gn * S2 * S2;
    const int cnt = g.wc_n * g.hc_n;
    for (int k = lane; k < cnt; k += 32) {
      const int dr = k / g.wc_n;
      raster_sample(gz, S2, g, k - dr * g.wc_n, dr, gface, a.near_z, a.far_z);
    }
  }
}

__global__ void __launch_bounds__(kThreads) render_resolve_kernel(const unsigned long long *__restrict__ zbuf,
                                                                  const float4 *__restrict__ colors, int N, int S, int F,
                                                                  float bg0, float bg1, float bg2,
                                                                  const float *__restrict__ background,
                                                                  unsigned char *__restrict__ out_rgb, float *__restrict__ out_alpha) {
  const long long pix = blockIdx.x * (long long)kThreads + threadIdx.x;
  const long long total = (long long)N * S * S;
  if (pix >= total) return;
  const int n = (int)(pix / ((long long)S * S));
  const int rem = (int)(pix - (long long)n * S * S);
  const int i = rem / S, j = rem - i * S;
  const int S2 = 2 * S;
  const unsigned long long *zb = zbuf + (long long)n * S2 * S2;
  const ulonglong2 top = *reinterpret_cast<const ulonglong2 *>(zb + (long long)(2 * i) * S2 + 2 * j);
  const ulonglong2 bot = *reinterpret_cast<const ulonglong2 *>(zb + (long long)(2 * i + 1) * S2 + 2 * j);
  const unsigned long long key[4] = {top.x, top.y, bot.x, bot.y};
  float r = 0.f, g = 0.f, b = 0.f;
  int cov = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {                      // R7: mean of the 2x2 samples, background colour where empty
    float cr = bg0, cg = bg1, cb = bg2;
    if (key[q] != kEmpty) {
      const float4 c = colors[(long long)n * F + (unsigned int)(key[q] & 0xffffffffu)];
      cr = c.x; cg = c.y; cb = c.z;
      ++cov;
    }
    r = __fadd_rn(r, cr); g = __fadd_rn(g, cg); b = __fadd_rn(b, cb);
  }
  const float alpha = 0.25f * (float)cov;
  const float rgb[3] = {__fmul_rn(r, 0.25f), __fmul_rn(g, 0.25f), __fmul_rn(b, 0.25f)};
  unsigned char *o = out_rgb + pix * 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) {                      // R8
    const float rend = __fmul_rn(fminf(fmaxf(rgb[k], 0.f), 1.f), 255.f);
    float v = rend;
    if (background) {
      const float img = background[pix * 3 + k];
      const float img255 = __fmul_rn(__fmul_rn(__fadd_rn(img, 1.f), 0.5f), 255.f);
      v = __fadd_rn(__fmul_rn(img255, __fsub_rn(1.f, alpha)), __fmul_rn(rend, alpha));
    }
    o[k] = (unsigned char)(int)fminf(fmaxf(v, 0.f), 255.f);
  }
  if (out_alpha) out_alpha[pix] = alpha;
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace

extern "C" {

size_t hd_render_workspace_bytes(int N, int S, int F) {
  if (N <= 0 || S <= 0 || F <= 0) return 0;
  return align256((size_t)N * 4 * S * S * sizeof(unsigned long long)) + align256((size_t)N * F * sizeof(float4)) +
         align256((size_t)N * 4 * sizeof(double));
}

int hd_render_mesh(const float *verts, long long verts_ld, int N, int V, const int *faces, int F, const float *cam, int cam_ld,
                   const hd_render_params *p, const float *background, int S, unsigned char *out_rgb, float *out_alpha, void *ws,
                   size_t ws_bytes, void *stream) {
  HD_REQUIRE(verts && faces && cam && p && out_rgb && ws, "hd_render_mesh: null pointer");
  HD_REQUIRE(S >= 1 && S <= 2048, "hd_render_mesh: S must lie in [1, 2048]");
  HD_REQUIRE(N >= 0 && V > 0 && F > 0 && verts_ld >= 3LL * V && cam_ld >= 3, "hd_render_mesh: bad N / V / F / leading dimensions");
  if (N == 0) return HD_OK;
  if (ws_bytes < hd_render_workspace_bytes(N, S, F)) {
    hd::set_last_error_text("hd_render_mesh: workspace smaller than hd_render_workspace_bytes(N, S, F)");
    return HD_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const long long nz = (long long)N * 4 * S * S;
  unsigned long long *zbuf = reinterpret_cast<unsigned long long *>(ws);
  float4 *colors = reinterpret_cast<float4 *>(reinterpret_cast<char *>(ws) + align256((size_t)nz * sizeof(unsigned long long)));
  double *mean = reinterpret_cast<double *>(reinterpret_cast<char *>(colors) + align256((size_t)N * F * sizeof(float4)));

  RenderArgs a;
  a.verts = verts; a.verts_ld = verts_ld; a.V = V; a.faces = faces; a.F = F; a.cam = cam; a.cam_ld = cam_ld; a.N = N; a.S = S;
  for (int k = 0; k < 3; ++k) { a.color[k] = p->color[k]; a.light[k] = p->light_dir[k]; }
  a.ambient = p->ambient; a.directional = p->directional;
  a.eye_z = p->eye_z; a.near_z = p->near_z; a.far_z = p->far_z;
  for (int k = 0; k < 9; ++k) a.rot[k] = p->rot[k];
  a.use_rot = p->use_rot != 0;

  int rc;
  if (a.use_rot) {
    render_mean_kernel<<<N, kThreads, 0, st>>>(verts, verts_ld, V, mean);
    if ((rc = hd::check_launch("render_mean_kernel"))) return rc;
  }
  render_clear_kernel<<<(int)std::min<long long>(hd::ceil_div(nz, kThreads), 132LL * 16), kThreads, 0, st>>>(zbuf, nz);
  if ((rc = hd::check_launch("render_clear_kernel"))) return rc;
  render_raster_kernel<<<hd::ceil_div((long long)N * F, kThreads), kThreads, 0, st>>>(a, mean, zbuf, colors);
  if ((rc = hd::check_launch("render_raster_kernel"))) return rc;
  render_resolve_kernel<<<hd::ceil_div((long long)N * S * S, kThreads), kThreads, 0, st>>>(
      zbuf, colors, N, S, F, p->bg[0], p->bg[1], p->bg[2], background, out_rgb, out_alpha);
  return hd::check_launch("render_resolve_kernel");
}

}  // extern "C"
