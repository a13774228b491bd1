// The encoder objective of the reference trainer (src/trainer_sequence_fc.py compute_losses_batched / _deltas / _prior, src/ops.py,
// src/tf_smpl/projection.py) for sm_90a, as a list of term descriptors (include/hd_b200.h, hd_loss_term) evaluated in a fixed number of
// launches whatever the number of terms:
//   forward:  loss_partial_kernel over a fixed partition of (term, block) -> per-block sums and weight counts; loss_reduce_kernel sums
//             each term's blocks in order and divides by the count (tf.losses' SUM_BY_NONZERO_WEIGHTS; a count of 0 gives 0);
//   backward: loss_grad_kernel, one thread per element of every gradient tensor, looping over the terms that read that tensor in term
//             order (a gather: no atomics).  An element's gradient depends only on its own frame, the term counts and the scales.
// The descriptors travel by value as a __grid_constant__ kernel parameter (up to HD_LOSS_MAX_TERMS), so nothing is copied to the device.
#include "conv_common.cuh"

namespace {

constexpr int PART_THREADS = 128;        // items per block of the partial-sum kernel
constexpr int SEG = 32;                  // floats per item of an unaligned MSE row (rows are split so that wide rows spread over threads)
constexpr int GRAD_THREADS = 256;

struct Term {
  hd_loss_term t;
  long long block0;                      // first block of the term in the forward partition
  long long items;                       // B * Tw * segments
  int segs;                              // items per frame
  int gp, gq, gc;                        // gradient target of p / q / cam (-1: none)
  long long op, oq, oc;                  // element offset of p / q / cam inside that target
};

struct Params {
  Term terms[HD_LOSS_MAX_TERMS];
  hd_loss_grad grads[HD_LOSS_MAX_GRADS];
  long long grad0[HD_LOSS_MAX_GRADS + 1];   // prefix of the targets' element counts
  int n, n_grads;
  long long blocks;
};
static_assert(sizeof(Params) < 32000, "kernel parameter limit");

// Workspace: [blocks] long long counts | [blocks] float partial sums | [HD_LOSS_MAX_TERMS] float divisors (the 8-byte counts first, so
// that every part is aligned whatever the block count).
inline size_t ws_bytes_for(long long blocks) {
  return (size_t)blocks * (sizeof(float) + sizeof(long long)) + HD_LOSS_MAX_TERMS * sizeof(float);
}

__device__ __forceinline__ const float *row_ptr(const float *base, long long clip, long long frame, int b, int t) {
  return base + (long long)b * clip + (long long)t * frame;
}

// procrustes2d_vis (projection.py:48-104) on the visible (vis > 0) keypoints of one frame, in double.  Returns false when no keypoint is
// visible: the reference divides 0 / 0 there; here the camera is (0.7, 0, 0) and the frame contributes nothing.
__device__ bool optimal_camera(const float *x, int xd, const float *y, int K, float cam[3]) {
  double n = 0, m1x = 0, m1y = 0, m2x = 0, m2y = 0;
  for (int k = 0; k < K; ++k)
    if (y[k * 3 + 2] > 0.f) {
      n += 1;
      m1x += x[k * xd]; m1y += x[k * xd + 1];
      m2x += y[k * 3]; m2y += y[k * 3 + 1];
    }
  if (n == 0) {
    cam[0] = 0.7f, cam[1] = 0.f, cam[2] = 0.f;
    return false;
  }
  m1x /= n, m1y /= n, m2x /= n, m2y /= n;
  double a00 = 1e-6, a01 = 0, a11 = 1e-6, b00 = 0, b01 = 0, b10 = 0, b11 = 0;
  for (int k = 0; k < K; ++k)
    if (y[k * 3 + 2] > 0.f) {
      const double u = x[k * xd] - m1x, v = x[k * xd + 1] - m1y, p = y[k * 3] - m2x, q = y[k * 3 + 1] - m2y;
      a00 += u * u, a01 += u * v, a11 += v * v;
      b00 += u * p, b01 += u * q, b10 += v * p, b11 += v * q;
    }
  const double det = a00 * a11 - a01 * a01;
  // trace(A^-1 B) / 2 with A^-1 = [[a11, -a01], [-a01, a00]] / det
  double s = (a11 * b00 - a01 * b10 - a01 * b01 + a00 * b11) / det / 2.0;
  s = fmin(fmax(s, 0.7), 10.0);
  cam[0] = (float)s;
  cam[1] = (float)(m2x / s - m1x);
  cam[2] = (float)(m2y / s - m1y);
  return true;
}

// The camera of a KP_L1 term's frame (b, t): the prediction's own, the optimal one, or identity.  False: the frame is skipped.
__device__ bool frame_camera(const hd_loss_term &t, int b, int f, float cam[3]) {
  if (t.proj == HD_LOSS_KP_CAMERA) {
    const float *c = row_ptr(t.cam, t.cam_clip, t.cam_frame, b, t.p_t0 + f);
    cam[0] = c[0], cam[1] = c[1], cam[2] = c[2];
    return true;
  }
  if (t.proj == HD_LOSS_KP_OPTCAM)
    return optimal_camera(row_ptr(t.p, t.p_clip, t.p_frame, b, t.p_t0 + f), t.D, row_ptr(t.q, t.q_clip, t.q_frame, b, t.q_t0 + f), t.K,
                          cam);
  cam[0] = 1.f, cam[1] = 0.f, cam[2] = 0.f;
  return true;
}

__device__ __forceinline__ float xhat(const hd_loss_term &t, const float *x, int k, int c, const float cam[3]) {
  const float v = x[k * t.D + c];
  return t.proj == HD_LOSS_KP_RAW ? v : cam[0] * (v + cam[1 + c]);
}

__device__ __forceinline__ float pelvis(const float *r, int c) { return (r[2 * 3 + c] + r[3 * 3 + c]) * 0.5f; }

// One item: sum of the term's weighted residuals over (a segment of) one frame, and the weight count it adds.
__device__ void item_value(const hd_loss_term &t, int segs, long long item, float &sum, long long &cnt) {
  const long long fr = item / segs;
  const int seg = (int)(item - fr * segs);
  const int b = (int)(fr / t.Tw), f = (int)(fr - (long long)b * t.Tw);
  const float *x = row_ptr(t.p, t.p_clip, t.p_frame, b, t.p_t0 + f);
  const float *y = t.q ? row_ptr(t.q, t.q_clip, t.q_frame, b, t.q_t0 + f) : nullptr;
  sum = 0.f, cnt = 0;
  if (t.kind == HD_LOSS_KP_L1) {
    float cam[3];
    const bool ok = frame_camera(t, b, f, cam);
    if (t.cam_out) {
      float *co = t.cam_out + ((long long)b * t.Tw + f) * 3;
      co[0] = cam[0], co[1] = cam[1], co[2] = cam[2];
    }
    for (int k = 0; k < t.K; ++k) {
      const float v = y[k * 3 + 2];
      if (v != 0.f) {
        cnt += 2;
        if (ok) sum += v * (fabsf(xhat(t, x, k, 0, cam) - y[k * 3]) + fabsf(xhat(t, x, k, 1, cam) - y[k * 3 + 1]));
      }
    }
    return;
  }
  const float w = t.w ? t.w[b] : 1.f;
  if (w == 0.f) return;
  if (t.proj) {      // pelvis-aligned rows of D / 3 joints
    float pp[3], pq[3];
    for (int c = 0; c < 3; ++c) pp[c] = pelvis(x, c), pq[c] = y ? pelvis(y, c) : 0.f;
    for (int i = 0; i < t.D; ++i) {
      const float d = (x[i] - pp[i % 3]) - (y ? y[i] - pq[i % 3] : 0.f);
      sum = fmaf(d, d, sum);
    }
    sum *= w;
    cnt = t.D;
    return;
  }
  const int i0 = seg * SEG, i1 = min(t.D, i0 + SEG);
  for (int i = i0; i < i1; ++i) {
    const float d = x[i] - (y ? y[i] : 0.f);
    sum = fmaf(d, d, sum);
  }
  sum *= w;
  cnt = seg == 0 ? t.D : 0;
}

__global__ void __launch_bounds__(PART_THREADS) loss_partial_kernel(const __grid_constant__ Params P, float *__restrict__ psum,
                                                                    long long *__restrict__ pcnt) {
  __shared__ float ss[PART_THREADS];
  __shared__ long long sc[PART_THREADS];
  int ti = 0;
  while (ti + 1 < P.n && P.terms[ti + 1].block0 <= (long long)blockIdx.x) ++ti;
  const Term &T = P.terms[ti];
  const long long item = ((long long)blockIdx.x - T.block0) * PART_THREADS + threadIdx.x;
  float s = 0.f;
  long long c = 0;
  if (item < T.items) item_value(T.t, T.segs, item, s, c);
  ss[threadIdx.x] = s, sc[threadIdx.x] = c;
  __syncthreads();
  for (int h = PART_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) ss[threadIdx.x] += ss[threadIdx.x + h], sc[threadIdx.x] += sc[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) psum[blockIdx.x] = ss[0], pcnt[blockIdx.x] = sc[0];
}

// Thread i: term i's blocks in order.  values[i] = scale * sum / count (0 when count is 0); div[i] = count.
__global__ void loss_reduce_kernel(const __grid_constant__ Params P, const float *__restrict__ psum, const long long *__restrict__ pcnt,
                                   float *__restrict__ div, float *__restrict__ values) {
  const int i = threadIdx.x;
  if (i >= P.n) return;
  const Term &T = P.terms[i];
  const long long nb = (T.items + PART_THREADS - 1) / PART_THREADS;
  float s = 0.f;
  long long c = 0;
  for (long long k = 0; k < nb; ++k) s += psum[T.block0 + k], c += pcnt[T.block0 + k];
  div[i] = (float)c;
  values[i] = c > 0 ? T.t.scale * (s / (float)c) : 0.f;
}

// Element e_rel of a tensor addressed as base + b * clip + (t0 + f) * frame + i (i < width): true and (b, f, i) when it lies in the
// term's window.
__device__ __forceinline__ bool locate(long long e, long long clip, long long frame, int t0, int B, int Tw, int width, int &b, int &f,
                                       int &i) {
  if (e < 0 || frame <= 0) return false;
  const long long bb = clip > 0 ? e / clip : 0;
  const long long r = e - bb * clip;
  const long long ff = r / frame;
  const long long ii = r - ff * frame;
  if (bb >= B || ff - t0 < 0 || ff - t0 >= Tw || ii >= width) return false;
  b = (int)bb, f = (int)(ff - t0), i = (int)ii;
  return true;
}

__device__ __forceinline__ float sgn(float r) { return r > 0.f ? 1.f : (r < 0.f ? -1.f : 0.f); }

// d term / d element for one side of a term: side 0 = p, 1 = q (MSE only), 2 = cam (KP_CAMERA only).  g0 = scale * upstream / count.
__device__ float term_grad(const hd_loss_term &t, int side, int b, int f, int i, float g0) {
  const float *x = row_ptr(t.p, t.p_clip, t.p_frame, b, t.p_t0 + f);
  const float *y = t.q ? row_ptr(t.q, t.q_clip, t.q_frame, b, t.q_t0 + f) : nullptr;
  if (t.kind == HD_LOSS_KP_L1) {
    if (side == 0 && i % t.D >= 2) return 0.f;     // z of a keypoint: no camera to solve
    float cam[3];
    if (!frame_camera(t, b, f, cam)) return 0.f;
    if (side == 0) {
      const int k = i / t.D, c = i - k * t.D;
      const float v = y[k * 3 + 2];
      const float g = g0 * v * sgn(xhat(t, x, k, c, cam) - y[k * 3 + c]);
      return t.proj == HD_LOSS_KP_RAW ? g : g * cam[0];
    }
    float acc = 0.f;     // cam: ds = sum g (X + t), dt_c = sum s g_c
    for (int k = 0; k < t.K; ++k) {
      const float v = y[k * 3 + 2];
      if (v == 0.f) continue;
      for (int c = 0; c < 2; ++c) {
        const float g = g0 * v * sgn(xhat(t, x, k, c, cam) - y[k * 3 + c]);
        if (i == 0) acc = fmaf(g, x[k * t.D + c] + cam[1 + c], acc);
        else if (i == 1 + c) acc = fmaf(g, cam[0], acc);
      }
    }
    return acc;
  }
  const float w = t.w ? t.w[b] : 1.f;
  if (w == 0.f) return 0.f;
  const float gw = 2.f * g0 * w;
  float out;
  if (t.proj) {
    const int c = i % 3, j = i / 3;
    const float px = pelvis(x, c), py = y ? pelvis(y, c) : 0.f;
    const float gi = gw * ((x[i] - px) - (y ? y[i] - py : 0.f));
    out = gi;
    if (j == 2 || j == 3) {
      float s = 0.f;
      for (int jj = 0; jj < t.D / 3; ++jj) s += gw * ((x[jj * 3 + c] - px) - (y ? y[jj * 3 + c] - py : 0.f));
      out = gi - 0.5f * s;
    }
  } else {
    out = gw * (x[i] - (y ? y[i] : 0.f));
  }
  return side == 1 ? -out : out;
}

__global__ void __launch_bounds__(GRAD_THREADS) loss_grad_kernel(const __grid_constant__ Params P, const float *__restrict__ dvalues,
                                                                 const float *__restrict__ div) {
  const long long e = (long long)blockIdx.x * GRAD_THREADS + threadIdx.x;
  if (e >= P.grad0[P.n_grads]) return;
  int g = 0;
  while (e >= P.grad0[g + 1]) ++g;
  const long long el = e - P.grad0[g];
  float acc = 0.f;
  for (int ti = 0; ti < P.n; ++ti) {
    const Term &T = P.terms[ti];
    if (T.gp != g && T.gq != g && T.gc != g) continue;
    const hd_loss_term &t = T.t;
    const float d = div[ti];
    if (d <= 0.f) continue;
    const float g0 = t.scale * dvalues[ti] / d;
    const int width = t.kind == HD_LOSS_KP_L1 ? t.K * t.D : t.D;
    int b, f, i;
    if (T.gp == g && locate(el - T.op, t.p_clip, t.p_frame, t.p_t0, t.B, t.Tw, width, b, f, i)) acc += term_grad(t, 0, b, f, i, g0);
    if (T.gq == g && locate(el - T.oq, t.q_clip, t.q_frame, t.q_t0, t.B, t.Tw, width, b, f, i)) acc += term_grad(t, 1, b, f, i, g0);
    if (T.gc == g && locate(el - T.oc, t.cam_clip, t.cam_frame, t.p_t0, t.B, t.Tw, 3, b, f, i)) acc += term_grad(t, 2, b, f, i, g0);
  }
  P.grads[g].grad[el] = acc;
}

// Validates the descriptors and fills the kernel parameters (forward partition; gradient targets when grads != NULL).
int build_params(const hd_loss_term *terms, int n, const hd_loss_grad *grads, int n_grads, Params &P, const char *who) {
  HD_REQUIRE(terms && n > 0 && n <= HD_LOSS_MAX_TERMS, "hd_loss: null descriptors or n outside [1, HD_LOSS_MAX_TERMS]");
  HD_REQUIRE(n_grads >= 0 && n_grads <= HD_LOSS_MAX_GRADS && (n_grads == 0 || grads), "hd_loss: bad gradient target list");
  P.n = n, P.n_grads = n_grads;
  long long blocks = 0;
  for (int i = 0; i < n; ++i) {
    const hd_loss_term &t = terms[i];
    Term &T = P.terms[i];
    T.t = t;
    HD_REQUIRE(t.kind == HD_LOSS_KP_L1 || t.kind == HD_LOSS_MSE_ROWS, "hd_loss: term: unknown kind");
    HD_REQUIRE(t.p && t.B > 0 && t.Tw > 0 && t.D > 0, "hd_loss: term: null p, or B / Tw / D <= 0");
    HD_REQUIRE(t.p_t0 >= 0 && t.p_t0 + t.Tw <= t.p_T && t.p_frame >= 0 && t.p_clip >= 0, "hd_loss: term: prediction window overruns T");
    if (t.q)
      HD_REQUIRE(t.q_t0 >= 0 && t.q_t0 + t.Tw <= t.q_T && t.q_frame >= 0 && t.q_clip >= 0, "hd_loss: term: target window overruns T");
    if (t.kind == HD_LOSS_KP_L1) {
      HD_REQUIRE(t.q && t.K > 0 && t.D >= 2, "hd_loss: term: KP_L1 needs labels, K > 0 and D >= 2");
      HD_REQUIRE(t.proj >= HD_LOSS_KP_CAMERA && t.proj <= HD_LOSS_KP_RAW, "hd_loss: term: unknown projection");
      HD_REQUIRE(t.proj != HD_LOSS_KP_CAMERA || (t.cam && t.cam_frame >= 0 && t.cam_clip >= 0), "hd_loss: term: KP_CAMERA needs cam");
      HD_REQUIRE(!t.cam_out || t.proj == HD_LOSS_KP_OPTCAM, "hd_loss: term: cam_out is for KP_OPTCAM terms");
      T.segs = 1;
    } else {
      HD_REQUIRE(!t.proj || (t.D % 3 == 0 && t.D / 3 >= 14), "hd_loss: term: pelvis alignment needs rows of K >= 14 joints x 3");
      T.segs = t.proj ? 1 : (t.D + SEG - 1) / SEG;
    }
    T.items = (long long)t.B * t.Tw * T.segs;
    T.block0 = blocks;
    blocks += (T.items + PART_THREADS - 1) / PART_THREADS;
    T.gp = T.gq = T.gc = -1;
    T.op = T.oq = T.oc = 0;
  }
  P.blocks = blocks;
  P.grad0[0] = 0;
  for (int g = 0; g < n_grads; ++g) {
    HD_REQUIRE(grads[g].src && grads[g].grad && grads[g].numel > 0, "hd_loss: gradient target: null pointer or numel <= 0");
    P.grads[g] = grads[g];
    P.grad0[g + 1] = P.grad0[g] + grads[g].numel;
    auto find = [&](const float *ptr, int &gi, long long &off) {
      if (ptr && gi < 0 && ptr >= grads[g].src && ptr < grads[g].src + grads[g].numel) gi = g, off = ptr - grads[g].src;
    };
    for (int i = 0; i < n; ++i) {
      Term &T = P.terms[i];
      find(T.t.p, T.gp, T.op);
      if (T.t.kind == HD_LOSS_MSE_ROWS) find(T.t.q, T.gq, T.oq);
      if (T.t.kind == HD_LOSS_KP_L1 && T.t.proj == HD_LOSS_KP_CAMERA) find(T.t.cam, T.gc, T.oc);
    }
  }
  for (int i = 0; i < n; ++i) {
    const Term &T = P.terms[i];
    HD_REQUIRE((T.gp < 0 || T.t.p_frame > 0) && (T.gq < 0 || T.t.q_frame > 0) && (T.gc < 0 || T.t.cam_frame > 0),
               "hd_loss: term: a side that receives a gradient needs a frame stride > 0");
  }
  return HD_OK;
}

long long blocks_of(const hd_loss_term *terms, int n) {
  static thread_local Params P;
  if (build_params(terms, n, nullptr, 0, P, "hd_loss_workspace_bytes") != HD_OK) return -1;
  return P.blocks;
}

}  // namespace

extern "C" {

size_t hd_loss_workspace_bytes(const hd_loss_term *terms, int n) {
  const long long blocks = blocks_of(terms, n);
  return blocks < 0 ? 0 : ws_bytes_for(blocks);
}

int hd_loss_forward(const hd_loss_term *terms, int n, float *values, void *ws, size_t ws_bytes, void *stream) {
  static thread_local Params P;
  const int rc = build_params(terms, n, nullptr, 0, P, "hd_loss_forward");
  if (rc != HD_OK) return rc;
  HD_REQUIRE(values && ws && ws_bytes >= ws_bytes_for(P.blocks) && ((uintptr_t)ws & 7) == 0,
             "hd_loss_forward: null values / ws, workspace too small or not 8-byte aligned");
  long long *pcnt = (long long *)ws;
  float *psum = (float *)(pcnt + P.blocks);
  float *div = psum + P.blocks;
  loss_partial_kernel<<<(unsigned)P.blocks, PART_THREADS, 0, (cudaStream_t)stream>>>(P, psum, pcnt);
  int e = hd::check_launch("loss_partial_kernel");
  if (e != HD_OK) return e;
  loss_reduce_kernel<<<1, HD_LOSS_MAX_TERMS, 0, (cudaStream_t)stream>>>(P, psum, pcnt, div, values);
  return hd::check_launch("loss_reduce_kernel");
}

int hd_loss_backward(const hd_loss_term *terms, int n, const hd_loss_grad *grads, int n_grads, const float *dvalues, const void *ws,
                     size_t ws_bytes, void *stream) {
  static thread_local Params P;
  const int rc = build_params(terms, n, grads, n_grads, P, "hd_loss_backward");
  if (rc != HD_OK) return rc;
  HD_REQUIRE(n_grads > 0 && dvalues && ws && ws_bytes >= ws_bytes_for(P.blocks) && ((uintptr_t)ws & 7) == 0,
             "hd_loss_backward: no gradient target, null dvalues / ws, or workspace too small or not 8-byte aligned");
  const float *div = (const float *)((const char *)ws + (size_t)P.blocks * (sizeof(float) + sizeof(long long)));
  const long long total = P.grad0[n_grads];
  loss_grad_kernel<<<(unsigned)((total + GRAD_THREADS - 1) / GRAD_THREADS), GRAD_THREADS, 0, (cudaStream_t)stream>>>(P, dvalues, div);
  return hd::check_launch("loss_grad_kernel");
}

}  // extern "C"
