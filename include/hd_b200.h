/*
 * hd_b200.h -- C-ABI of the HMMR video->SMPL hot path for the H100 (sm_90a) (libhd_b200.so).
 *
 * The reference (akanazawa/human_dynamics) is pure Python/TF1 and has no FFI layer; its
 * boundary for this path is the Python call surface of graph-building functions plus one
 * sess.run (SURVEY.md 8b).  Each entry point below replaces the arithmetic of the cited
 * reference function; the Python shim under src/ (same module paths, names and argument
 * meaning as the reference) binds these with ctypes -- see INTEGRATION.md.
 *
 * Conventions: every pointer is a DEVICE pointer to fp32 (or int32 where typed) unless it
 * says "host"; tensors are row-major, activations NHWC; `stream` is a cudaStream_t passed
 * as void*; all calls are asynchronous on `stream`, never synchronise, never allocate,
 * and return an hd_status (0 = ok).  No torch types cross this boundary.
 */
#ifndef HD_B200_H_
#define HD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  HD_OK = 0,
  HD_ERR_INVALID = 1,      /* bad shape / null pointer / unsupported combination */
  HD_ERR_WORKSPACE = 2,    /* workspace too small */
  HD_ERR_CUDA = 3,         /* a CUDA runtime / driver call failed (see hd_last_error) */
  HD_ERR_UNSUPPORTED = 4   /* device is not sm_90 or requested impl not available */
} hd_status;

int hd_version(void);
const char *hd_status_string(int status);
/* Last CUDA error text recorded by this thread's most recent failing call ("" if none). */
const char *hd_last_error(void);
/* Number of kernels this library has launched since load / since the last reset (host counter). */
long long hd_launch_count(void);
void hd_launch_count_reset(void);

/* ------------------------------------------------------------------------------------------
 * Fused implicit-GEMM convolution / fully-connected layer.
 * Replaces every slim conv2d / fully_connected (+ the BatchNorm/GroupNorm/ReLU/bias/residual
 * ops around it) on the path: src/models.py:65-74 (resnet_v2_50 convs), :102-113 (IEF FCs),
 * :173-184,:209-221 (temporal convs), :283-294 (fc2_res).
 *
 *   a[n,iy,ix,ci] = in[n,iy,ix,ci]                                (zero outside the image)
 *   if pre_scale:  a = a*pre_scale[n*pre_img_stride+ci] + pre_shift[...]; if pre_relu: a=max(a,0)
 *        (prologue acts on real pixels only: padding stays 0, like padding relu(bn(x)) in TF)
 *   acc[n,oy,ox,co] = sum_{ky,kx,ci} a[n, oy*stride-pad_t+ky, ox*stride-pad_l+kx, ci] * W[(ky,kx,ci),co]
 *   v = acc*post_scale[co] + post_shift[co]   (NULL scale = 1, NULL shift = 0)
 *   if res: v += res[(n*res_H + oy*res_stride)*res_W + ox*res_stride][co]
 *   if post_relu: v = max(v,0)
 *   out[(n*Ho+oy)*Wo+ox][co] = v          (out may be NULL when out_hi/out_lo are given, see below)
 * ------------------------------------------------------------------------------------------ */
enum { HD_IMPL_SIMT = 0, HD_IMPL_TC_3XTF32 = 1, HD_IMPL_TC_1XTF32 = 2, HD_IMPL_TC_3XF16 = 3 };

typedef struct {
  const float *in;  long long in_ld;          /* floats between consecutive pixels (>= Cin) */
  int n_img, H, W, Cin;
  int Ho, Wo, KH, KW, stride, pad_t, pad_l;
  const float *w_kn;                          /* [K, Cout] row-major, K=(ky,kx,ci) (TF HWIO flattened) */
  const void *w_nk_hi;                        /* [Cout_pad, K] K-major head of the split weights: fp32 holding TF32 values (impl 1,2)
                                                 or fp16 (impl 3) */
  const void *w_nk_lo;                        /* remainder, same layout: RN_tf32(w - hi), or RN_f16((w - hi) * 2^11) */
  int Cout;  int K_pad;
  const float *pre_scale, *pre_shift;  int pre_img_stride;  int pre_relu;
  const float *post_scale, *post_shift;  int post_relu;
  const float *res;  long long res_ld;  int res_H, res_W, res_stride;
  float *out;  long long out_ld;
  int impl;
  const void *tmap_hi, *tmap_lo;              /* HOST pointers to 128-byte CUtensorMap blobs from hd_make_weight_tmap */
  /* Pre-split activations (impl 3 only).  When in_hi/in_lo are set the A operand is read from two fp16 arrays of the
   * same [pixels, in_ld] geometry as `in` (hi = RN_f16(a), lo = RN_f16((a - hi) * 2^11), a = the ALREADY pre-activated
   * input) with cp.async straight into the swizzled tile -- no register staging, no prologue (pre_scale must be NULL).
   * When out_hi/out_lo are set the epilogue additionally (or, with out == NULL, only) writes
   *   y = v * post2_scale[co] + post2_shift[co]; if post2_relu: y = max(y, 0)      (NULL scale/shift = 1 / 0)
   * as such a pair [pixels, out2_ld]: the next layer's pre-activated, pre-split A operand. */
  const void *in_hi, *in_lo;
  void *out_hi, *out_lo;  long long out2_ld;
  const float *post2_scale, *post2_shift;  int post2_relu;
  /* Activation tensor maps (impl 3, pre-split input, Cout % 32 == 0, residual row == output row): HOST pointers to 128-byte
   * CUtensorMap blobs from hd_make_act_tmap over `res`, `out`, `out_hi`, `out_lo` (each required iff that pointer is set).
   * The sm_90a kernel does not read them: it encodes its own residual and output maps from `res`, `out`, `out_hi` and `out_lo`
   * on every launch, and results do not depend on these maps or on HD_CONV_NO_TMA_EPILOGUE in `flags`.  They are kept only for
   * ABI compatibility: out_subsample (below) is still accepted exactly when they are given and the flag is unset. */
  const void *tmap_res, *tmap_out, *tmap_out_hi, *tmap_out_lo;
  int flags;
  /* optional: weight maps to use instead of tmap_hi / tmap_lo (64-row box; the kernel loads a 64- or 128-wide N tile as one or
   * two boxes); give both or neither
   * (tmap_lo_n64 may be NULL for impl 2), else HD_ERR_INVALID. */
  const void *tmap_hi_n64, *tmap_lo_n64;
  /* out_subsample = s > 1 (only with the activation tensor maps above and HD_CONV_NO_TMA_EPILOGUE unset; HD_ERR_UNSUPPORTED
   * elsewhere): `out` is a dense [n_img, ceil(Ho/s), ceil(Wo/s), Cout]
   * tensor that receives only the output pixels with oy % s == 0 and ox % s == 0 -- i.e. x[:, ::s, ::s, :], slim's identity shortcut
   * of the NEXT, strided unit (max_pool2d(x, [1,1], stride), A.4), written by the producing conv3 itself: the full-resolution fp32
   * block output has no other reader (the next unit's convs read out_hi / out_lo), so 3/4 of it is never written and no separate
   * hd_subsample pass runs.  out_ld is the row pitch of that dense tensor; tmap_out is not used.  0 / 1 = off. */
  int out_subsample;
} hd_conv_desc;

enum {
  HD_CONV_NO_TMA_EPILOGUE = 1,
  /* in_hi / in_lo are the padded RGBX fp16 planes written by hd_pack_conv1_planes / hd_process_image_planes: the 7x7 stride-2
   * conv1 of the ResNet root is then described as Cin = 32 (one kernel row = 8 pixels x 4 channels, 7 real + 1 zero-weight),
   * KH = 8 (7 real + 1 zero-weight), KW = 1, stride = 2, pad = 0, H = Hi + 6, W = even(Wi + 8), in_ld = 4, K = 256. */
  HD_CONV_INPUT_PLANES = 2
};

int hd_conv_gemm(const hd_conv_desc *d, void *stream);
/* Same launch; additionally CTA (0,0) of the tensor-core kernel writes per-role clock64 counters to dbg[0..15]
 * (device int64; layout in conv_simt.cu).  Tuning aid, not part of the reference surface. */
int hd_conv_gemm_profile(const hd_conv_desc *d, void *stream, long long *dbg);

/* Encode the TMA descriptor (CUtensorMap, 128 B, written to host memory `tmap_out`) for a K-major weight matrix
 * [rows, k_pad] of elem_bytes-wide elements (4 = fp32/tf32 path, 2 = fp16 path) with a {128 bytes x box_rows} box and
 * 128-byte swizzle.  box_rows must be 64 (the tensor-core kernel loads its 64- or 128-wide N tile as one or two boxes) and
 * divide rows. */
int hd_make_weight_tmap(const void *w_nk, int rows, int k_pad, int box_rows, int elem_bytes, void *tmap_out);
/* Same for a row-major activation matrix [rows, cols] with leading dimension ld_elems (elem_bytes 4 = fp32, 2 = fp16): box
 * {32 columns x 128 rows}, 128-byte (fp32) / 64-byte (fp16) swizzle (see tmap_res above). */
int hd_make_act_tmap(const void *base, long long rows, int cols, long long ld_elems, int elem_bytes, void *tmap_out);

/* ---- ResNet root / tail pieces (slim resnet_v2_50, called from src/models.py:65-74) ---- */
/* Input of the tensor-core conv1 (HD_CONV_INPUT_PLANES): img fp32 [N,H,W,3] -> two fp16 planes [N, H+6, WP, 4] (head and
 * 2^11-scaled remainder of every sample, channel 3 = 0), the image at row/column offset 3 inside a zero border that the
 * caller clears ONCE (the kernel writes the interior only).  WP = plane row length in pixels (even, >= W + 8). */
int hd_pack_conv1_planes(const float *img, void *plane_hi, void *plane_lo, int N, int H, int W, int WP, void *stream);
/* conv1: 7x7 stride 2, explicit zero pad 3+3, + bias.  in [N,H,W,3] -> out [N,H/2,W/2,64]; w [7*7*3,64]. */
int hd_conv1_7x7s2(const float *in, const float *w, const float *bias, float *out, int N, int H, int W, void *stream);
/* pool1: 3x3 stride 2 max pool, TF SAME padding (pad 0 top/left, 1 bottom/right for even sizes).
 * Optional second output (out_hi/out_lo non-NULL): relu(v*scale[c] + shift[c]) as an fp16 head/remainder pair
 * (the first bottleneck unit's pre-activation, pre-split for the tensor-core kernel); `out` may then be NULL (the first unit's
 * shortcut is a conv of the pre-activation, so nobody reads the fp32 pool output). */
int hd_maxpool3x3s2_same(const float *in, float *out, int N, int H, int W, int C, const float *scale, const float *shift,
                         void *out_hi, void *out_lo, void *stream);
/* slim's identity shortcut of a strided unit: max_pool2d(x, [1,1], stride) = x[:, ::s, ::s, :] (A.4).  in [N,H,W,C] -> out
 * [N,ceil(H/s),ceil(W/s),C]; lets the residual of the unit's conv3 be a plain row-aligned tensor. */
int hd_subsample(const float *in, float *out, int N, int H, int W, int C, int stride, void *stream);
/* postnorm BN+ReLU then global mean over HxW: in [N,HW,C] -> out [N,C]. */
int hd_bnrelu_avgpool(const float *in, const float *scale, const float *shift, float *out, int N, int HW, int C, void *stream);

/* ---- training-mode batch norm (slim batch_norm with is_training=True; resnet_arg_scope, src/models.py:65-74 under
 * trainer_sequence_fc.py:562-575).  x is an NHWC map viewed as [rows, C] with row pitch ld floats (rows = frames x H x W).  Writes
 *   mean_b[c] = mean over the rows, var_b[c] = biased variance over the rows (both accumulated in fp64 about row 0's value),
 *   scale[c] = gamma[c] / sqrt(var_b + eps), shift[c] = beta[c] - mean_b * scale    (the pre_* / post_* vectors of hd_conv_gemm)
 * and, when `mean` / `var` are non-NULL, mean_b / var_b as fp32.  When moving_mean / moving_var are non-NULL (both or neither) they
 * take one in-place float32 step of TF's assign_moving_average: m -= (m - v) * (float)(1 - decay), with v = mean_b for the mean and
 * the Bessel-corrected var_b * rows / (rows - 1) for the variance.  Partials per fixed chunk of rows are merged in a fixed order:
 * repeats are bit-identical.  `workspace` (16-byte aligned) holds hd_bn_stats_workspace_bytes(rows, C) bytes.  x 16-byte aligned,
 * C % 4 == 0, ld % 4 == 0, ld >= C, rows >= 2, else HD_ERR_INVALID and nothing is launched. */
size_t hd_bn_stats_workspace_bytes(long long rows, int C);
int hd_bn_batch_stats(const float *x, long long rows, int C, long long ld, const float *gamma, const float *beta, float eps,
                      float *scale, float *shift, float *mean, float *var, float *moving_mean, float *moving_var, double decay,
                      void *workspace, size_t workspace_bytes, void *stream);
/* The same moving-average step from a saved mean_b / var_b (the fp32 outputs of hd_bn_batch_stats over `rows` rows), bit-identical to
 * the step hd_bn_batch_stats takes itself: lets a trainer apply the update ops of an iteration after its forward pass. */
int hd_bn_moving_update(const float *mean, const float *var, long long rows, int C, double decay, float *moving_mean, float *moving_var,
                        void *stream);

/* ---- backward of the training-mode trunk (csrc/resnet_grad.cu): what the ResNet needs to train with freeze_phi=False
 * (trainer_sequence_fc.py:681-685).  Deterministic: no atomics, every sum over a partition fixed by the shapes and merged in a fixed
 * order, so repeats are bit-identical and results do not depend on the device's SM count.  Every argument is checked before any launch
 * (HD_ERR_INVALID). ----
 * hd_conv_wgrad: the weight gradient of a conv with hd_conv_gemm's geometry (x [n_img, H, W, Cin] at pixel pitch x_ld; output
 *   [n_img, Ho, Wo, Cout]; input pixel of (oy, ox, ky, kx) = (oy*stride - pad_t + ky, ox*stride - pad_l + kx), zero outside):
 *     dw[(ky*KW + kx)*Cin + ci, co] = sum_{n,oy,ox} a[n, iy, ix, ci] * dy[(n*Ho + oy)*Wo + ox][co]     (dy row pitch dy_ld)
 *     a = relu(fma(x, pre_scale[ci], pre_shift[ci])) on real pixels when pre_scale is given (hd_conv_gemm's prologue; padding stays 0),
 *     else x;   db[co] = sum of dy's column co (when db is non-NULL: one extra all-ones row of the GEMM's A operand).
 *   An implicit GEMM on the tensor cores (wgmma m64n64k8 in the 3xTF32 split; a producer warpgroup gathers and splits the operands
 *   into a 3-stage shared-memory ring, float4 gathers when Cin, Cout, x_ld, dy_ld % 4 == 0 and x, dy are 16-byte aligned), reduced over
 *   the pixels in fixed chunks of 2048 whose fp32 partials hd_conv_wgrad_workspace_bytes(n_img*Ho*Wo, KH*KW*Cin, Cout, db != NULL)
 *   bytes of workspace hold (the bias: per-chunk column sums of dy taken while loading it); a second launch adds them in chunk order
 *   in fp64. */
size_t hd_conv_wgrad_workspace_bytes(long long pixels, int K, int Cout, int bias);
int hd_conv_wgrad(const float *x, long long x_ld, int n_img, int H, int W, int Cin, int Ho, int Wo, int KH, int KW, int stride, int pad_t,
                  int pad_l, const float *pre_scale, const float *pre_shift, const float *dy, long long dy_ld, int Cout, float *dw, float *db,
                  void *workspace, size_t workspace_bytes, void *stream);
/* hd_bn_relu_backward: training-mode batch norm + ReLU backward over the raw map x [rows, C] (dense) that hd_bn_batch_stats normalised
 * into scale / shift (and its biased variance var), gamma the layer's gamma:
 *   z = fma(x, scale, shift), g = dz * (z > 0)  (TF's ReluGrad is 0 at 0), xhat = (x - mean_b) * rstd, rstd = 1 / sqrt(var + eps)
 *   dbeta = sum_rows g,  dgamma = sum_rows g * xhat,  dx = gamma * rstd * (g - mean(g) - xhat * mean(g * xhat)) + addend
 * with the batch mean re-accumulated in fp64 about row 0 (as hd_bn_batch_stats does), fp64 chunk partials merged in a fixed order.
 * dz: [rows, C], or with dz_group > 1 [rows / dz_group, C] broadcast over each group of dz_group rows and divided by dz_group (the
 * gradient of a mean over H x W: the tail's global pooling).  addend (nullable): added to dx, [rows, C]; with add_stride > 1 it is the
 * dense [frames, ceil(add_H/s), ceil(add_W/s), C] gradient of x[:, ::s, ::s] (the strided identity shortcut), scattered to every s-th
 * row and column of the [frames, add_H, add_W] map.  dx must not alias x, dz or addend.  Three launches; workspace
 * hd_bn_relu_backward_workspace_bytes(rows, C) (16-byte aligned); C % 4 == 0, x 16-byte aligned, rows >= 2. */
size_t hd_bn_relu_backward_workspace_bytes(long long rows, int C);
int hd_bn_relu_backward(const float *x, const float *dz, int dz_group, long long rows, int C, const float *scale, const float *shift,
                        const float *var, const float *gamma, float eps, const float *addend, int add_H, int add_W, int add_stride,
                        float *dx, float *dgamma, float *dbeta, void *workspace, size_t workspace_bytes, void *stream);
/* Backward of hd_maxpool3x3s2_same (pool1): in [N,H,W,C] the pool's input, dout [N,ceil(H/2),ceil(W/2),C] -> din [N,H,W,C].  Each window
 * sends its gradient to one input, its FIRST maximum in scan order (ky, then kx) [TF-ext: TF's CPU MaxPoolGrad]; computed as a gather
 * (each input adds the windows that chose it, in window order).  din must not alias in / dout. */
int hd_maxpool3x3s2_same_backward(const float *in, const float *dout, float *din, int N, int H, int W, int C, void *stream);
/* out [N,Ho,Wo,C] = in [N,Hi,Wi,C] spread to every stride-th row and column (out[n, y, x] = in[n, y/s, x/s] where y % s == 0 and
 * x % s == 0, else 0): with it, the data gradient of a stride-s conv2d_same 3x3 is a stride-1 SAME conv over the flipped weights. */
int hd_zero_insert(const float *in, float *out, int N, int Hi, int Wi, int C, int stride, int Ho, int Wo, void *stream);

/* ---- crop pre-processing, the caller of the path: process_image (src/evaluation/run_video.py:56-107) + resize_img
 * (src/util/common.py:7-14), batched.  frames uint8 [N,H,W,3]; geom int32 [N,4] (16-byte aligned) = {Hs, Ws, x0, y0}: size of the
 * cv2.resize'd frame and the top-left corner of the SxS crop in its coordinates (may lie outside: edge replication = the
 * reference's np.pad(mode='edge')); out fp32 [N,S,S,3] = crop of resize(2*(frame/255 - 0.5)) (bilinear, cv2 conventions).
 * plane_hi / plane_lo (optional, both or neither; then `out` may be NULL): the same crop written directly as the padded RGBX
 * fp16 planes [N,S+6,WP,4] the tensor-core conv1 reads (hd_pack_conv1_planes layout; border cleared once by the caller). */
int hd_process_image(const unsigned char *frames, int N, int H, int W, const int *geom, float *out, int S, void *plane_hi,
                     void *plane_lo, int WP, void *stream);
/* Host bookkeeping of process_image for one frame (no CUDA call): bbox = {cx, cy, scale} as float64 -> geom = the {Hs, Ws, x0, y0} row
 * hd_process_image takes, and optionally the reference's `center` (after the crop) and `start_pt` (in the edge-padded scaled image)
 * (run_video.py:69-100; floor / round-half-to-even in double like the reference's numpy code).  HD_ERR_INVALID when the reference would
 * return a crop smaller than img_size x img_size. */
int hd_crop_geometry(int H, int W, const double *bbox, int img_size, int *geom, int *center, int *start_pt);

/* ---- training-time tube augmentation: TubePreprocessor.preprocess_image (src/util/tube_augmentation.py:114-186 with
 * src/util/data_utils.py's jitter_center, jitter_scale, pad_image_edge, rotate_img, flip_image), per frame, F frames of one
 * source size H x W from any number of tubes.  Two launches, no host synchronisation:
 *   1. one thread per frame: centre + trans; sf = 2^scale; Hs = int(float(H) * sf), Ws likewise; keypoints and centre scaled by
 *      Hs/H, Ws/W (centre truncated); the S x S slice of the edge-padded scaled image around it; with HD_AUG_ROTATE, rotate_img by
 *      rot[f] (keypoints about (S/2, S/2), gt3d about its scalar mean, pose[:3] <- rot2aa(R^T rodrigues(pose[:3]))); where flip[f]
 *      is set, flip_image (25-keypoint swap, reflect_pose, reflect_joints3d); labels -> [2x/S - 1, 2y/S - 1, vis > 0] * (vis > 0).
 *      Writes the frame's geometry row and the transformed labels.
 *   2. one thread per output pixel: the crop straight from the source frame (TF 1.x resize_bilinear taps, edge replication by
 *      clamping into the scaled image, contrib.image.rotate's bilinear taps with zero fill, the width mirror), then (v - 0.5) * 2.
 * frames: uint8 [F,H,W,3] (HD_AUG_SRC_U8; value = u8 / 255 in float32) or float32 [F,H,W,3] in [0, 1].  Walks: trans int32 [F,2]
 * (x, y), scale float32 [F], rot float32 [F] (HD_AUG_ROTATE only, else ignored), flip int32 [F] (HD_AUG_FLIP only, else ignored).
 * Labels: labels float32 [F,3,K] (x row, y row, visibility row), centers int32 [F,2] (x, y), poses float32 [F,72], gt3ds float32
 * [F,14,3]; the *_out arrays have the same shapes (centers_out = the scaled jittered centre, the reference's `centers`).
 * geom int32 [F,16] (16-byte aligned): {Hs, Ws, cx, cy, x0, y0, flip, 0} then, as float bits, the rotation's projective
 * transform a0..a5 and the resize steps H/Hs, W/Ws; (x0, y0) = the crop's top-left corner in the scaled image.
 * Outputs: crops float32 [F,S,S,3] in [-1, 1] and / or plane_hi / plane_lo, the padded RGBX fp16 planes [F,S+6,WP,4] of
 * hd_pack_conv1_planes (border cleared once by the caller).  A centre whose crop leaves the edge-padded image (where the reference's
 * tf.slice fails) is not an error here: the crop keeps clamping into the scaled image.  trans_max only enters the keypoints' float
 * rounding (the reference pads by S/2 + trans_max + 50 before it slices).
 * HD_ERR_INVALID (before any launch): a null pointer, F, H, W, K or S <= 0, S odd, trans_max < 0, an unknown flag bit, HD_AUG_FLIP
 * with K != 25, or a bad plane layout (WP even and >= S + 8, 16-byte aligned planes). */
#define HD_AUG_SRC_U8 1
#define HD_AUG_ROTATE 2
#define HD_AUG_FLIP 4
typedef struct {
  const void *frames;
  int F, H, W, flags;
  const int *trans;
  const float *scale, *rot;
  const int *flip;
  const float *labels;
  int K;
  const int *centers;
  const float *poses, *gt3ds;
  int S, trans_max;
  int *geom;
  float *labels_out;
  int *centers_out;
  float *poses_out, *gt3ds_out;
  float *crops;
  void *plane_hi, *plane_lo;
  int WP;
} hd_tube_aug_args;                                   /* host struct */
int hd_tube_augment(const hd_tube_aug_args *a, void *stream);

/* ---- f_movie GroupNorm statistics (tf.contrib.layers.group_norm at src/models.py:155,188) ----
 * x [B,T,C]; per (clip, group) mean / biased variance over T*(C/groups) elements (two-pass);
 * gain[b,c] = rsqrt(var+eps)*gamma[c]; offset[b,c] = beta[c] - mean*gain[b,c]. */
int hd_groupnorm_stats(const float *x, const float *gamma, const float *beta, float *gain, float *offset,
                       int B, int T, int C, int groups, float eps, void *stream);

/* GroupNorm + ReLU straight to the tensor-core conv's A operand format: y = relu(group_norm(x)) as an fp16 head / 2^11-scaled
 * remainder pair [B*T, C] (same statistics and affine as hd_groupnorm_stats + the conv prologue).  T * C/groups <= 1280. */
int hd_groupnorm_relu_split(const float *x, const float *gamma, const float *beta, void *out_hi, void *out_lo, int B, int T, int C,
                            int groups, float eps, void *stream);
/* fp32 [n] -> fp16 head / remainder pair (n % 4 == 0, 16-byte aligned). */
int hd_split_f16(const float *x, void *hi, void *lo, long long n, void *stream);

/* ---- IEF pieces too small / too narrow for the tensor-core tile (src/models.py:101-113,400-413) ----
 * fc1, theta part: h1 = relu(P + theta . W) with P [N,C] = phi . W1[:2048] + b1 (hoisted), theta rows of K <= 96 at stride theta_ld,
 * W [K,C]; writes h1 as an fp16 head / remainder pair (fc2's A operand) and / or fp32. */
int hd_ief_fc1_theta(const float *P, const float *theta, int theta_ld, const float *W, int K, int C, void *out_hi, void *out_lo,
                     float *out_f32, int N, void *stream);
/* fc3 + IEF update: out[n, :D] = prev[n, :D] + h2[n] . W + bias, h2 [N,K] (K % 64 == 0), W [K,D], D <= 96; fixed summation order. */
int hd_ief_fc3(const float *h2, const float *W, const float *bias, const float *prev, int prev_ld, float *out, int out_ld, int N, int K,
               int D, void *stream);

/* ---- IEF glue (src/models.py:349-371): dst[n*dst_ld + :85] = [1, 0, 0, theta[n,3:75], theta[n,75:85]] ---- */
int hd_ief_delta_init(const float *theta, float *dst, int dst_ld, int N, void *stream);

/* ---- network-level entries (SURVEY.md 8b): library-owned layer plans for the three networks on the path ----
 * A plan packs the TF-named weights once (BatchNorm folded, K-major fp16 head / remainder split, TMA descriptors) and owns its
 * activation buffers: `*_create` allocates device memory and copies weights (synchronous, once); `*_forward` is a fixed sequence of
 * the per-layer entries above on `stream` -- no allocation, no synchronisation -- and is bit-identical to the Python host plans
 * (human_dynamics_b200/nets.py).  Precision mode: HD_IMPL_TC_3XF16 (FP32-class).
 * Weights are pulled through a callback: get(user, "<TF variable name>", &numel) returns a HOST pointer to the fp32 array in the
 * TensorFlow layout (conv HWIO, FC [in,out]) -- e.g. "resnet_v2_50/block1/unit_1/bottleneck_v2/conv1/weights" -- or NULL if absent
 * (then create fails with HD_ERR_INVALID and hd_net_error names the variable); the arrays only have to stay valid during `*_create`.
 * A plan is bound to the device that was current at creation and is not re-entrant: one `*_forward` at a time per hd_net (its
 * activation buffers are the state); use one plan per stream for concurrency.  `*_forward` can be captured in a CUDA graph.
 * hd_net_destroy frees the device memory immediately: synchronise the streams that used the plan first. */
typedef struct hd_net hd_net;
typedef const float *(*hd_weight_fn)(void *user, const char *tf_name, long long *numel);
void hd_net_destroy(hd_net *net);
const char *hd_net_error(const hd_net *net);
long long hd_net_num_launches(const hd_net *net);
/* encoder_resnet (src/models.py:50-77): images [n_frames,size,size,3] fp32 in [-1,1] -> phi [n_frames,2048].  size even. */
int hd_resnet50_create(hd_weight_fn get, void *user, int n_frames, int size, hd_net **net);
int hd_resnet50_forward(hd_net *net, const float *images, float *phi, void *stream);
/* az_fc2_groupnorm (src/models.py:121-228): phi [B,T,2048] -> movie strips [B,T,2048] (out != phi).  T <= 20. */
int hd_fmovie_create(hd_weight_fn get, void *user, int B, int T, int num_conv_layers, hd_net **net);
int hd_fmovie_forward(hd_net *net, const float *phi, float *out, void *stream);
/* call_hmr_ief (src/models.py:299-415) as wired by tester.py:196-207 (scope single_view_ief, 3 stages, use_optcam, deltas started
 * from the main prediction): phi [N,2048] -> theta [N,85] and, for the num_delta non-zero delta_t values in ascending order,
 * deltas [N,num_delta,85] = [1,0,0 | pose | beta].  IEF starts from the checkpoint's `mean_param`. */
int hd_ief_create(hd_weight_fn get, void *user, int N, const int *delta_t, int num_delta, hd_net **net);
int hd_ief_forward(hd_net *net, const float *phi, float *theta, float *deltas, void *stream);

/* ---- SMPL (src/tf_smpl/batch_smpl.py:26-162, batch_lbs.py:15-60,133-194, projection.py:16-29) ---- */
typedef struct {
  int num_verts, num_kps, lbs_nnz, kp_nnz_total;
  const float *v_template;     /* [V*3] */
  const float *dirs;           /* [10+207, V*3]: shapedirs rows then posedirs rows (batch_smpl.py:45-48,60-63) */
  const float *J_template;     /* [24*3]  = J_regressor^T v_template */
  const float *J_shapedirs;    /* [10, 24*3] = J_regressor^T shapedirs  (exact refactoring of batch_smpl.py:110-118) */
  const int *lbs_idx;          /* [V, lbs_nnz] joint ids of the non-zero skinning weights (padded with weight 0) */
  const float *lbs_w;          /* [V, lbs_nnz] */
  const int *kp_ptr;           /* [K+1] CSC offsets into kp_vidx / kp_w (cocoplus_regressor, batch_smpl.py:76-82) */
  const int *kp_vidx;          /* [kp_nnz_total] */
  const float *kp_w;           /* [kp_nnz_total] */
  int parents[24];             /* kintree_table[0] as int32 (root -1), batch_smpl.py:66 */
} hd_smpl_consts;

/* Host-side packing of the SMPL model (the contents of the official pickle as dense float64 arrays) into the arrays hd_smpl_consts points
 * at -- what SMPL.__init__ does in the reference (batch_smpl.py:27-86) plus the layouts the kernels want.  Pure host code, no CUDA call:
 * the caller uploads the outputs and stores the device pointers in hd_smpl_consts.  All pointers are HOST memory.
 *   in : v_template [V,3], shapedirs [V,3,10], posedirs [V,3,207], J_regressor [24,V], weights [V,24], kp_regressor [K,V] (cocoplus_regressor,
 *        or its first 14 rows for joint_type 'lsp', batch_smpl.py:81-82), kintree_parents = kintree_table[0] as stored (uint32, root 4294967295)
 *   out: v_template_out [V*3] f32, dirs [217, V*3] f32, J_template [72] f32, J_shapedirs [10,72] f32, lbs_idx / lbs_w [V, lbs_nnz] (ELL: joint
 *        ids ascending, padding = joint 0 with weight 0), kp_ptr [K+1] / kp_vidx / kp_w [kp_nnz_total] (CSC over keypoints), parents int[24]
 * hd_smpl_pack_sizes reports lbs_nnz (4, or the per-vertex maximum rounded up to a multiple of 4, at most 24) and kp_nnz_total first. */
int hd_smpl_pack_sizes(int V, int K, const double *weights, const double *kp_regressor, int *lbs_nnz, int *kp_nnz_total);
int hd_smpl_pack(int V, int K, const double *v_template, const double *shapedirs, const double *posedirs, const double *J_regressor,
                 const double *weights, const double *kp_regressor, const unsigned int *kintree_parents, float *v_template_out, float *dirs,
                 float *J_template, float *J_shapedirs, int *lbs_idx, float *lbs_w, int lbs_nnz, int *kp_ptr, int *kp_vidx, float *kp_w,
                 int *parents);
size_t hd_smpl_workspace_bytes(int N);
/* beta rows of 10 at stride beta_ld, theta rows of 72 at stride theta_ld, cam rows of 3 at stride cam_ld (so the
 * three can alias columns [75:85], [3:75], [0:3] of one [N,85] omega buffer, src/omega.py:231-235).
 * verts [N,V,3], joints [N,K,3], Rs [N,24,3,3], Jtr [N,24,3]; cam + kps [N,K,2] optional (both or neither).
 * Any output pointer except verts may be NULL.  Pose n lands in output slot n*out_mul + out_off of every output
 * array (out_mul=1, out_off=0 = dense), so D delta heads can write the [B,T,D,...] stacking of tester.py:252-253
 * in place. */
int hd_smpl_forward(const hd_smpl_consts *c, const float *beta, int beta_ld, const float *theta, int theta_ld, int N,
                    float *verts, float *joints, float *Rs, float *Jtr,
                    const float *cam, int cam_ld, float *kps, int out_mul, int out_off,
                    void *ws, size_t ws_bytes, void *stream);
/* Staged form of the same computation for large batches: the dense shape/pose blend (batch_smpl.py:110-112,127-133) is one
 * [N,256] x [256, V*3] GEMM on the tensor cores (hd_conv_gemm over `coef` with the packed `dirs`, bias = v_template), so the
 * rest is HBM-shaped:  hd_smpl_pose (Rodrigues + FK; also writes the GEMM operand rows coef[n] = [beta | R-I | 0]) ->
 * hd_conv_gemm -> hd_smpl_lbs (skinning of the blended v_posed [N, vp_ld]) -> hd_smpl_joints (keypoints + projection).
 * ws of hd_smpl_pose: N*216 floats. */
int hd_smpl_pose(const hd_smpl_consts *c, const float *beta, int beta_ld, const float *theta, int theta_ld, int N, float *Rs,
                 float *Jtr, float *A12, float *coef /* fp32 rows, nullable */, int coef_ld,
                 void *coef_hi, void *coef_lo /* the same rows as an fp16 head / 2^11-scaled remainder pair, nullable */,
                 void *a12t_hi, void *a12t_lo /* [N,12,32] fp16 head / unscaled remainder of A transposed: operand of hd_smpl_lbs_tc, nullable */,
                 int out_mul, int out_off, void *ws, size_t ws_bytes, void *stream);
/* Skinning with the 6890x24 blend-weight x transform contraction on the tensor cores (batch_smpl.py:141-151):
 * w_hi / w_lo = dense skinning weights [roundup128(V), 32] (24 joints + zero padding) as an fp16 head / unscaled remainder pair;
 * a12t_hi / a12t_lo from hd_smpl_pose; v_posed [N, vp_ld] (vp_ld % 4 == 0, >= roundup4(3V)) -> verts slot n*out_mul + out_off. */
int hd_smpl_lbs_tc(const void *w_hi, const void *w_lo, const void *a12t_hi, const void *a12t_lo, const float *v_posed, long long vp_ld,
                   float *verts, int N, int V, int out_mul, int out_off, void *stream);
int hd_smpl_lbs(const hd_smpl_consts *c, const float *v_posed, long long vp_ld, const float *A12, float *verts, int N, int out_mul,
                int out_off, void *stream);
int hd_smpl_joints(const hd_smpl_consts *c, const float *verts, const float *cam, int cam_ld, float *joints, float *kps, int N,
                   int out_mul, int out_off, void *stream);
/* batch_rodrigues: theta [M,3] -> R [M,3,3]. */
int hd_rodrigues(const float *theta, float *R, int M, void *stream);
/* batch_rot2aa (src/tf_smpl/batch_lbs.py:63-105): R [M,3,3] -> axis-angle [M,3]. */
int hd_rot2aa(const float *Rs, float *aa, int M, void *stream);
/* batch_global_rigid_transformation: Rs [N,24,3,3], Js [N,24,3], parents host int[24] -> new_J [N,24,3], A [N,24,4,4]. */
int hd_global_rigid(const float *Rs, const float *Js, const int *parents_host, float *new_J, float *A44, int N,
                    int rotate_base, void *stream);
/* batch_orth_proj_idrot: X [N,P,3], cam [N,3] -> out [N,P,2]. */
int hd_orth_proj(const float *X, const float *cam, float *out, int N, int P, void *stream);

/* ---- SMPL backward (reverse mode of the forward above; gradients w.r.t. beta / theta / the helpers' inputs, never the constants) ----
 * Deterministic: no floating-point atomics, every reduction runs in a fixed order, and pose n's gradients depend only on pose n's
 * inputs and upstream gradients (bit-identical across launches, batch splits and permutations).  Any upstream gradient pointer marked
 * nullable stands for zeros.
 *
 * Extra model arrays the backward reads, packed once on the host (human_dynamics_b200/smpl.py:pack_grad_arrays) and passed explicitly:
 *   kpv_ptr [V+1] / kpv_kidx / kpv_w [kp_nnz_total]: the keypoint regressor vertex-major (CSR over vertices, keypoint ids ascending) --
 *     the transpose of hd_smpl_consts' CSC copy;
 *   lbt_ptr [num_tiles*24+1] / lbt_v / lbt_w: the non-zero skinning weights joint-major within each tile of HD_SMPL_GRAD_TILE vertices
 *     (entries of tile t, joint k at [lbt_ptr[t*24+k], lbt_ptr[t*24+k+1]), vertex ids ascending), num_tiles = ceil(V / HD_SMPL_GRAD_TILE).
 * Full sequence for one batch (see INTEGRATION.md):
 *   hd_smpl_pose (recompute A12 and the blend operand) -> hd_conv_gemm (recompute v_posed) -> hd_smpl_lbs_backward (g_v, dL/dv_posed,
 *   dL/dA) -> hd_conv_gemm (dL/dc = dL/dv_posed . dirs^T, 3xTF32) -> hd_smpl_pose_backward (FK + Rodrigues backward -> dL/dbeta, dL/dtheta).
 * hd_smpl_backward_workspace_bytes(N, V): one buffer holding, in this order and each at a 256-byte boundary, A12 f32 [N,288],
 * dA12 f32 [N,288], dc f32 [N,HD_SMPL_GRAD_CLD], rs f32 [N,216] (hd_smpl_pose's ws), coef_hi / coef_lo f16 [N,256] each,
 * v_posed f32 [N,vp_ld] and dv_posed f32 [N,vp_ld], vp_ld = roundup4(3V).  0 when N <= 0 or V <= 0. */
enum { HD_SMPL_GRAD_TILE = 256, HD_SMPL_GRAD_CLD = 224 };
typedef struct {
  int num_verts, num_kps, num_tiles, tile_verts;   /* tile_verts must be HD_SMPL_GRAD_TILE */
  const int *kpv_ptr;          /* [V+1] */
  const int *kpv_kidx;         /* [kp_nnz_total] */
  const float *kpv_w;          /* [kp_nnz_total] */
  const int *lbt_ptr;          /* [num_tiles*24+1] */
  const int *lbt_v;            /* [lbt_ptr[num_tiles*24]] */
  const float *lbt_w;          /* [lbt_ptr[num_tiles*24]] */
} hd_smpl_grad_consts;
size_t hd_smpl_backward_workspace_bytes(int N, int V);
/* Skinning + keypoint backward (batch_smpl.py:141-157 reversed):  g_v = dverts_v + sum_k Kreg[k,v] djoints_k;
 * dv_posed_v = (sum_k w_vk R_k)^T g_v;  dA12_k = sum_v w_vk g_v (x) [v_posed_v; 1]  (rows of [R | t], 12 per joint).
 * v_posed [N, vp_ld] (recomputed), A12 [N,288] from hd_smpl_pose, dverts [N,V,3], djoints [N,K,3] (nullable) -> dv_posed [N, vp_ld]
 * (columns 3V..vp_ld-1 set to 0, so it can be the A operand of the dc GEMM), dA12 [N,288]. */
int hd_smpl_lbs_backward(const hd_smpl_consts *c, const hd_smpl_grad_consts *g, const float *v_posed, long long vp_ld, const float *A12,
                         const float *dverts, const float *djoints, float *dv_posed, float *dA12, int N, void *stream);
/* Pose-side backward, one warp per pose (batch_smpl.py:115-137, batch_lbs.py:42-60,133-194 reversed): recomputes J, R and the FK chain
 * from beta / theta, walks the tree levels in reverse from dA12 (nullable) and dJtr [N,24,3] (nullable), adds dRs [N,24,3,3] (nullable)
 * and dc[n, 10:217] (the pose-blend coefficients R_j - I, j = 1..23) to the local rotations, differentiates Rodrigues in fp64 (the
 * reference's expression with the +1e-8 shift; finite at theta = 0), and writes
 *   dbeta[n*dbeta_ld + b] = dc[n, b] + sum_j J_shapedirs[b, j] . dJ_j,   dtheta[n*dtheta_ld + 3j + i].
 * dc rows of >= 217 at stride dc_ld (nullable). */
int hd_smpl_pose_backward(const hd_smpl_consts *c, const float *beta, int beta_ld, const float *theta, int theta_ld, int N,
                          const float *dA12, const float *dc, int dc_ld, const float *dRs, const float *dJtr, float *dbeta, int dbeta_ld,
                          float *dtheta, int dtheta_ld, void *stream);
/* batch_rodrigues backward: theta [M,3], dR [M,3,3] -> dtheta [M,3]. */
int hd_rodrigues_backward(const float *theta, const float *dR, float *dtheta, int M, void *stream);
/* batch_global_rigid_transformation backward: Rs [N,24,3,3], Js [N,24,3], parents host int[24], dnew_J [N,24,3] (nullable),
 * dA [N,24,4,4] (nullable; its constant last rows are ignored) -> dRs [N,24,3,3], dJs [N,24,3]. */
int hd_global_rigid_backward(const float *Rs, const float *Js, const int *parents_host, const float *dnew_J, const float *dA44, float *dRs,
                             float *dJs, int N, int rotate_base, void *stream);
/* batch_orth_proj_idrot backward: X [N,P,3], cam [N,3], dout [N,P,2] -> dX [N,P,3] (z column 0), dcam [N,3]:
 * dX_xy = s dout, ds = sum_p (xy + t) . dout_p, dt = s sum_p dout_p. */
int hd_orth_proj_backward(const float *X, const float *cam, const float *dout, float *dX, float *dcam, int N, int P, void *stream);

/* ---- Backward of the trainable layers: f_movie, the IEF heads and fc2_res (csrc/net_grad.cu) ----
 * The GEMMs of the backward run on hd_conv_gemm in its 3xTF32 mode (gradients carry an arbitrary scale, so they never go through the
 * fp16 split with its +-65504 clamp); the entries below supply its operands and the non-GEMM parts.  For a KH x 1 SAME conv over T
 * (f_movie, KH = 3, pad 1) or an FC layer (KH = 1, pad 0) with input x [B*T, Cin], weight W [KH, Cin, Cout] (TF HWIO) and output
 * gradient dY [B*T, Cout]:
 *   dX = conv(dY, W'), W'[k', co, ci] = W[KH-1-k', ci, co]        hd_conv_gemm (3xTF32, in = dY) over hd_pack_weight(BACKWARD_DATA)
 *   dW = Xcol^T . dY   (M = KH*Cin, N = Cout, K = B*T)            hd_conv_gemm (3xTF32) with in = hd_im2col_t(x) as [KH*Cin, K_pad]
 *                                                                 pixels and the B operand hd_transpose_split(dY, tf32) [Cout_pad, K_pad]
 *   db = column sums of dY                                        hd_col_sum
 * Deterministic: no floating-point atomics, every reduction in a fixed order; an input gradient's row depends only on that row. */
enum { HD_PACK_FORWARD = 0, HD_PACK_BACKWARD_DATA = 1 };
/* Device-side weight packing into the K-major [rows, k_pad] head / remainder layout of hd_conv_gemm's B operand (TMA maps from
 * hd_make_weight_tmap); the only writer of that layout.  w: fp32 [KH, Cin, Cout]: an FC [in, out] with KH = 1, or, in forward mode, any
 * HWIO conv with KH*KW passed as KH (backward-data mode too: the flip of the flattened (ky, kx) index, KH*KW-1-k, is the 2-D flip
 * (KH-1-ky, KW-1-kx), so a KH x KW conv's pack is its dX conv over dY with SAME padding mirrored).  elem_bytes 2 = fp16 head / 2^11-scaled remainder (impl 3), 4 = TF32
 * head / remainder in fp32 storage (impl 1).
 *   HD_PACK_FORWARD:       dst[co, kh*Cin + ci] = W[kh, ci, co]  (hi = RN_f16(w), lo = RN_f16((w - hi) * 2^11); TF32: hi = RN_tf32(w),
 *                          lo = RN_tf32(w - hi));
 *   HD_PACK_BACKWARD_DATA: dst[ci, k'*Cout + co] = W[KH-1-k', ci, co]  (FC: W^T).
 * Rows / columns past the matrix are zero.  rows % 64 == 0, k_pad % 32 (tf32) / % 64 (fp16) == 0, hi / lo 16-byte aligned. */
int hd_pack_weight(const float *w, int KH, int Cin, int Cout, int mode, int elem_bytes, void *hi, void *lo, int rows, int k_pad, void *stream);
/* Transpose with optional split: hi[r*out_ld + k] (and lo) = split(x[k*ld + r]) for r < cols, k < rows; 0 for r in [cols, out_rows) or
 * k in [rows, out_cols).  mode 0 = plain fp32 (lo NULL), 1 = TF32 head / remainder, 2 = fp16 head / 2^11-scaled remainder.  Used for
 * the dY^T operand of a weight-gradient GEMM (mode 1; pass column offsets in hi / lo to stack several products along K) and for the
 * transposed inputs of FC weight gradients (mode 0). */
int hd_transpose_split(const float *x, long long rows, int cols, long long ld, int mode, void *hi, void *lo, long long out_ld, int out_rows,
                       long long out_cols, void *stream);
/* Transposing im2col of x [B, T, C] for a KH x 1 conv over T with `pad` leading zero taps:
 *   out[(kh*C + c)*out_ld + b*T + t] = a[b, t + kh - pad, c]  (0 outside the clip), columns [B*T, out_cols) = 0,
 *   a = x, or with gain / offset [B, C] (hd_groupnorm_stats) a = x*gain + offset, then ReLU when relu != 0. */
int hd_im2col_t(const float *x, int B, int T, int C, int KH, int pad, const float *gain, const float *offset, int relu, float *out,
                long long out_ld, long long out_cols, void *stream);
/* GroupNorm (+ ReLU) backward (tf.contrib.layers.group_norm, A7).  Recomputes mean / rstd per (clip, group) with the arithmetic of
 * hd_groupnorm_stats; with z = x*gain + offset the forward's pre-ReLU value, g = dy * (z > 0) (relu != 0; TF's ReluGrad is 0 at 0),
 * x^ = (x - mean)*rstd, g^ = g*gamma:  dx = rstd*(g^ - mean(g^) - x^*mean(g^ x^)) + addend (nullable), and per-clip partials
 * dgamma_part[b, c] = sum_t g x^, dbeta_part[b, c] = sum_t g (reduce over clips with hd_col_sum).  Any T; dx must not alias x / dy. */
int hd_groupnorm_relu_backward(const float *x, const float *gamma, const float *beta, const float *dy, const float *addend, float *dx,
                               float *dgamma_part, float *dbeta_part, int B, int T, int C, int groups, float eps, int relu, void *stream);
/* out[c] = sum over rows of x[r*ld + c], fixed order (bias gradients, GroupNorm affine gradients, mean_param). */
int hd_col_sum(const float *x, long long rows, int cols, long long ld, float *out, void *stream);
/* dx[i] = y[i] > 0 ? dy[i] : 0 (y = the ReLU's output; dx may alias dy). */
int hd_relu_backward(const float *y, const float *dy, float *dx, long long n, void *stream);
/* Short-K input gradient of an FC layer with D <= 96 outputs (the IEF fc3, D = 85 / 72):
 * out[n, k] = (mask[n, k] > 0) * sum_j g[n*g_ld + j] * Wt[j, k], Wt = W^T [D, K] fp32, out / mask dense [N, K] (mask nullable). */
int hd_fc_small_dgrad(const float *g, int g_ld, const float *Wt, int K, int D, const float *mask, float *out, int N, void *stream);
/* out[r, c] = a[r, c] + b[r, c] at independent row strides (out may alias a or b): gradient accumulation of the IEF glue. */
int hd_add_strided(const float *a, long long lda, const float *b, long long ldb, float *out, long long ldo, int rows, int cols, void *stream);

/* ---- Adversarial pose prior D_pose (src/discriminators.py; csrc/dpose.cu) ----
 * Input x [N, 23, 9]: the rotation matrices of the 23 non-root joints.  Variables (TF HWIO / [in, out], fp32):  D_conv1 W1 [9, 32], b1;
 * D_conv2 W2 [32, 32], b2; the heads pose_out_j0..22 stacked as wj [23, 32], bj [23]; D_alljoints_fc1 [736, 1024], fc2 [1024, 1024]
 * (both on hd_conv_gemm); D_alljoints_out w_out [1024], b_out [1].  Output logits [N, 24] (row stride 24):
 *   h1 = relu(x W1 + b1), h2 = relu(h1 W2 + b2)  [N, 23, 32]        hd_dpose_trunk_forward (also logits[:, j] = h2[:, j] . wj[j] + bj[j])
 *   f1 = relu(h2 [N, 736] . Wfc1 + bfc1), f2 = relu(f1 . Wfc2 + bfc2)  hd_conv_gemm (h2 is its input as written, in_ld 736)
 *   logits[:, 23] = f2 . w_out + b_out                             hd_dpose_out_forward
 * Backward of an upstream g [N, 24]: df2 = g[:, 23] w_out^T * (f2 > 0) (hd_fc_small_dgrad, D = 1), df1 and dflat [N, 736] by hd_conv_gemm
 * (3xTF32) dX with hd_relu_backward between them, then hd_dpose_trunk_backward: dx [N, 23, 9] (nullable) and, with a workspace of
 * hd_dpose_workspace_bytes(N), per-block partial sums that hd_dpose_grad_reduce sums into the packed gradient grad[HD_DPOSE_GRAD_FLOATS]:
 *   dW1 [9,32] @0 | db1 @288 | dW2 [32,32] @320 | db2 @1344 | dwj [23,32] @1376 | dbj @2112 | dw_out [1024] @2135 | db_out @3159.
 * Deterministic: a row's logits / dx depend on that row only; weight sums use a fixed partition and order, no atomics.
 * HD_ERR_INVALID: a null pointer, N <= 0, a workspace smaller than hd_dpose_workspace_bytes(N), or unaligned h / w_out (16 bytes). */
enum { HD_DPOSE_JOINTS = 23, HD_DPOSE_GRAD_FLOATS = 3160 };
size_t hd_dpose_workspace_bytes(int N);
int hd_dpose_trunk_forward(const float *x, const float *W1, const float *b1, const float *W2, const float *b2, const float *wj,
                           const float *bj, float *h1, float *h2, float *logits, int N, void *stream);
int hd_dpose_out_forward(const float *h, const float *w_out, const float *b_out, float *logits, int N, void *stream);
/* dflat = d flatten(h2) from fc1's dX; hf = f2 (read with ws); x is read with ws, W1 with dx. */
int hd_dpose_trunk_backward(const float *x, const float *h1, const float *h2, const float *dflat, const float *g, const float *hf,
                            const float *W1, const float *W2, const float *wj, float *dx, void *ws, size_t ws_bytes, int N, void *stream);
int hd_dpose_grad_reduce(const void *ws, size_t ws_bytes, int N, float *grad, void *stream);

/* ---- The trainer's encoder objective (src/trainer_sequence_fc.py:791-1018, src/ops.py, src/tf_smpl/projection.py; csrc/losses.cu) ----
 * One objective is a host array of term descriptors.  A term reads B clips x a window of Tw frames: frame f of clip b of a tensor X is
 * the row X + b * X_clip + (X_t0 + f) * X_frame (strides in floats; X_T = frames per clip, for the bound check).  Two kinds:
 *   HD_LOSS_KP_L1     sum_{b,f,k,c<2} v * |xhat - x| / (2 * #{v != 0}),  labels q [K, 3] = (x, y, v) per frame, p [K, D] (xy first).
 *                     xhat = s * (p_xy + t) with cam = (s, tx, ty) read at p's frame (HD_LOSS_KP_CAMERA, compute_loss_e_kp after
 *                     batch_orth_proj_idrot), the optimal camera of procrustes2d_vis over the points with v > 0 (HD_LOSS_KP_OPTCAM: 1e-6 I
 *                     before the 2 x 2 inverse, scale clipped to [0.7, 10], no gradient through it; written to cam_out [B, Tw, 3] when
 *                     given), or p_xy itself (HD_LOSS_KP_RAW).  A frame without a visible point in an OPTCAM term contributes 0 to value
 *                     and gradient and gets the camera (0.7, 0, 0) (the reference's value is NaN there).
 *   HD_LOSS_MSE_ROWS  scale * sum_{b,f,i<D} w[b] * (p - q)^2 / (D * #{rows with w[b] != 0}),  w NULL = 1, q NULL = 0; proj = 1 aligns
 *                     both rows by the pelvis first (rows of D / 3 >= 14 joints x 3, LSP hips 2 and 3: align_by_pelvis).
 * A count of 0 gives a value of 0.  The counts come from the weights alone.
 * hd_loss_forward writes values[n] with two launches (fixed-partition partial sums, fixed-order reduce) for any n; the workspace of
 * hd_loss_workspace_bytes(terms, n) (8-byte aligned) keeps the counts for the backward.  hd_loss_backward (one launch) WRITES grad for every target
 * {src, grad, numel}: for each element of src, the sum over the terms whose p / q (MSE) / cam (KP_CAMERA) lie inside src, in term order,
 * of dvalues[i] * d value_i / d element (dvalues: device, n floats); KP_L1 labels are constants (a target over them gets 0).  A target must be laid out like src (same strides); an element no
 * term reads gets 0.  L1's gradient at a residual of exactly 0 is 0.  Deterministic, no atomics; a frame's gradient depends only on
 * its own data, the counts and dvalues.  HD_ERR_INVALID (checked before any launch): null pointers, n outside [1, HD_LOSS_MAX_TERMS],
 * more than HD_LOSS_MAX_GRADS targets, B / Tw / D / K <= 0, a window that overruns X_T, pelvis alignment on rows of fewer than 14
 * joints, a gradient through a side with frame stride 0, or a workspace smaller than hd_loss_workspace_bytes (which is 0 for an
 * invalid list). */
enum { HD_LOSS_KP_L1 = 0, HD_LOSS_MSE_ROWS = 1 };
enum { HD_LOSS_KP_CAMERA = 0, HD_LOSS_KP_OPTCAM = 1, HD_LOSS_KP_RAW = 2 };
enum { HD_LOSS_MAX_TERMS = 64, HD_LOSS_MAX_GRADS = 16 };
typedef struct {
  int kind, proj;                 /* HD_LOSS_KP_L1: HD_LOSS_KP_*;  HD_LOSS_MSE_ROWS: 1 = pelvis alignment, 0 = none */
  int B, Tw, p_t0, q_t0, p_T, q_T;
  int K, D;                       /* KP_L1: keypoints, floats per keypoint of p;  MSE_ROWS: K unused, floats per row */
  const float *p;
  long long p_clip, p_frame;
  const float *q;
  long long q_clip, q_frame;
  const float *cam;               /* KP_CAMERA only */
  long long cam_clip, cam_frame;
  const float *w;                 /* MSE_ROWS: per-clip weights [B] or NULL */
  float *cam_out;                 /* KP_OPTCAM: [B, Tw, 3] or NULL */
  float scale;                    /* MSE_ROWS: the term's factor (0.5 for compute_loss_mse / _e_smooth); KP_L1: 1 */
} hd_loss_term;
typedef struct {
  const float *src;
  float *grad;
  long long numel;
} hd_loss_grad;
size_t hd_loss_workspace_bytes(const hd_loss_term *terms, int n);
int hd_loss_forward(const hd_loss_term *terms, int n, float *values, void *ws, size_t ws_bytes, void *stream);
int hd_loss_backward(const hd_loss_term *terms, int n, const hd_loss_grad *grads, int n_grads, const float *dvalues, const void *ws,
                     size_t ws_bytes, void *stream);

/* ---- Mesh rendering (the visualiser of src/util/render/nmr_renderer.py:43-240: NMR with camera_mode='look_at',
 * perspective=False, anti_aliasing and fill_back on), one colour per mesh.  The model is R1-R8 of oracle/render_ref.py:
 *   x = s*(X + tx), y = -s*(Y + ty), z = Z - eye_z  (R1); a 2S x 2S sample grid whose sample (r, c) sits at image
 *   ((2c + 1 - 2S) / 2S, (2r + 1 - 2S) / 2S), the convention of kps (R2); strict barycentric coverage (R3); depth 1/sum(w_i/z_i),
 *   dropped outside (near_z, far_z), nearest wins, ties to the lower face index (R4); each face once, lit with its eye-facing
 *   normal (R5): colour * (ambient + directional * relu(n . light_dir)), light_dir used as given (R6); pixel = mean of its 2x2
 *   samples with bg where empty, alpha = covered fraction (R7); out = uint8(rend) or, with a background image in [-1, 1],
 *   uint8(img255 * (1 - alpha) + rend * alpha), rend = clip(rgb, 0, 1) * 255, img255 = (img + 1) * 0.5 * 255, float32 (R8).
 * verts [N,V,3] with frame stride verts_ld floats (>= 3V), cam rows of 3 at stride cam_ld (so slices of verts_delta / omegas are read in
 * place); faces int32 [F,3] (a face with an index outside [0, V) is skipped); background [N,S,S,3] fp32 or NULL; out_rgb uint8
 * [N,S,S,3]; out_alpha fp32 [N,S,S] or NULL.  use_rot: vertices become rot * (v - mean_v) + mean_v with the per-frame vertex mean
 * (VisRenderer.rotated, nmr_renderer.py:176-225); rot is row-major.  Bit-identical across launches, batch sizes and chunkings.
 * Workspace: a [N, 2S, 2S] 64-bit z-buffer plus a [N, F] colour table, hd_render_workspace_bytes(N, S, F) bytes (0 when an
 * argument is <= 0).  When the stream reaches the end of the call, the workspace starts with that z-buffer: uint64
 * key = (float_bits(depth) << 32) | face per sample, all ones where empty (an inspection aid for tests and debugging).  HD_ERR_INVALID: a null pointer, S outside [1, 2048], N < 0, V or F <= 0, verts_ld < 3V or cam_ld < 3. */
typedef struct {
  float color[3], light_dir[3], ambient, directional, bg[3], near_z, far_z, eye_z;   /* NMR: eye_z = -(1/tan 30deg + 1) */
  float rot[9];
  int use_rot;
} hd_render_params;                                   /* host struct */
size_t hd_render_workspace_bytes(int N, int S, int F);
int hd_render_mesh(const float *verts, long long verts_ld, int N, int V, const int *faces, int F, const float *cam, int cam_ld,
                   const hd_render_params *p, const float *background /* [N,S,S,3] in [-1,1], nullable */, int S,
                   unsigned char *out_rgb /* [N,S,S,3] */, float *out_alpha /* [N,S,S], nullable */, void *ws, size_t ws_bytes,
                   void *stream);

/* ---- Evaluation (the per-frame metrics of src/evaluation/eval.py compute_errors_batched over eval_util.py) ----
 * hd_eval_frames: one launch, one warp per frame, for every frame of n_seq tubes laid end to end (device seq_start[n_seq + 1],
 * seq_start[0] = 0, non-decreasing, seq_start[n_seq] = N).  Writes one fp64 row of HD_EVAL_COLS per frame into out [N, HD_EVAL_COLS]:
 *   KP, KP_PA, KP_PCK   mean pixel error over the visible keypoints (vis != 0), the same after the optimal 2-D camera (eps 1e-6 I,
 *                       scale = trace(A^-1 x^T y) / 2, trans = mu2 / scale - mu1) and the fraction of aligned errors < 0.05 * img_size;
 *                       NaN when no keypoint or fewer than min_visible keypoints are visible.  The prediction is brought to pixels as
 *                       ((k + 1) * 0.5) * img_size in fp32 with one rounding per operation, like the reference's float32 numpy.
 *   JOINTS, JOINTS_PA   MPJPE after pelvis alignment (LSP hips 2 and 3) and after the similarity transform of the prediction onto the
 *                       ground truth (rotation with det +1, scale = trace(R K) / var1); computed for every frame (the reference keeps the
 *                       VIS3D frames); NaN without joints_gt.
 *   ACCEL               mean over the J joints of |p[f] - 2 p[f+1] + p[f+2]| for the prediction, NaN when f + 2 leaves the tube.
 *   ACCEL_ERROR         the same of (prediction - ground truth), NaN unless the whole triple lies in the tube and is VIS3D.
 *   VIS3D               1 when joints_gt is given and sum(kps_gt[f, :min(K,14), 2]) > min_visible, else 0.
 * Everything past the fp32 pixel scaling is fp64.  Inputs are fp32 rows at the given strides (in floats), so a [N,25,3] prediction's
 * first 14 joints are read in place.  A frame's row depends only on its tube; no atomics, bit-identical across launches and batchings.
 * hd_eval_mesh_tpose: mean vertex distance between the T-pose meshes of beta_gt and beta_pred per frame without running SMPL: at theta = 0
 * every joint transform is the identity, so verts = (sum_k w_vk) * v_shaped and the difference is (sum_k w_vk) * shapedirs_v * (beta_gt -
 * beta_pred); from c->dirs and c->lbs_w, fp64, one fixed-order mean per frame.  One launch.
 * hd_eval_verts_error: mean vertex distance per frame between meshes a [N, V, 3] and b at frame strides a_ld / b_ld floats (>= 3V),
 * fp64, fixed-order reduction.  One launch.
 * HD_ERR_INVALID (before any launch): a null pointer, N < 0, n_seq < 1, K outside [1, 32], J outside [4, 32], a row stride shorter than
 * its row, img_size <= 0, min_visible < 0, V <= 0. */
enum { HD_EVAL_KP = 0, HD_EVAL_KP_PA = 1, HD_EVAL_KP_PCK = 2, HD_EVAL_JOINTS = 3, HD_EVAL_JOINTS_PA = 4, HD_EVAL_ACCEL = 5,
       HD_EVAL_ACCEL_ERROR = 6, HD_EVAL_VIS3D = 7, HD_EVAL_COLS = 8 };
typedef struct {
  int N, n_seq;
  const int *seq_start;           /* device [n_seq + 1] */
  int K, J;                       /* keypoints (<= 32) and 3-D joints (4..32; 14 in the reference's evaluation) per frame */
  const float *kps_gt;            /* [N, K, 3] x, y, vis in pixels */
  long long kps_gt_ld;            /* >= 3K */
  const float *kps_pred;          /* [N, K, 2] in [-1, 1] */
  long long kps_pred_ld;          /* >= 2K */
  const float *joints_gt;         /* [N, J, 3] or NULL (dataset without 3-D) */
  long long joints_gt_ld;         /* >= 3J */
  const float *joints_pred;       /* [N, J, 3] */
  long long joints_pred_ld;       /* >= 3J */
  float img_size;
  int min_visible;
  double *out;                    /* [N, HD_EVAL_COLS] */
} hd_eval_frames_args;
int hd_eval_frames(const hd_eval_frames_args *a, void *stream);
int hd_eval_mesh_tpose(const hd_smpl_consts *c, const float *beta_gt, int beta_gt_ld, const float *beta_pred, int beta_pred_ld, int N,
                       double *out, void *stream);
int hd_eval_verts_error(const float *a, long long a_ld, const float *b, long long b_ld, int N, int V, double *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* HD_B200_H_ */
