// Device-side parameter block shared by the SIMT and wgmma implicit-GEMM kernels.
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"

namespace hd {

struct ConvParams {
  const float *in; long long in_ld;
  int n_img, H, W, Cin, Ho, Wo, KH, KW, stride, pad_t, pad_l;
  const float *w_kn; int Cout; int K; int M;
  const float *pre_scale, *pre_shift; int pre_img_stride, pre_relu;
  const float *post_scale, *post_shift; int post_relu;
  const float *res; long long res_ld; int res_H, res_W, res_stride;
  float *out; long long out_ld;
  int vec_out;   // out/res/post vectors allow float4 access
  int K_pad;     // tensor-core path: padded K of the packed weights
  const void *in_hi, *in_lo;      // pre-split fp16 activations (cp.async producer) or nullptr
  void *out_hi, *out_lo; long long out2_ld;
  const float *post2_scale, *post2_shift; int post2_relu;
  int out_sub;     // > 1: `out` is the dense [n, ceil(Ho/s), ceil(Wo/s), Cout] subsample, only rows with oy % s == 0 && ox % s == 0 are written
  int planes;      // A operand = padded RGBX fp16 planes of the resnet conv1 input (see conv_tc.cu producer)
  long long *dbg;  // optional: per-role cycle counters of CTA (0,0) (hd_conv_gemm_profile), else nullptr
};

#ifdef __CUDACC__
// (a0, a1) -> packed fp16 heads hi = RN_f16(a) and 2^11-scaled remainders lo = RN_f16((a - hi) * 2^11): the operand format of
// the fp16-split tensor-core path.  The value is first clamped to the finite fp16 range: an activation beyond +-65504 then
// saturates (hi = +-65504, lo = 0) instead of turning into inf / NaN that would spread through the trunk.
__device__ __forceinline__ void split_f16x2(float a0, float a1, uint32_t &hi, uint32_t &lo) {
  a0 = fminf(fmaxf(a0, -65504.f), 65504.f);
  a1 = fminf(fmaxf(a1, -65504.f), 65504.f);
  const __half2 h2 = __floats2half2_rn(a0, a1);
  const float2 f2 = __half22float2(h2);
  const __half2 l2 = __floats2half2_rn((a0 - f2.x) * 2048.0f, (a1 - f2.y) * 2048.0f);
  hi = *reinterpret_cast<const uint32_t *>(&h2);
  lo = *reinterpret_cast<const uint32_t *>(&l2);
}
#endif

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

inline int fill_params(const hd_conv_desc *d, ConvParams &p) {
  const bool heads = d && d->impl == HD_IMPL_TC_1XF16;    // pre-split operands are the fp16 heads alone
  if (!d || !(d->in || (d->in_hi && (d->in_lo || heads))) || !(d->out || (d->out_hi && (d->out_lo || heads)))) {
    set_last_error_text("hd_conv_gemm: null in/out");
    return HD_ERR_INVALID;
  }
  if (heads && (d->w_nk_lo || d->tmap_lo || d->tmap_lo_n64 || d->in_lo || d->out_lo)) {
    set_last_error_text("hd_conv_gemm: impl 4 (1xFP16) reads and writes heads only: w_nk_lo, tmap_lo, tmap_lo_n64, in_lo and out_lo must be NULL");
    return HD_ERR_INVALID;
  }
  if (d->n_img <= 0 || d->H <= 0 || d->W <= 0 || d->Cin <= 0 || d->Cout <= 0 || d->KH <= 0 || d->KW <= 0 ||
      d->stride <= 0 || d->Ho <= 0 || d->Wo <= 0 || (d->in_ld < d->Cin && !(d->flags & HD_CONV_INPUT_PLANES)) || (d->out && d->out_ld < d->Cout) || (d->out_hi && d->out2_ld < d->Cout)) {
    set_last_error_text("hd_conv_gemm: bad shape");
    return HD_ERR_INVALID;
  }
  if ((d->pre_scale == nullptr) != (d->pre_shift == nullptr)) {
    set_last_error_text("hd_conv_gemm: pre_scale and pre_shift must be given together");
    return HD_ERR_INVALID;
  }
  if (d->res && (d->res_ld < d->Cout || d->res_H <= 0 || d->res_W <= 0 || d->res_stride <= 0)) {
    set_last_error_text("hd_conv_gemm: bad residual geometry");
    return HD_ERR_INVALID;
  }
  p.in = d->in; p.in_ld = d->in_ld;
  p.n_img = d->n_img; p.H = d->H; p.W = d->W; p.Cin = d->Cin; p.Ho = d->Ho; p.Wo = d->Wo;
  p.KH = d->KH; p.KW = d->KW; p.stride = d->stride; p.pad_t = d->pad_t; p.pad_l = d->pad_l;
  p.w_kn = d->w_kn; p.Cout = d->Cout; p.K = d->KH * d->KW * d->Cin;
  const long long M = (long long)d->n_img * d->Ho * d->Wo;
  if (M > 0x7fffffffLL) { set_last_error_text("hd_conv_gemm: M overflows int32"); return HD_ERR_INVALID; }
  p.M = (int)M;
  p.pre_scale = d->pre_scale; p.pre_shift = d->pre_shift; p.pre_img_stride = d->pre_img_stride; p.pre_relu = d->pre_relu;
  p.post_scale = d->post_scale; p.post_shift = d->post_shift; p.post_relu = d->post_relu;
  p.res = d->res; p.res_ld = d->res_ld; p.res_H = d->res_H; p.res_W = d->res_W; p.res_stride = d->res_stride;
  p.out = d->out; p.out_ld = d->out_ld;
  p.in_hi = d->in_hi; p.in_lo = d->in_lo; p.out_hi = d->out_hi; p.out_lo = d->out_lo; p.out2_ld = d->out2_ld;
  p.post2_scale = d->post2_scale; p.post2_shift = d->post2_shift; p.post2_relu = d->post2_relu;
  p.vec_out = (d->Cout % 4 == 0) && (!d->out || ((d->out_ld % 4 == 0) && aligned16(d->out))) &&
              (!d->out_hi || ((d->out2_ld % 4 == 0) && aligned16(d->out_hi) && aligned16(d->out_lo))) &&
              (!d->res || ((d->res_ld % 4 == 0) && aligned16(d->res))) &&
              (!d->post_scale || aligned16(d->post_scale)) && (!d->post_shift || aligned16(d->post_shift));
  p.K_pad = d->K_pad;
  p.planes = (d->flags & HD_CONV_INPUT_PLANES) ? 1 : 0;
  p.out_sub = d->out_subsample > 1 ? d->out_subsample : 0;
  if (p.out_sub && !d->out) { set_last_error_text("hd_conv_gemm: out_subsample needs `out`"); return HD_ERR_INVALID; }
  p.dbg = nullptr;
  return HD_OK;
}

int launch_conv_simt(const ConvParams &p, cudaStream_t st);
int launch_conv_tc(const ConvParams &p, const hd_conv_desc *d, cudaStream_t st);

}  // namespace hd
