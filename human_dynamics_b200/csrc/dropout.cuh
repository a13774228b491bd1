// Dropout masks of the IEF heads (src/models.py:101-105, slim.dropout after the ReLU of fc1 and fc2), as a pure function of
// (seed, step, site, row, column): nothing is stored, so the forward kernels draw the mask where they write the activation and the
// mask is the same for any launch configuration, stream, split of the rows or order of the heads.  oracle/dropout_ref.py restates
// it in numpy, bit for bit.
//
//   element (n, j) of a [N, C] site, w = n*C + j:
//     word   = Philox4x32-10(counter = (w >> 2, site, step & 0xffffffff, step >> 32), key = (seed & 0xffffffff, seed >> 32))[w & 3]
//     u      = float((word & 0x7fffff) | 0x3f800000) - 1                  (TF's Uint32ToFloat: the low 23 bits)
//     keep   = floor(p + u) == 1, the sum rounded to fp32                  (TF 1.8 nn.dropout: binary = floor(keep_prob + uniform))
//     y      = (x / p) * keep                                             (nn.dropout: div(x, keep_prob) * binary, fp32)
// Generator: Philox4x32-10 with the Random123 / cuRAND multipliers and Weyl constants (TF's random_uniform uses the same one).
#pragma once
#include <cstdint>

namespace hd {

// One dropout site of one call: p = nn.dropout's fp32 keep_prob (p == 1: every element kept, y = x).
struct DropoutSite {
  unsigned long long seed, step;
  unsigned int site;
  float p;
};

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k.x += 0x9E3779B9u; k.y += 0xBB67AE85u; }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

// The four words of elements w = 4*g .. 4*g + 3 of a site.
__device__ __forceinline__ uint4 dropout_words(const DropoutSite &d, unsigned long long g) {
  return philox4x32_10(make_uint4((uint32_t)g, d.site, (uint32_t)d.step, (uint32_t)(d.step >> 32)),
                       make_uint2((uint32_t)d.seed, (uint32_t)(d.seed >> 32)));
}

__device__ __forceinline__ bool dropout_keep(uint32_t word, float p) {
  const float u = __fsub_rn(__uint_as_float((word & 0x7fffffu) | 0x3f800000u), 1.0f);
  return __fadd_rn(p, u) >= 1.0f;            // p + u < 2, so floor(p + u) is 1 exactly when the fp32 sum reaches 1
}

__device__ __forceinline__ float dropout_apply(float x, uint32_t word, float p) {
  return __fmul_rn(__fdiv_rn(x, p), dropout_keep(word, p) ? 1.0f : 0.0f);
}

// y[e] = dropout of x[e] for the 4 consecutive elements 4*g .. 4*g + 3.
__device__ __forceinline__ float4 dropout_apply4(const DropoutSite &d, unsigned long long g, float4 x) {
  const uint4 w = dropout_words(d, g);
  return make_float4(dropout_apply(x.x, w.x, d.p), dropout_apply(x.y, w.y, d.p), dropout_apply(x.z, w.z, d.p),
                     dropout_apply(x.w, w.w, d.p));
}

}  // namespace hd
