// wgmma implicit-GEMM convolution / FC for sm_90a with FP32-class accuracy via 3xTF32 / 3xFP16 error compensation.
//
//   D[128 x BN] (fp32)  =  sum over K chunks of   A_hi*B_hi  +  (A_lo*B_hi + A_hi*B_lo)
//
// SPLIT = false drops the bracket: one MMA per product on the heads alone (1xTF32, impl 2; 1xFP16, impl 4).  Nothing of a
// remainder is then loaded, stored or kept: no A_lo / B_lo tiles in a stage, no cross-term fragment, no pair remainder written.
//
// A (activations) never exists in HBM in im2col form.  For pre-split fp16 activations (every ResNet trunk layer, the SMPL
// blend GEMM) one producer warpgroup cp.asyncs the 128-row hi/lo pair of one K chunk straight into the 128-byte-swizzled
// K-major layout the wgmma shared-memory descriptor expects.  Otherwise eight producer warps gather the tile (zero padding,
// stride, per-channel BN/GN affine + ReLU prologue fused; up to three chunks of loads in flight per thread), split every
// value into its head `hi` (rounded to nearest: TF32 = low 13 mantissa bits clear, or fp16) and the remainder `lo`, and
// store both there.  B (weights, pre-split offline into hi/lo, K-major) arrives by TMA in 64-row boxes.  Two consumer
// warpgroups issue wgmma, each for 64 of the 128 rows.
//
// Accumulation precision: the tensor core does not round the fp32 accumulator to nearest on every MMA, so a long K
// summed in one accumulator drifts (relative error grows linearly with K).  Accumulation is therefore two-level: the
// dominant A_hi*B_hi term is summed by the tensor core for only PCH K-chunks, then added -- round-to-nearest, on the
// CUDA cores -- into per-thread fp32 running sums.  The two cross terms (2^-11 smaller) accumulate in their own
// register fragment for the whole tile.  Per consumer thread that is 3 x BN/2 fp32 registers.
//
// N tile: 128 for pre-split layers with Cout > 64 that give the SMs enough tiles (wide_n_tile), 64 otherwise.  The 128-wide
// tile needs 3 x 64 accumulator registers per consumer thread and halves the A gathers and the shared-memory reads per MMA
// of the 64-wide one.  Pre-split 1x1 layers with K <= 128 (SHORT) flush the running sums once per tile, so they need only the
// two fragments: 64-wide tiles, two CTAs per SM, one CTA's epilogue running under the other's loads and MMAs.  The root conv1 over
// the planes (Cout = 64) puts the channels on the wgmma's M side instead (CM, below): 64 channels x 256 pixels.
//
// Persistent: grid = min(#tiles, #SMs) (SHORT: 2 x #SMs); each CTA walks tiles blockIdx.x, +gridDim.x, ...  Barrier phases run
// continuously across tiles, and the producers keep prefetching the next tile's chunks while the consumers run the
// fused epilogue (scale/shift, residual, ReLU, fp32 output or its strided subsample, the next layer's fp16 pair)
// straight from the accumulator fragments.  RES (pre-split input, residual row-aligned with the output, K <= 512): each
// consumer warpgroup's 64 residual rows arrive by TMA in a shared-memory slot while the tile's main loop runs.  Pre-split
// layers stage their outputs in shared memory (the fp32 output over the residual slot) and write them with TMA stores; a staged
// pass runs column pair by column pair, the thread's two rows sharing each pair's epilogue vectors.
//
// Warp roles:
//   warps 0-7    two consumer warpgroups: wgmma issue, drains, epilogue (warpgroup g owns tile rows 64 g .. 64 g + 63)
//   warps 8-11   BN = 128 (384 threads): the cp.async A producers, 8 rows each; registers 256 x 232 + 128 x 40
//   warps 8-15   BN = 64 (512 threads): the A producers, 4 rows each; registers 256 x 152 + 256 x 104
//   warps 8-11   SHORT (384 threads, 2 CTAs per SM): the A producers, 8 rows each; registers 256 x 104 + 128 x 32
// Producer thread 0 also issues the chunk's B tile (TMA).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cstdlib>
#include "conv_common.cuh"
#include "tc_ptx.cuh"

namespace hd {
namespace {

constexpr int BM = 128;
constexpr int BOX_BYTES = 64 * 128;         // one 64-row weight box (hd_make_weight_tmap)
constexpr int W_PROD = 8;                   // first producer warp
// `stage` argument (pre-split layers): which outputs the epilogue stages in shared memory and writes by TMA (launch_tc)
constexpr int STAGE_OUT = 1, STAGE_PAIR = 2;

using namespace ptx;

// SHORT: pre-split layers with K <= PCH chunks (K <= 128), two CTAs per SM.  The running sums flush exactly once per tile, so the
// flushed fragment itself holds them; the CTA has one operand stage, and each warpgroup's residual slot doubles as its output
// staging.
//
// CM (channels on M, Cout = 64): the tile is 64 output channels x 256 pixels and computes the transpose, D^T = W^T A^T.  The
// weight box is the wgmma A operand (m64) and consumer warpgroup g's 128 pixel rows of the A tile its B operand (n128).  A 64-wide
// K chunk (SPLIT) then costs the shared-memory port 144 KB of wgmma reads and 80 KB of writes for twice the products of the 128 x 64
// tile's 96 + 48 KB (DESIGN.md 4.1).  Each output element gets the same products in the same K order as on the 128 x 64 tile.
template <bool SPLIT, bool HALF, bool ASPLIT, int BN, bool RES = false, bool SHORT = false, bool CM = false>
struct Cfg {
  static_assert(BN == 64 || (BN == 128 && HALF && ASPLIT), "128-wide N tiles: pre-split fp16 path only");
  static_assert(!RES || ASPLIT, "residual by TMA: pre-split fp16 path only");
  static_assert(!SHORT || (BN == 64 && HALF && ASPLIT), "two CTAs per SM: 64-wide pre-split fp16 tiles only");
  static_assert(!CM || (BN == 64 && HALF && ASPLIT && !RES && !SHORT), "channels on M: 64-channel pre-split fp16 tiles, no residual");
  static constexpr int CTAS = SHORT ? 2 : 1;                    // CTAs per SM (__launch_bounds__, persistent grid)
  static constexpr int TM = CM ? 256 : BM;                      // pixel rows of a tile (of the A tile in shared memory)
  static constexpr int A_BYTES = TM * 128;                      // A head tile: TM rows x one 128-byte swizzle row (32 tf32 or 64 fp16 of K)
  static constexpr int PROD_THREADS = BN == 128 || SHORT || CM ? 128 : 256;
  static constexpr int NUM_THREADS = 256 + PROD_THREADS;
  static constexpr int ROW_STEP = PROD_THREADS / 8;             // a producer thread's rows: rb + ROW_STEP * i
  static constexpr int ROWS = TM / ROW_STEP;
  static constexpr int PROD_REGS = SHORT ? 32 : CM ? 56 : BN == 128 ? 40 : 104, CONS_REGS = SHORT ? 104 : CM ? 224 : BN == 128 ? 232 : 152;
  // setmaxnreg only moves registers inside the CTA's launch allocation (65536 / CTAS / NUM_THREADS per thread, in steps of 8): a
  // split beyond it leaves the consumers' increase waiting forever
  static_assert(256 * CONS_REGS + PROD_THREADS * PROD_REGS <= NUM_THREADS * (65536 / (CTAS * NUM_THREADS) / 8 * 8),
                "setmaxnreg split beyond the CTA's registers");
  static constexpr int NACC = CM ? 64 : BN / 2;                 // fp32 registers of one m64nBN (CM: m64n128) fragment per thread
  // RES: the residual slots do not fit beside three 64 KB stages (BN = 128) or four 48 KB ones plus the output staging (BN = 64).
  // Residual layers have K <= 512 (<= 8 chunks).  CM: two 80 KB stages beside the 2 x 32 KB output staging.
  static constexpr int STAGES = SHORT ? 1 : CM ? 2 : BN == 128 ? (RES ? 2 : 3) : (RES ? 3 : 4);
  static constexpr int BKE = HALF ? 64 : 32;                    // K elements per chunk (one 128-byte row)
  static constexpr int B_TILE_BYTES = BN * 128;
  // a stage: the A head tile (+ its remainder), then the B head tile (+ its remainder).  !SPLIT keeps the stage counts of the split
  // kernels: the pipeline depth in chunks is the same, each chunk is half the bytes.
  static constexpr int B_OFFSET = (SPLIT ? 2 : 1) * A_BYTES;
  static constexpr int STAGE_BYTES = (SPLIT ? 2 : 1) * (A_BYTES + B_TILE_BYTES);
  static constexpr int RES_OFFSET = STAGES * STAGE_BYTES;
  // one warpgroup's 64 rows x BN fp32 residual (BN / 32 TMA boxes); SHORT: also the warpgroup's output staging
  static constexpr int RES_SLOT_BYTES = RES || SHORT ? 64 * BN * 4 : 0;
  static constexpr int STG_OFFSET = SHORT ? RES_OFFSET : RES_OFFSET + 2 * RES_SLOT_BYTES;
  // ASPLIT: one warpgroup's output staging, two 64-row x 128-byte TMA boxes (64 columns of fp32, or of the fp16 head and remainder);
  // CM: four, for the warpgroup's 128 pixel rows
  static constexpr int STG_BYTES = ASPLIT ? (CM ? 4 : 2) * BOX_BYTES : 0;
  static_assert(!SHORT || STG_BYTES == RES_SLOT_BYTES, "SHORT: the staging buffer is the residual slot");
  static constexpr int BAR_OFFSET = SHORT ? RES_OFFSET + 2 * RES_SLOT_BYTES : STG_OFFSET + 2 * STG_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFFSET + 128 + 1024;    // + alignment slack
  static_assert(SMEM_BYTES <= 232448, "dynamic shared memory beyond the 227 KB a CTA can opt into");
  static_assert(CTAS * (SMEM_BYTES + 1024) <= 233472, "CTAS CTAs (and the 1 KB each reserves) beyond an SM's 228 KB");
  static constexpr int PF = HALF ? 2 : 3;                       // producer prefetch ring depth (chunks in flight per thread)
  static constexpr int V = HALF ? 2 : 1;                        // float4 loads per row per chunk per thread
};

// The staged epilogue of a column pair: y = relu?(y * sc + sh (+ r, ADD_R)), each product and sum rounded on its own (__fmul_rn /
// __fadd_rn are never contracted), so every kernel that runs it gives the same bits.  sc / sh apply where their vector is given.
template <bool ADD_R = false>
__device__ __forceinline__ void epi2_rn(float &y0, float &y1, const float *has_sc, float2 sc, const float *has_sh, float2 sh,
                                        const float2 *r, int relu) {
  if (has_sc) { y0 = __fmul_rn(y0, sc.x); y1 = __fmul_rn(y1, sc.y); }
  if (has_sh) { y0 = __fadd_rn(y0, sh.x); y1 = __fadd_rn(y1, sh.y); }
  if (ADD_R) { const float2 v = *r; y0 = __fadd_rn(y0, v.x); y1 = __fadd_rn(y1, v.y); }
  if (relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
}

template <int R>
struct RowState {       // R output rows of one producer thread: image index and top-left input coordinate
  int n[R], iy[R], ix[R];
};

template <bool SPLIT, int PCH, bool HALF, bool GATHER, bool ASPLIT, int BN, bool RES, bool SHORT, bool CM>
__global__ void __launch_bounds__((Cfg<SPLIT, HALF, ASPLIT, BN, RES, SHORT, CM>::NUM_THREADS), (Cfg<SPLIT, HALF, ASPLIT, BN, RES, SHORT, CM>::CTAS))
conv_gemm_tc_kernel(const ConvParams p, const __grid_constant__ CUtensorMap tmap_hi, const __grid_constant__ CUtensorMap tmap_lo,
                    const __grid_constant__ CUtensorMap tmap_res, const __grid_constant__ CUtensorMap tmap_out,
                    const __grid_constant__ CUtensorMap tmap_out_hi, const __grid_constant__ CUtensorMap tmap_out_lo, const int stage) {
  using C = Cfg<SPLIT, HALF, ASPLIT, BN, RES, SHORT, CM>;
  // BN = 128, SHORT and CM keep the profile's start stamps and summed clocks in memory (hd_conv_gemm_profile): spill-free registers
  constexpr bool MEM_STAMPS = BN == 128 || SHORT || CM;
  constexpr int BKE = C::BKE, PF = C::PF, V = C::V, STAGES = C::STAGES, R = C::ROWS, RS = C::ROW_STEP, NA = C::NACC;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t *smem = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + C::BAR_OFFSET;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  auto res_bar = [&](int g) { return bar_base + 8u * (2 * STAGES + g); };   // RES: warpgroup g's residual slot has landed

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_k = (GATHER ? p.K_pad : p.K) / BKE;   // GATHER: ragged Cin (conv1: K=147 zero-padded to 192)
  const int tiles_n = (p.Cout + BN - 1) / BN;
  const int num_tiles = ((p.M + C::TM - 1) / C::TM) * tiles_n;
  const int my_tiles = (num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), ASPLIT ? C::PROD_THREADS + 1 : 9);   // 8 producer warps (ASPLIT: every producer thread, hardware arrive when its cp.asyncs land)
                                                  // + 1 arrive.expect_tx from the thread that issues the B load
      mbar_init(empty_bar(s), 8);    // one arrive per consumer warp once its wgmmas have read the stage
    }
    if (RES) for (int g = 0; g < 2; ++g) mbar_init(res_bar(g), 1);   // one arrive.expect_tx per tile
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= W_PROD) {
    // =============================== A producers (PROD_THREADS) ===============================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(C::PROD_REGS));
    const int t = threadIdx.x - W_PROD * 32;  // 0 .. PROD_THREADS - 1
    const int j = t & 7;                  // 16-byte chunk within the 128-byte K row
    const int rb = t >> 3;                // rows rb + RS*i, i < R (all with the same row & 7, so one swizzle offset)
    const uint32_t sw_off = (uint32_t)((j ^ (rb & 7)) << 4);
    const bool prof = p.dbg != nullptr && blockIdx.x == 0 && t == 0;
    long long t_wait = 0, t_start = prof && !MEM_STAMPS ? clock64() : 0;
    if (MEM_STAMPS && prof) { p.dbg[0] = clock64(); p.dbg[1] = 0; }   // start stamp in memory, replaced by the loop's length
    auto wait_empty = [&](int s, uint32_t ph) {     // MEM_STAMPS: the profile's wait clocks are summed in memory too
      if (MEM_STAMPS && prof) p.dbg[1] -= clock64();
      const long long tw0 = !MEM_STAMPS && prof ? clock64() : 0;
      mbar_wait(empty_bar(s), ph ^ 1u);
      if (!MEM_STAMPS && prof) t_wait += clock64() - tw0;
      if (MEM_STAMPS && prof) p.dbg[1] += clock64();
    };
    const int total = my_tiles * num_k;
    auto load_b = [&](int s, int ti, int kc) {      // producer thread 0: the chunk's B tile (weights, hi and lo) by TMA
      if (t != 0) return;
      const int n0 = (((int)blockIdx.x + ti * (int)gridDim.x) % tiles_n) * BN;
      const uint32_t b_hi = smem_base + s * C::STAGE_BYTES + C::B_OFFSET;
      // BN = 128: two 64-row boxes.  Weight rows are padded to 64, so the second box is either wholly inside the weights or
      // wholly past Cout; then it is not loaded, and the stale columns it would have filled only reach outputs c >= Cout,
      // which the epilogue never stores.
      const int boxes = (BN == 128 && n0 + 64 < p.Cout) ? 2 : 1;
      mbar_arrive_expect_tx(full_bar(s), (SPLIT ? 2 : 1) * boxes * BOX_BYTES);
      for (int b = 0; b < boxes; ++b) {
        tma_load_2d(b_hi + b * BOX_BYTES, &tmap_hi, full_bar(s), kc * BKE, n0 + 64 * b);
        if (SPLIT) tma_load_2d(b_hi + C::B_TILE_BYTES + b * BOX_BYTES, &tmap_lo, full_bar(s), kc * BKE, n0 + 64 * b);
      }
    };

    auto enter_tile = [&](int ti, RowState<R> &rs) {
      const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
      const int m0 = (tile / tiles_n) * C::TM;
      const int hw = p.Ho * p.Wo;
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const int m = m0 + rb + RS * i;
        if (m < p.M) {
          const int n = m / hw;
          const int r = m - n * hw;
          const int oy = r / p.Wo, ox = r - oy * p.Wo;
          rs.n[i] = n; rs.iy[i] = oy * p.stride - p.pad_t; rs.ix[i] = ox * p.stride - p.pad_l;
        } else {
          rs.n[i] = -1; rs.iy[i] = 0; rs.ix[i] = 0;
        }
      }
    };
    if constexpr (ASPLIT) {
      // ---- pre-split fp16 activations: cp.async straight into the swizzled tile, STAGES chunks in flight, no registers ----
      const __half *ihi = reinterpret_cast<const __half *>(p.in_hi);
      const __half *ilo = reinterpret_cast<const __half *>(p.in_lo);
      // SHORT: launch_conv_tc takes it for layers that meet the lean loop's conditions, and the other loops are not compiled
      if (SHORT || (!CM && !p.planes && p.KH * p.KW <= 32 && (long long)p.n_img * p.H * p.W * p.in_ld < (1ll << 31))) {
        // Lean loop (on the long-K layers these warps can pace the whole kernel: the general loop below spends instructions per
        // chunk on two integer divisions and 64-bit addressing).  Per tile: one 32-bit
        // element offset and one tap-validity bit mask per row.  Per chunk: (tap, channel) advance incrementally -- a 64-wide chunk
        // lies inside one tap because Cin % 64 == 0 -- and a row costs a shift, an add and two cp.asyncs.  Taken when the input's
        // element offsets fit 32 bits and the kernel window fits the 32-bit tap mask; anything else runs the general loop.
        const uint32_t off0 = (uint32_t)rb * 128u + sw_off;       // row rb + RS i of the tile: + i * RS * 128
        int base[R];
        uint32_t mask[R];
        int kc = 0, ti = 0, tap = 0, ci0 = 0, kx = 0, ky = 0, tap_off = 0;
        for (int q = 0; q < total; ++q) {
          if (kc == 0) {
            const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
            const int m0 = (tile / tiles_n) * C::TM + rb;
            const int hw = p.Ho * p.Wo;
#pragma unroll
            for (int i = 0; i < R; ++i) {
              const int m = m0 + RS * i;
              uint32_t mk = 0;
              int b = 0;
              if (m < p.M) {
                const int n = m / hw;
                const int r = m - n * hw;
                const int oy = r / p.Wo, ox = r - oy * p.Wo;
                const int iy0 = oy * p.stride - p.pad_t, ix0 = ox * p.stride - p.pad_l;
                b = ((n * p.H + iy0) * p.W + ix0) * p.in_ld + j * 8;
                int t = 0;
                for (int yy = 0; yy < p.KH; ++yy)
                  for (int xx = 0; xx < p.KW; ++xx, ++t)
                    if ((unsigned)(iy0 + yy) < (unsigned)p.H && (unsigned)(ix0 + xx) < (unsigned)p.W) mk |= 1u << t;
              }
              base[i] = SHORT && !(mk & 1u) ? -1 : b;        // SHORT (1x1 windows): the row's one tap bit is the sign of its offset
              mask[i] = mk;
            }
            tap = 0; ci0 = 0; kx = 0; ky = 0; tap_off = 0;
          }
          const int s = q % STAGES;
          const uint32_t ph = (uint32_t)(q / STAGES) & 1u;
          wait_empty(s, ph);
          load_b(s, ti, kc);
          const uint32_t a_hi = smem_base + s * C::STAGE_BYTES + off0;
          const int eo = SHORT ? ci0 : tap_off + ci0;
#pragma unroll
          for (int i = 0; i < R; ++i) {
            const bool ok = SHORT ? base[i] >= 0 : (mask[i] >> tap) & 1u;
            const int e = ok ? base[i] + eo : 0;
            cp_async16(a_hi + i * RS * 128, ihi + e, ok ? 16u : 0u);
            if (SPLIT) cp_async16(a_hi + C::A_BYTES + i * RS * 128, ilo + e, ok ? 16u : 0u);
          }
          asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(full_bar(s)) : "memory");
          ci0 += BKE;
          if (ci0 == p.Cin) {
            ci0 = 0; ++tap;
            if (++kx == p.KW) { kx = 0; ++ky; }
            tap_off = (ky * p.W + kx) * p.in_ld;
          }
          if (++kc == num_k) { kc = 0; ++ti; }
        }
      } else if (!SHORT && p.planes && (long long)p.n_img * p.H * p.W * p.in_ld < (1ll << 31)) {
        // resnet conv1 over the padded RGBX fp16 planes, same lean scheme: Cin = 32 halves = one kernel row of 7(+1) pixels x 4, so a
        // 64-wide chunk holds TWO kernel rows (taps 2 kc and 2 kc + 1); this thread's 16-byte piece is pixels 2*(j&3), 2*(j&3)+1 of row
        // 2 kc + (j >> 2).  KH = 8: row 7 is a phantom (zero weights) and is zero-filled.  No padding tests: the planes are pre-padded.
        const uint32_t off0 = (uint32_t)rb * 128u + sw_off;
        const int jt = j >> 2;
        const int row_step = 2 * p.W * (int)p.in_ld;                // two kernel rows per chunk
        int base[R];
        int kc = 0, ti = 0;
        for (int q = 0; q < total; ++q) {
          if (kc == 0) {
            const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
            const int m0 = (tile / tiles_n) * C::TM + rb;
            const int hw = p.Ho * p.Wo;
#pragma unroll
            for (int i = 0; i < R; ++i) {
              const int m = m0 + RS * i;
              int b = -1;
              if (m < p.M) {
                const int n = m / hw;
                const int r = m - n * hw;
                const int oy = r / p.Wo, ox = r - oy * p.Wo;
                b = ((n * p.H + oy * p.stride + jt) * p.W + ox * p.stride) * (int)p.in_ld + (j & 3) * 8;
              }
              base[i] = b;
            }
          }
          const int s = q % STAGES;
          const uint32_t ph = (uint32_t)(q / STAGES) & 1u;
          wait_empty(s, ph);
          load_b(s, ti, kc);
          const uint32_t a_hi = smem_base + s * C::STAGE_BYTES + off0;
          const bool tap_ok = 2 * kc + jt < 7;
          const int eo = kc * row_step;
#pragma unroll
          for (int i = 0; i < R; ++i) {
            const bool ok = tap_ok && base[i] >= 0;
            const int e = ok ? base[i] + eo : 0;
            // neighbouring output pixels read overlapping 64-byte windows (each 16-byte piece 4x): keep them in L1
            cp_async16_ca(a_hi + i * RS * 128, ihi + e, ok ? 16u : 0u);
            if (SPLIT) cp_async16_ca(a_hi + C::A_BYTES + i * RS * 128, ilo + e, ok ? 16u : 0u);
          }
          asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(full_bar(s)) : "memory");
          if (++kc == num_k) { kc = 0; ++ti; }
        }
      } else if (!SHORT && !CM) {     // CM: launch_conv_f16 takes it only for layers the lean plane loop runs
      RowState<R> rs;
      int kc = 0, ti = 0;
      for (int q = 0; q < total; ++q) {
        if (kc == 0) enter_tile(ti, rs);
        const int s = q % STAGES;
        const uint32_t ph = (uint32_t)(q / STAGES) & 1u;
        wait_empty(s, ph);
        load_b(s, ti, kc);
        const int kb = kc * BKE;
        // planes (resnet conv1 over the padded RGBX fp16 planes, Cin = 32 halves = one kernel row of 7(+1) pixels x 4): a 64-wide
        // chunk holds TWO kernel rows; this thread's 16-byte piece is pixels 2*(j&3), 2*(j&3)+1 of row ky.  KH = 8: row 7 is a
        // phantom (zero weights) and is zero-filled.
        const int tap = p.planes ? 2 * kc + (j >> 2) : kb / p.Cin;
        const int ci = p.planes ? (j & 3) * 8 : kb - tap * p.Cin + j * 8;
        const int ky = tap / p.KW, kx = tap - ky * p.KW;
        const bool tap_ok = !p.planes || tap < 7;
        const uint32_t a_hi = smem_base + s * C::STAGE_BYTES, a_lo = a_hi + C::A_BYTES;
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int iy = rs.iy[i] + ky, ix = rs.ix[i] + kx;
          const bool ok = tap_ok && rs.n[i] >= 0 && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
          const size_t e = ok ? ((size_t)((size_t)rs.n[i] * p.H + iy) * p.W + ix) * p.in_ld + ci : 0;
          const uint32_t off = (uint32_t)(rb + RS * i) * 128u + sw_off;
          if (p.planes) {        // conv1: neighbouring output pixels read overlapping 64-byte windows (each 16-byte piece 4x): keep them in L1
            cp_async16_ca(a_hi + off, ihi + e, ok ? 16u : 0u);
            if (SPLIT) cp_async16_ca(a_lo + off, ilo + e, ok ? 16u : 0u);
          } else {
            cp_async16(a_hi + off, ihi + e, ok ? 16u : 0u);
            if (SPLIT) cp_async16(a_lo + off, ilo + e, ok ? 16u : 0u);
          }
        }
        // the barrier itself is told to arrive (without a pending-count increment) once this thread's copies have landed:
        // chunks are published the moment their data is in smem, with no producer thread in the loop, so up to STAGES
        // chunks are genuinely in flight.  The MMA thread issues the generic->async proxy fence after its wait.
        asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(full_bar(s)) : "memory");
        if (++kc == num_k) { kc = 0; ++ti; }
      }
      }
      cp_async_commit();
      cp_async_wait<0>();
      if (prof) { p.dbg[0] = clock64() - (MEM_STAMPS ? p.dbg[0] : t_start); if (!MEM_STAMPS) p.dbg[1] = t_wait; }
    } else {
    RowState<R> pf_rs, st_rs;              // prefetch-side and store-side row state (may be one tile apart)
    float4 ring[PF][4 * V];
    uint32_t vmask[PF];
    int pf_kc = 0, pf_ti = 0;              // next chunk to prefetch
    auto prefetch = [&](float4 *dst, uint32_t &vm) {
      if (pf_kc == 0) enter_tile(pf_ti, pf_rs);
      if (GATHER) {
        // Ragged Cin (conv1, 7x7x3): K is laid out ky-major with each kernel row's KW*Cin contiguous input floats padded to a
        // multiple of 8 (21 -> 24), so a thread's 8 consecutive k belong to ONE kernel row and are 8 consecutive floats in
        // memory: one address per (row, chunk), element-wise bounds only for the left/right image edge.
        const int seg = p.KW * p.Cin, segp = (seg + 7) & ~7;
        const int g8 = (pf_kc * BKE + j * (4 * V)) / 8;          // 8-float group index along the padded K
        const int gpr = segp >> 3;                               // groups per kernel row
        const int ky = g8 / gpr, r0 = (g8 - ky * gpr) * 8;
        vm = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int iy = pf_rs.iy[i] + ky;
          const bool okr = pf_rs.n[i] >= 0 && ky < p.KH && iy >= 0 && iy < p.H;
          const int c0 = pf_rs.ix[i] * p.Cin + r0;               // float offset inside the input row (may be < 0 at the left edge)
          const float *src = p.in + ((size_t)((size_t)(okr ? pf_rs.n[i] : 0) * p.H + (okr ? iy : 0)) * p.W) * p.in_ld + c0;
          const int rowlen = p.W * p.Cin;
          float xs[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const bool ok = okr && (r0 + e) < seg && (c0 + e) >= 0 && (c0 + e) < rowlen;
            xs[e] = ok ? __ldg(src + e) : 0.f;
          }
          dst[i * V] = make_float4(xs[0], xs[1], xs[2], xs[3]);
          dst[i * V + V - 1] = make_float4(xs[4], xs[5], xs[6], xs[7]);
          if (pf_rs.n[i] >= 0) vm |= 1u << i;
        }
        if (++pf_kc == num_k) { pf_kc = 0; ++pf_ti; }
        return;
      }
      const int kb = pf_kc * BKE;
      const int tap = kb / p.Cin, ci = kb - tap * p.Cin + j * (4 * V);
      const int ky = tap / p.KW, kx = tap - ky * p.KW;
      vm = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int iy = pf_rs.iy[i] + ky, ix = pf_rs.ix[i] + kx;
        const bool ok = pf_rs.n[i] >= 0 && (unsigned)iy < (unsigned)p.H && (unsigned)ix < (unsigned)p.W;
        if (ok) {
          const float4 *src = reinterpret_cast<const float4 *>(p.in + ((size_t)((size_t)pf_rs.n[i] * p.H + iy) * p.W + ix) * p.in_ld + ci);
#pragma unroll
          for (int v = 0; v < V; ++v) dst[i * V + v] = __ldg(src + v);
          vm |= 1u << i;
        } else {
#pragma unroll
          for (int v = 0; v < V; ++v) dst[i * V + v] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      if (++pf_kc == num_k) { pf_kc = 0; ++pf_ti; }
    };
    int st_kc = 0, st_ti = 0;
    auto consume = [&](int q, float4 *cur, uint32_t vm) {
      if (st_kc == 0) enter_tile(st_ti, st_rs);
      const int s = q % STAGES;
      const uint32_t ph = (uint32_t)(q / STAGES) & 1u;
      long long tw0 = prof ? clock64() : 0;
      mbar_wait(empty_bar(s), ph ^ 1u);
      if (prof) t_wait += clock64() - tw0;
      load_b(s, st_ti, st_kc);
      uint8_t *a_hi = smem + s * C::STAGE_BYTES;
      uint8_t *a_lo = a_hi + C::A_BYTES;
      const int pci = p.pre_scale ? (st_kc * BKE) % p.Cin + j * (4 * V) : 0;
      // row by row (keeps the live set small): prologue affine (+ReLU) on real pixels only, then split every value into a
      // head and a remainder that the tensor core reads exactly (zero-mean rounding):
      //   TF32: hi = RN_tf32(x), lo = RN_tf32(x - hi);   FP16: hi = RN_f16(x), lo = RN_f16((x - hi) * 2^11)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float xs[4 * V];
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const float4 x = cur[i * V + v];
          xs[4 * v] = x.x; xs[4 * v + 1] = x.y; xs[4 * v + 2] = x.z; xs[4 * v + 3] = x.w;
        }
        if (p.pre_scale && (vm & (1u << i))) {
          const size_t po = (size_t)(p.pre_img_stride != 0 ? st_rs.n[i] : 0) * p.pre_img_stride + pci;
#pragma unroll
          for (int v = 0; v < V; ++v) {
            const float4 sc = __ldg(reinterpret_cast<const float4 *>(p.pre_scale + po) + v);
            const float4 sh = __ldg(reinterpret_cast<const float4 *>(p.pre_shift + po) + v);
            xs[4 * v] = xs[4 * v] * sc.x + sh.x; xs[4 * v + 1] = xs[4 * v + 1] * sc.y + sh.y;
            xs[4 * v + 2] = xs[4 * v + 2] * sc.z + sh.z; xs[4 * v + 3] = xs[4 * v + 3] * sc.w + sh.w;
          }
          if (p.pre_relu) {
#pragma unroll
            for (int e = 0; e < 4 * V; ++e) xs[e] = fmaxf(xs[e], 0.f);
          }
        }
        uint32_t h[4], l[4];
        if (!HALF) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float hf = rn_tf32(xs[e]);
            h[e] = __float_as_uint(hf);
            l[e] = __float_as_uint(rn_tf32(xs[e] - hf));
          }
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) split_f16x2(xs[2 * e], xs[2 * e + 1], h[e], l[e]);
        }
        const uint32_t off = (uint32_t)(rb + 32 * i) * 128u + sw_off;
        *reinterpret_cast<uint4 *>(a_hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
        if (SPLIT) *reinterpret_cast<uint4 *>(a_lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the UMMA (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(full_bar(s));
      if (++st_kc == num_k) { st_kc = 0; ++st_ti; }
    };
    // prime the ring with PF-1 chunks, then: issue chunk q+PF-1, consume chunk q
#pragma unroll
    for (int u = 0; u < PF - 1; ++u)
      if (u < total) prefetch(ring[u], vmask[u]);
    for (int q0 = 0; q0 < total; q0 += PF) {
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        const int q = q0 + u;
        if (q < total) {
          if (q + PF - 1 < total) prefetch(ring[(u + PF - 1) % PF], vmask[(u + PF - 1) % PF]);
          consume(q, ring[u], vmask[u]);
        }
      }
    }
    if (prof) { p.dbg[0] = clock64() - t_start; p.dbg[1] = t_wait; }
    }   // !ASPLIT
  } else if (warp < W_PROD) {
    // =============================== consumers: wgmma, drains, epilogue ===============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(C::CONS_REGS));
    const int wg = warp >> 2;                             // rows 64 wg .. 64 wg + 63 of the tile
    const bool prof = p.dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
    long long t_wait = 0, t_start = prof && !MEM_STAMPS && !RES ? clock64() : 0;
    if ((RES || MEM_STAMPS) && prof) p.dbg[2] = clock64();    // start stamp in memory (keeps the BN = 128 and SHORT consumers spill-free)
    if (prof) { p.dbg[3] = 0; p.dbg[4] = 0; p.dbg[5] = 0; p.dbg[6] = 0; }   // epilogue clocks and their split, summed in memory for the same reason
    const int hw = p.Ho * p.Wo;
    const int frow = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's fragment rows: frow, frow + 8
    const int fcol = 2 * (lane & 3);                            // and columns 8 j + fcol, + 1
    // SHORT: the single flush per tile is done in place, so the running sums are acc itself and take no registers of their own
    // !SPLIT: no cross terms, so no accx fragment
    float acc[NA], accx[SPLIT ? NA : 1], sums_[SHORT ? 1 : NA];
    float *const sums = SHORT ? acc : sums_;
#pragma unroll
    for (int i = 0; i < NA; ++i) {
      acc[i] = 0.f;
      if constexpr (SPLIT) accx[i] = 0.f;
    }
    // RES: the warpgroup's 64 residual rows of a tile arrive by TMA in 32-column boxes (128-byte swizzle: row r at r * 128 B, its
    // 16-byte piece k at (k ^ (r & 7)) * 16), issued by the warpgroup's first thread as soon as the previous tile's epilogue has read
    // the slot, so the load overlaps the tile's main loop.  Boxes wholly past M or Cout are not loaded (their values are never read);
    // partial ones are zero-filled by TMA and count their full bytes.
    uint8_t *res_sm = smem + C::RES_OFFSET + wg * C::RES_SLOT_BYTES;
    const bool res_issuer = RES && (threadIdx.x & 127) == 0;
    // ASPLIT: the same thread issues the warpgroup's output stores (bulk async-groups belong to the thread that commits them)
    const bool stg_issuer = ASPLIT && (threadIdx.x & 127) == 0;
    auto load_res = [&](int ti) {
      const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
      const int r0 = (tile / tiles_n) * BM + 64 * wg, c0 = (tile % tiles_n) * BN;
      const int cols = p.Cout - c0 < BN ? p.Cout - c0 : BN;
      const int boxes = r0 < p.M ? (cols + 31) / 32 : 0;
      const uint32_t slot = smem_base + C::RES_OFFSET + wg * C::RES_SLOT_BYTES;
      mbar_arrive_expect_tx(res_bar(wg), boxes * (64 * 128));
      for (int b = 0; b < boxes; ++b) tma_load_2d(slot + b * (64 * 128), &tmap_res, res_bar(wg), c0 + 32 * b, r0);
    };
    if (res_issuer && my_tiles > 0) load_res(0);
    int q = 0;
    for (int ti = 0; ti < my_tiles; ++ti) {
      if (!SHORT) {
#pragma unroll
        for (int i = 0; i < NA; ++i) sums[i] = 0.f;
      }
      for (int kc = 0; kc < num_k; ++kc, ++q) {
        const int s = q % STAGES;
        const uint32_t ph = (uint32_t)(q / STAGES) & 1u;
        const bool group_start = (kc % PCH) == 0;
        if (MEM_STAMPS && prof) p.dbg[3] -= clock64();    // summed in memory, like the epilogue's clocks
        const long long tw0 = !MEM_STAMPS && prof ? clock64() : 0;
        mbar_wait(full_bar(s), ph);
        if (!MEM_STAMPS && prof) t_wait += clock64() - tw0;
        if (MEM_STAMPS && prof) p.dbg[3] += clock64();
        if (ASPLIT) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // cp.async (generic proxy) data -> wgmma (async proxy)
        const uint32_t a_hi = smem_base + s * C::STAGE_BYTES + wg * (C::TM / 2 * 128);   // the warpgroup's half of the A tile's rows
        const uint32_t a_lo = a_hi + C::A_BYTES;
        const uint32_t b_hi = smem_base + s * C::STAGE_BYTES + C::B_OFFSET;
        const uint32_t b_lo = b_hi + C::B_TILE_BYTES;
        const uint64_t da_hi = make_smem_desc(a_hi), da_lo = make_smem_desc(a_lo);
        const uint64_t db_hi = make_smem_desc(b_hi), db_lo = make_smem_desc(b_lo);
        fence_regs(acc);
        if constexpr (SPLIT) fence_regs(accx);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {                // K = 8 tf32 / 16 fp16 = 32 bytes per wgmma: advance inside the swizzle row
          const uint64_t adv = (uint64_t)((k * 32) >> 4);
          if constexpr (CM) {                         // the transposed products: weights (A) x the warpgroup's 128 pixels (B)
            if constexpr (SPLIT) {
              wgmma_m64n128k16_f16(accx, db_hi + adv, da_lo + adv, (kc | k) != 0);
              wgmma_m64n128k16_f16(accx, db_lo + adv, da_hi + adv, 1u);
            }
            wgmma_m64n128k16_f16(acc, db_hi + adv, da_hi + adv, !(group_start && k == 0));
          } else if constexpr (BN == 128) {
            if constexpr (SPLIT) {
              wgmma_m64n128k16_f16(accx, da_lo + adv, db_hi + adv, (kc | k) != 0);
              wgmma_m64n128k16_f16(accx, da_hi + adv, db_lo + adv, 1u);
            }
            wgmma_m64n128k16_f16(acc, da_hi + adv, db_hi + adv, !(group_start && k == 0));
          } else if constexpr (HALF) {
            if constexpr (SPLIT) {
              wgmma_m64n64k16_f16(accx, da_lo + adv, db_hi + adv, (kc | k) != 0);
              wgmma_m64n64k16_f16(accx, da_hi + adv, db_lo + adv, 1u);
            }
            wgmma_m64n64k16_f16(acc, da_hi + adv, db_hi + adv, !(group_start && k == 0));
          } else {
            if constexpr (SPLIT) {
              wgmma_m64n64k8_tf32(accx, da_lo + adv, db_hi + adv, (kc | k) != 0);
              wgmma_m64n64k8_tf32(accx, da_hi + adv, db_lo + adv, 1u);
            }
            wgmma_m64n64k8_tf32(acc, da_hi + adv, db_hi + adv, !(group_start && k == 0));
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(acc);
        if constexpr (SPLIT) fence_regs(accx);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(s));       // this warp's share of the stage has been read
        if (!SHORT && ((kc % PCH) == PCH - 1 || kc == num_k - 1)) {
#pragma unroll
          for (int i = 0; i < NA; ++i) sums[i] += acc[i];      // round-to-nearest fp32 adds
        }
      }
      if (SHORT) {                                       // the one flush: 0 + acc, as above (a -0 becomes +0)
#pragma unroll
        for (int i = 0; i < NA; ++i) acc[i] = __fadd_rn(0.f, acc[i]);
      }
      if constexpr (SPLIT) {
#pragma unroll
        for (int i = 0; i < NA; ++i) sums[i] += accx[i] * (HALF ? (1.0f / 2048.0f) : 1.0f);
      }
      if (prof) p.dbg[4] -= clock64();                   // the epilogue's clocks, summed in memory (see above)
      const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
      const int m0 = (tile / tiles_n) * C::TM, n0 = (tile % tiles_n) * BN;
      if (RES && prof) p.dbg[5] -= clock64();            // of the epilogue: waiting for the residual
      if (RES) mbar_wait(res_bar(wg), (uint32_t)ti & 1u);
      if (RES && prof) p.dbg[5] += clock64();
      // Epilogue from the fragments, per row and pair of adjacent columns c, c + 1 (the four threads of a quad cover 8 contiguous
      // columns of a row): v = acc * scale + shift (+ residual) (ReLU) -> fp32 output (or its strided subsample), and the next
      // layer's pre-activation relu?(v * s2 + b2) as an fp16 head / remainder pair.
      auto row_geom = [&](int m, int &n_img, int &oy, int &ox) {
        n_img = 0; oy = 0; ox = 0;
        if (p.out_sub || (!RES && p.res && !(p.res_stride == 1 && p.res_H == p.Ho && p.res_W == p.Wo))) {
          n_img = m / hw;
          const int r = m - n_img * hw;
          oy = r / p.Wo; ox = r - oy * p.Wo;
        }
      };
      auto res_row = [&](int m, int n_img, int oy, int ox) -> const float * {     // residual read from global memory (!RES)
        if (RES || !p.res) return nullptr;
        const size_t rr = (p.res_stride == 1 && p.res_H == p.Ho && p.res_W == p.Wo)
                              ? (size_t)m
                              : ((size_t)n_img * p.res_H + (size_t)oy * p.res_stride) * p.res_W + (size_t)ox * p.res_stride;
        return p.res + rr * p.res_ld;
      };
      auto out_row = [&](int m, int n_img, int oy, int ox) -> float * {
        if (!p.out) return nullptr;
        if (!p.out_sub) return p.out + (size_t)m * p.out_ld;
        if (oy % p.out_sub != 0 || ox % p.out_sub != 0) return nullptr;
        const int Hs = (p.Ho + p.out_sub - 1) / p.out_sub, Ws = (p.Wo + p.out_sub - 1) / p.out_sub;
        return p.out + ((size_t)((size_t)n_img * Hs + oy / p.out_sub) * Ws + ox / p.out_sub) * p.out_ld;
      };
      // vec_out (Cout % 4 == 0, 16-byte aligned rows and vectors: pairs are 8-byte aligned).  RES: rs is the residual pair in the slot.
      auto value2 = [&](int c, const float2 *rs, const float *rrow, float &y0, float &y1) {
        if (p.post_scale) { const float2 sc = __ldg(reinterpret_cast<const float2 *>(p.post_scale + c)); y0 *= sc.x; y1 *= sc.y; }
        if (p.post_shift) { const float2 sh = __ldg(reinterpret_cast<const float2 *>(p.post_shift + c)); y0 += sh.x; y1 += sh.y; }
        if (RES) { const float2 r = *rs; y0 += r.x; y1 += r.y; }
        else if (rrow) { const float2 r = *reinterpret_cast<const float2 *>(rrow + c); y0 += r.x; y1 += r.y; }
        if (p.post_relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
      };
      // the next layer's A operand: second affine (+ReLU) = its pre-activation, split into fp16 head/remainder
      auto pair2 = [&](int c, float a0, float a1, uint32_t &hh, uint32_t &ll) {
        if (p.post2_scale) { const float2 sc = __ldg(reinterpret_cast<const float2 *>(p.post2_scale + c)); a0 *= sc.x; a1 *= sc.y; }
        if (p.post2_shift) { const float2 sh = __ldg(reinterpret_cast<const float2 *>(p.post2_shift + c)); a0 += sh.x; a1 += sh.y; }
        if (p.post2_relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
        split_f16x2(a0, a1, hh, ll);
      };
      if constexpr (CM) {
        // Channels on M: this thread holds channels ch + 8 h of the warpgroup's pixels 8 j + fcol (+ 1), j < 16.  Transposed on
        // the way in, v goes into the staging buffer as 2 x 2 TMA boxes of 64 pixel rows x 32 fp32 channels (row r at r * 128 B,
        // its 16-byte piece k at (k ^ (r & 7)) * 16; a thread's pixels all have r & 7 = fcol + e), and leaves by TMA stores.  Every
        // product and sum is rounded on its own, as on the 128 x 64 tile.  The root conv1 writes the fp32 output alone
        // (launch_conv_f16 takes this tile for nothing else).
        const bool st32 = (stage & STAGE_OUT) != 0;
        uint8_t *stg = smem + C::STG_OFFSET + wg * C::STG_BYTES;
        const uint32_t stg_a = smem_base + C::STG_OFFSET + wg * C::STG_BYTES;
        const int r0 = m0 + 128 * wg;
        const int ch = (warp & 3) * 16 + (lane >> 2);
        auto acquire = [&]() {   // the staging buffer may be rewritten: its last stores have been read
          if (prof) p.dbg[6] -= clock64();
          if (stg_issuer) bulk_wait_read<0>();
          named_bar_sync(3 + wg, 128);
          if (prof) p.dbg[6] += clock64();
        };
        if (st32) {
          acquire();
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int c = ch + 8 * h;
            const float sc = p.post_scale ? __ldg(p.post_scale + c) : 0.f, sh = p.post_shift ? __ldg(p.post_shift + c) : 0.f;
            uint8_t *cb = stg + (c >> 5) * BOX_BYTES + (c & 3) * 4;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int r = 8 * (j & 7) + fcol + e;          // row of box 2 (j >> 3) + (c >> 5)
                float y = sums[4 * j + 2 * h + e];
                if (p.post_scale) y = __fmul_rn(y, sc);
                if (p.post_shift) y = __fadd_rn(y, sh);
                if (p.post_relu) y = fmaxf(y, 0.f);
                *reinterpret_cast<float *>(cb + (j >> 3) * 2 * BOX_BYTES + r * 128 + ((((c & 31) >> 2) ^ (fcol + e)) << 4)) = y;
                sums[4 * j + 2 * h + e] = y;
              }
            }
          }
          fence_proxy_async();
          named_bar_sync(3 + wg, 128);
          if (stg_issuer) {
#pragma unroll
            for (int b = 0; b < 4; ++b)
              if (r0 + 64 * (b >> 1) < p.M) tma_store_2d(&tmap_out, stg_a + b * BOX_BYTES, 32 * (b & 1), r0 + 64 * (b >> 1));
            bulk_commit();
          }
        }
      } else if constexpr (ASPLIT) {
        // Staged: per 64-column pass, (1) v; the fp32 output goes into 32-column x 64-row boxes in the TMA box layout (row r at
        // r * 128 B, its 16-byte piece k at (k ^ (r & 7)) * 16), over the residual pair just read (RES) or in the staging
        // buffer, and v replaces the sums; (2) the pair from v into the staging buffer (head box, remainder box: 64 fp16
        // columns each).  A filled buffer is published (proxy fence, warpgroup barrier), and the warpgroup's first thread
        // writes it with TMA bulk-tensor stores, which clip rows >= M and columns >= Cout, and goes on without waiting; it
        // waits for their reads only before the buffer is filled again.  The strided subsample and a pair pitch that is not a
        // multiple of 16 bytes are stored from registers.
        const bool st32 = (stage & STAGE_OUT) != 0, st2 = (stage & STAGE_PAIR) != 0;
        uint8_t *stg = smem + C::STG_OFFSET + wg * C::STG_BYTES;
        const uint32_t stg_a = smem_base + C::STG_OFFSET + wg * C::STG_BYTES;
        const int r0 = m0 + 64 * wg;
        const uint32_t rsw = (uint32_t)(lane >> 2);            // the swizzle of this thread's rows: (frow + 8 h) & 7
        auto acquire = [&](bool after_out) {   // the staging buffer may be rewritten: its last stores have been read
          if (prof) p.dbg[6] -= clock64();                     // of the epilogue: waiting for stores to be read
          if (stg_issuer) {
            if (after_out) bulk_wait_read<1>();                // RES: the fp32 stores just issued read the slot, not the buffer
            else bulk_wait_read<0>();
          }
          named_bar_sync(3 + wg, 128);
          if (prof) p.dbg[6] += clock64();
        };
#pragma unroll
        for (int cc = 0; cc < BN / 64; ++cc) {
          const int c0 = n0 + 64 * cc;
          const bool issue = stg_issuer && r0 < p.M && c0 < p.Cout;
          if (st32 && !RES) acquire(false);
          // A thread's two rows (frow, frow + 8) have the same columns.  Where everything is staged and no residual comes from global
          // memory (every trunk layer but the strided subsamples) the pass goes column pair by column pair: the epilogue vectors of a
          // pair are read once for both rows, from one base pointer per vector, and nothing per row is kept but its validity.  Each
          // product and sum is rounded on its own (__fmul_rn / __fadd_rn are never contracted), as in the row-by-row loops.
          const bool rok[2] = {m0 + frow < p.M, m0 + frow + 8 < p.M};
          if (!RES && !st32 && st2 && !p.out && !p.res) {
            // The pair alone, no residual (every unit's conv1 and conv2): v and the pair in one pass, the four epilogue vectors of a
            // column pair read once for both rows, v kept in registers.  The arithmetic is that of the row-by-row pass and the pair
            // pass below, each product and sum rounded on its own.
            acquire(false);
            uint8_t *brow = stg + (frow - 64 * wg) * 128 + 4 * (lane & 3);
            const float *vsc = p.post_scale ? p.post_scale + c0 + fcol : nullptr, *vsh = p.post_shift ? p.post_shift + c0 + fcol : nullptr;
            const float *v2sc = p.post2_scale ? p.post2_scale + c0 + fcol : nullptr, *v2sh = p.post2_shift ? p.post2_shift + c0 + fcol : nullptr;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * cc + jj;
              if (c0 + 8 * jj + fcol >= p.Cout) continue;
              const float2 sc = vsc ? __ldg(reinterpret_cast<const float2 *>(vsc + 8 * jj)) : make_float2(0.f, 0.f);
              const float2 sh = vsh ? __ldg(reinterpret_cast<const float2 *>(vsh + 8 * jj)) : make_float2(0.f, 0.f);
              const float2 sc2 = v2sc ? __ldg(reinterpret_cast<const float2 *>(v2sc + 8 * jj)) : make_float2(0.f, 0.f);
              const float2 sh2 = v2sh ? __ldg(reinterpret_cast<const float2 *>(v2sh + 8 * jj)) : make_float2(0.f, 0.f);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                if (!rok[h]) continue;
                float a0 = sums[4 * j + 2 * h], a1 = sums[4 * j + 2 * h + 1];
                epi2_rn(a0, a1, vsc, sc, vsh, sh, nullptr, p.post_relu);
                epi2_rn(a0, a1, v2sc, sc2, v2sh, sh2, nullptr, p.post2_relu);
                uint32_t hh, ll;
                split_f16x2(a0, a1, hh, ll);
                uint32_t *hs = reinterpret_cast<uint32_t *>(brow + h * 1024 + (((uint32_t)jj ^ rsw) * 16));
                hs[0] = hh;
                if (SPLIT) hs[BOX_BYTES / 4] = ll;
              }
            }
            fence_proxy_async();
            named_bar_sync(3 + wg, 128);
            if (issue) {
              tma_store_2d(&tmap_out_hi, stg_a, c0, r0);
              if (SPLIT) tma_store_2d(&tmap_out_lo, stg_a + BOX_BYTES, c0, r0);
            }
            if (stg_issuer) bulk_commit();
            continue;
          }
          if (st32 && (RES || !p.res)) {
            uint8_t *brow = (RES ? res_sm + 2 * cc * BOX_BYTES : stg) + (frow - 64 * wg) * 128 + 8 * (lane & 1);    // row frow + 8 h: + 1024 h
            const float *vsc = p.post_scale ? p.post_scale + c0 + fcol : nullptr, *vsh = p.post_shift ? p.post_shift + c0 + fcol : nullptr;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * cc + jj;
              if (c0 + 8 * jj + fcol >= p.Cout) continue;
              const uint32_t piece = (uint32_t)(2 * (jj & 3) + ((lane & 3) >> 1)) ^ rsw;
              const float2 sc = vsc ? __ldg(reinterpret_cast<const float2 *>(vsc + 8 * jj)) : make_float2(0.f, 0.f);
              const float2 sh = vsh ? __ldg(reinterpret_cast<const float2 *>(vsh + 8 * jj)) : make_float2(0.f, 0.f);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                if (!rok[h]) continue;
                float2 *f32 = reinterpret_cast<float2 *>(brow + h * 1024 + (jj >> 2) * BOX_BYTES + piece * 16);
                float y0 = sums[4 * j + 2 * h], y1 = sums[4 * j + 2 * h + 1];
                epi2_rn<RES>(y0, y1, vsc, sc, vsh, sh, f32, p.post_relu);
                *f32 = make_float2(y0, y1);
                sums[4 * j + 2 * h] = y0; sums[4 * j + 2 * h + 1] = y1;
              }
            }
          } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int m = m0 + frow + 8 * h;
            if (m >= p.M) continue;
            int n_img, oy, ox;
            row_geom(m, n_img, oy, ox);
            const float *rrow = res_row(m, n_img, oy, ox);
            float *orow = st32 ? nullptr : out_row(m, n_img, oy, ox);
            uint8_t *brow = (RES ? res_sm + 2 * cc * BOX_BYTES : stg) + (frow - 64 * wg + 8 * h) * 128 + 8 * (lane & 1);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * cc + jj;
              const int c = n0 + 8 * j + fcol;
              if (c >= p.Cout) continue;
              // columns 8 j + fcol, + 1: box jj / 4 of the pass, piece 2 (jj % 4) + fcol / 4
              const uint32_t piece = (uint32_t)(2 * (jj & 3) + ((lane & 3) >> 1)) ^ rsw;
              float2 *f32 = reinterpret_cast<float2 *>(brow + (jj >> 2) * BOX_BYTES + piece * 16);
              float y0 = sums[4 * j + 2 * h], y1 = sums[4 * j + 2 * h + 1];
              value2(c, f32, rrow, y0, y1);
              if (st32) *f32 = make_float2(y0, y1);
              else if (orow) *reinterpret_cast<float2 *>(orow + c) = make_float2(y0, y1);
              sums[4 * j + 2 * h] = y0; sums[4 * j + 2 * h + 1] = y1;
            }
          }
          }
          if (st32) {
            fence_proxy_async();
            named_bar_sync(3 + wg, 128);
            if (issue) {
              const uint32_t src = RES ? smem_base + C::RES_OFFSET + wg * C::RES_SLOT_BYTES + 2 * cc * BOX_BYTES : stg_a;
              tma_store_2d(&tmap_out, src, c0, r0);
              if (c0 + 32 < p.Cout) tma_store_2d(&tmap_out, src + BOX_BYTES, c0 + 32, r0);
            }
            if (stg_issuer) bulk_commit();
          }
          if (p.out_hi) {
            if (st2) acquire(RES && st32 && !SHORT);          // SHORT: the pair is staged in the slot the fp32 stores read
            if (st2) {
              uint8_t *brow = stg + (frow - 64 * wg) * 128 + 4 * (lane & 3);
              const float *vsc = p.post2_scale ? p.post2_scale + c0 + fcol : nullptr, *vsh = p.post2_shift ? p.post2_shift + c0 + fcol : nullptr;
#pragma unroll
              for (int jj = 0; jj < 8; ++jj) {
                const int j = 8 * cc + jj;
                if (c0 + 8 * jj + fcol >= p.Cout) continue;
                const float2 sc = vsc ? __ldg(reinterpret_cast<const float2 *>(vsc + 8 * jj)) : make_float2(0.f, 0.f);
                const float2 sh = vsh ? __ldg(reinterpret_cast<const float2 *>(vsh + 8 * jj)) : make_float2(0.f, 0.f);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  if (!rok[h]) continue;
                  float a0 = sums[4 * j + 2 * h], a1 = sums[4 * j + 2 * h + 1];
                  epi2_rn(a0, a1, vsc, sc, vsh, sh, nullptr, p.post2_relu);
                  uint32_t hh, ll;
                  split_f16x2(a0, a1, hh, ll);
                  // columns 8 j + fcol, + 1 of the pass: piece jj of the 128-byte row
                  uint32_t *hs = reinterpret_cast<uint32_t *>(brow + h * 1024 + (((uint32_t)jj ^ rsw) * 16));
                  hs[0] = hh;
                  if (SPLIT) hs[BOX_BYTES / 4] = ll;
                }
              }
            } else {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int m = m0 + frow + 8 * h;
              if (m >= p.M) continue;
              __half *hrow = reinterpret_cast<__half *>(p.out_hi) + (size_t)m * p.out2_ld;
              __half *lrow = SPLIT ? reinterpret_cast<__half *>(p.out_lo) + (size_t)m * p.out2_ld : nullptr;
              uint8_t *brow = stg + (frow - 64 * wg + 8 * h) * 128 + 4 * (lane & 3);
#pragma unroll
              for (int jj = 0; jj < 8; ++jj) {
                const int j = 8 * cc + jj;
                const int c = n0 + 8 * j + fcol;
                if (c >= p.Cout) continue;
                uint32_t hh, ll;
                pair2(c, sums[4 * j + 2 * h], sums[4 * j + 2 * h + 1], hh, ll);
                if (st2) {       // columns 8 j + fcol, + 1 of the pass: piece jj of the 128-byte row
                  uint32_t *hs = reinterpret_cast<uint32_t *>(brow + (((uint32_t)jj ^ rsw) * 16));
                  hs[0] = hh;
                  if (SPLIT) hs[BOX_BYTES / 4] = ll;
                } else {
                  *reinterpret_cast<uint32_t *>(hrow + c) = hh;
                  if (SPLIT) *reinterpret_cast<uint32_t *>(lrow + c) = ll;
                }
              }
            }
            }
            if (st2) {
              fence_proxy_async();
              named_bar_sync(3 + wg, 128);
              if (issue) {
                tma_store_2d(&tmap_out_hi, stg_a, c0, r0);
                if (SPLIT) tma_store_2d(&tmap_out_lo, stg_a + BOX_BYTES, c0, r0);
              }
              if (stg_issuer) bulk_commit();
            }
          }
        }
      } else {
      // register-staged producers: every output from registers
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + frow + 8 * h;
        if (m >= p.M) continue;
        int n_img, oy, ox;
        row_geom(m, n_img, oy, ox);
        const float *rrow = res_row(m, n_img, oy, ox);
        float *orow = out_row(m, n_img, oy, ox);
        __half *hrow = p.out_hi ? reinterpret_cast<__half *>(p.out_hi) + (size_t)m * p.out2_ld : nullptr;
        __half *lrow = SPLIT && p.out_hi ? reinterpret_cast<__half *>(p.out_lo) + (size_t)m * p.out2_ld : nullptr;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = n0 + 8 * j + fcol;
          if (c >= p.Cout) continue;
          const bool two = c + 1 < p.Cout;
          float y[2] = {sums[4 * j + 2 * h], sums[4 * j + 2 * h + 1]};
          if (p.vec_out) {
            value2(c, nullptr, rrow, y[0], y[1]);
            if (orow) *reinterpret_cast<float2 *>(orow + c) = make_float2(y[0], y[1]);
            if (hrow) {
              uint32_t hh, ll;
              pair2(c, y[0], y[1], hh, ll);
              *reinterpret_cast<uint32_t *>(hrow + c) = hh;
              if (SPLIT) *reinterpret_cast<uint32_t *>(lrow + c) = ll;
            }
          } else {             // ragged / unaligned outputs (IEF 85- and 72-wide heads): element-wise
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if (e == 1 && !two) break;
              float v = y[e];
              if (p.post_scale) v *= __ldg(p.post_scale + c + e);
              if (p.post_shift) v += __ldg(p.post_shift + c + e);
              if (rrow) v += rrow[c + e];
              if (p.post_relu) v = fmaxf(v, 0.f);
              if (orow) orow[c + e] = v;
            }
          }
        }
      }
      }
      if (RES && ti + 1 < my_tiles) {
        if (prof) p.dbg[6] -= clock64();
        named_bar_sync(1 + wg, 128);                       // every thread of the warpgroup has read the slot
        if (res_issuer) {
          if (SHORT) {                                     // every store staged in the slot has read it
            if (stage) bulk_wait_read<0>();
          } else if (stage & STAGE_OUT) {                  // the slot's fp32 stores have read it (the pair's may still run)
            if (stage & STAGE_PAIR) bulk_wait_read<1>();
            else bulk_wait_read<0>();
          }
          load_res(ti + 1);
        }
        if (prof) p.dbg[6] += clock64();
      }
      if (prof) p.dbg[4] += clock64();
    }
    if (stg_issuer) bulk_wait_all();                       // the last stores have completed before the CTA exits
    if (prof) { p.dbg[2] = clock64() - (RES || MEM_STAMPS ? p.dbg[2] : t_start); if (!MEM_STAMPS) p.dbg[3] = t_wait; }
    if (prof) { p.dbg[7] = C::TM; p.dbg[8] = BN; }       // the tile: pixels x output channels
  }
}

// Chained 1x1 pair (hd_conv_gemm_chain): conv3 of a bottleneck unit (K = 64 -> 256, bias, row-aligned residual, fp32 output or its
// strided subsample, the next unit's pre-activation as the post2 pair) and conv1 of the identity unit after it (K = 256 -> 64, whose
// A operand is exactly that pair) in one persistent kernel.  Tile: 128 rows, the two consumer warpgroups 64 rows each, one producer
// warpgroup.  Per tile, for each 64-column segment s of conv3's output: conv3's wgmmas (one K chunk, flushed once as in SHORT), its
// staged epilogue (v into the residual slot and out by TMA store, or from registers for out_subsample), the pair of v written into
// the warpgroup's pair chunk -- 64 rows x 128 bytes in the 128-byte swizzle, conv1's A layout for K chunk s -- and conv1's wgmmas on
// it.  conv1 sees its K chunks in the same order as on its own, with the running sums flushed every PCH = 2 chunks, and every
// epilogue product and sum is rounded as in the two launches: the outputs are the same bits.  conv1's epilogue stages its pair in
// the pair chunk and writes it by TMA.  Neither the pair between the two convs nor conv1's reads of it ever reach HBM.
//
// Shared memory: two A stages (conv3's 128 x 64 input pair), two weight stages (conv3's segment box and conv1's chunk box, head and
// remainder), per warpgroup two 16 KB residual slots (segment parity; each the fp32 staging of its segment, the next-but-one
// segment's residual is loaded into it once the store has read it) and the 16 KB pair chunk.
template <bool SPLIT>
struct ChainCfg {
  static constexpr int NUM_THREADS = 384;
  static constexpr int SEGS = 4;                                   // conv3's 256 output columns = conv1's four 64-wide K chunks
  static constexpr int A_BYTES = BM * 128;
  static constexpr int A_STAGE = (SPLIT ? 2 : 1) * A_BYTES;
  static constexpr int W1_OFFSET = (SPLIT ? 2 : 1) * BOX_BYTES;   // in a weight stage: conv3's box (+ remainder), then conv1's
  static constexpr int W_STAGE = 2 * W1_OFFSET;
  static constexpr int RES_SLOT = 64 * 64 * 4;
  static constexpr int PAIR_BYTES = 2 * BOX_BYTES;
  static constexpr int W_OFFSET = 2 * A_STAGE;
  static constexpr int RES_OFFSET = W_OFFSET + 2 * W_STAGE;
  static constexpr int PAIR_OFFSET = RES_OFFSET + 4 * RES_SLOT;   // slot e of warpgroup g at 2 g + e
  static constexpr int BAR_OFFSET = PAIR_OFFSET + 2 * PAIR_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFFSET + 128 + 1024;
  static_assert(SMEM_BYTES <= 232448, "dynamic shared memory beyond the 227 KB a CTA can opt into");
  static constexpr int PROD_REGS = 40, CONS_REGS = 232;
  static_assert(256 * CONS_REGS + 128 * PROD_REGS <= NUM_THREADS * (65536 / NUM_THREADS / 8 * 8), "setmaxnreg split beyond the CTA's registers");
};

template <bool SPLIT>
__global__ void __launch_bounds__(384, 1)
conv_chain_tc_kernel(const ConvParams p, const ConvParams q, const __grid_constant__ CUtensorMap tw3_hi,
                     const __grid_constant__ CUtensorMap tw3_lo, const __grid_constant__ CUtensorMap tw1_hi,
                     const __grid_constant__ CUtensorMap tw1_lo, const __grid_constant__ CUtensorMap tmap_res,
                     const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_r1_hi,
                     const __grid_constant__ CUtensorMap tmap_r1_lo, const int st32) {
  using C = ChainCfg<SPLIT>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t *smem = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + C::BAR_OFFSET;
  auto full_a = [&](int s) { return bar_base + 8u * s; };
  auto empty_a = [&](int s) { return bar_base + 8u * (2 + s); };
  auto full_w = [&](int s) { return bar_base + 8u * (4 + s); };
  auto empty_w = [&](int s) { return bar_base + 8u * (6 + s); };
  auto res_bar = [&](int g, int e) { return bar_base + 8u * (8 + 2 * g + e); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = (p.M + BM - 1) / BM;
  const int my_tiles = (num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(full_a(s), 128);       // every producer thread, hardware arrive when its cp.asyncs land
      mbar_init(empty_a(s), 8);        // one arrive per consumer warp once its conv3 wgmmas have read the stage
      mbar_init(full_w(s), 1);         // arrive.expect_tx of the weight loads
      mbar_init(empty_w(s), 8);
    }
    for (int i = 0; i < 4; ++i) mbar_init(bar_base + 8u * (8 + i), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= W_PROD) {
    // ---- producers: conv3's input pair by cp.async (1x1, stride 1: input row m is output row m), the weights by TMA ----
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(C::PROD_REGS));
    const int t = threadIdx.x - W_PROD * 32, j = t & 7, rb = t >> 3;
    const uint32_t off0 = (uint32_t)rb * 128u + (uint32_t)((j ^ (rb & 7)) << 4);
    const __half *ihi = reinterpret_cast<const __half *>(p.in_hi);
    const __half *ilo = reinterpret_cast<const __half *>(p.in_lo);
    int wq = 0;
    for (int ti = 0; ti < my_tiles; ++ti) {
      const int m0 = ((int)blockIdx.x + ti * (int)gridDim.x) * BM;
      const int sa = ti & 1;
      mbar_wait(empty_a(sa), ((uint32_t)(ti >> 1) & 1u) ^ 1u);
      const uint32_t a_hi = smem_base + sa * C::A_STAGE + off0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int m = m0 + rb + 16 * i;
        const bool ok = m < p.M;
        const int e = ok ? m * (int)p.in_ld + j * 8 : 0;
        cp_async16(a_hi + i * 16 * 128, ihi + e, ok ? 16u : 0u);
        if (SPLIT) cp_async16(a_hi + C::A_BYTES + i * 16 * 128, ilo + e, ok ? 16u : 0u);
      }
      asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(full_a(sa)) : "memory");
      if (t == 0) {
        for (int s = 0; s < C::SEGS; ++s, ++wq) {
          const int sw = wq & 1;
          mbar_wait(empty_w(sw), ((uint32_t)(wq >> 1) & 1u) ^ 1u);
          mbar_arrive_expect_tx(full_w(sw), 2 * C::W1_OFFSET);
          const uint32_t wb = smem_base + C::W_OFFSET + sw * C::W_STAGE;
          tma_load_2d(wb, &tw3_hi, full_w(sw), 0, 64 * s);                    // conv3's output channels 64 s .. 64 s + 63
          if (SPLIT) tma_load_2d(wb + BOX_BYTES, &tw3_lo, full_w(sw), 0, 64 * s);
          tma_load_2d(wb + C::W1_OFFSET, &tw1_hi, full_w(sw), 64 * s, 0);     // conv1's K chunk s
          if (SPLIT) tma_load_2d(wb + C::W1_OFFSET + BOX_BYTES, &tw1_lo, full_w(sw), 64 * s, 0);
        }
      }
    }
    cp_async_commit();
    cp_async_wait<0>();
  } else {
    // ---- consumers ----
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(C::CONS_REGS));
    const int wg = warp >> 2;
    const int frow = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's fragment rows: frow, frow + 8
    const int fcol = 2 * (lane & 3);                            // and columns 8 j + fcol, + 1
    const uint32_t rsw = (uint32_t)(lane >> 2);                 // the swizzle of this thread's rows
    const bool issuer = (threadIdx.x & 127) == 0;               // the warpgroup's TMA loads and stores (bulk groups are per thread)
    const uint32_t pb_a = smem_base + C::PAIR_OFFSET + wg * C::PAIR_BYTES;
    uint8_t *const pbrow = smem + C::PAIR_OFFSET + wg * C::PAIR_BYTES + (frow - 64 * wg) * 128 + 4 * (lane & 3);
    auto slot_a = [&](int e) { return smem_base + C::RES_OFFSET + (2 * wg + e) * C::RES_SLOT; };
    // segment u = 4 ti + s of this CTA's walk: its residual rows in slot u & 1
    auto load_res = [&](int u) {
      if ((u >> 2) >= my_tiles) return;
      const int r0 = ((int)blockIdx.x + (u >> 2) * (int)gridDim.x) * BM + 64 * wg, c0 = 64 * (u & 3);
      const int boxes = r0 < p.M ? 2 : 0;
      mbar_arrive_expect_tx(res_bar(wg, u & 1), boxes * BOX_BYTES);
      for (int b = 0; b < boxes; ++b) tma_load_2d(slot_a(u & 1) + b * BOX_BYTES, &tmap_res, res_bar(wg, u & 1), c0 + 32 * b, r0);
    };
    if (issuer) { load_res(0); load_res(1); }
    float acc3[32], accx3[SPLIT ? 32 : 1], acc1[32], accx1[SPLIT ? 32 : 1], sums1[32];
    const int hw = p.Ho * p.Wo;
    int wq = 0;
    for (int ti = 0; ti < my_tiles; ++ti) {
      const int m0 = ((int)blockIdx.x + ti * (int)gridDim.x) * BM, r0 = m0 + 64 * wg;
      const bool rok[2] = {m0 + frow < p.M, m0 + frow + 8 < p.M};
      const int sa = ti & 1;
      mbar_wait(full_a(sa), (uint32_t)(ti >> 1) & 1u);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // cp.async (generic proxy) data -> wgmma (async proxy)
      const uint32_t a_hi = smem_base + sa * C::A_STAGE + wg * 64 * 128;
      const uint64_t da_hi = make_smem_desc(a_hi), da_lo = make_smem_desc(a_hi + C::A_BYTES);
      const uint64_t dp_hi = make_smem_desc(pb_a), dp_lo = make_smem_desc(pb_a + BOX_BYTES);
#pragma unroll
      for (int i = 0; i < 32; ++i) sums1[i] = 0.f;
      for (int s = 0; s < C::SEGS; ++s, ++wq) {
        const int u = 4 * ti + s, e = u & 1, sw = wq & 1;
        mbar_wait(full_w(sw), (uint32_t)(wq >> 1) & 1u);
        const uint32_t wb = smem_base + C::W_OFFSET + sw * C::W_STAGE;
        const uint64_t d3_hi = make_smem_desc(wb), d3_lo = make_smem_desc(wb + BOX_BYTES);
        const uint64_t d1_hi = make_smem_desc(wb + C::W1_OFFSET), d1_lo = make_smem_desc(wb + C::W1_OFFSET + BOX_BYTES);
        // conv3, output columns 64 s .. 64 s + 63: one K chunk, the products of the 128 x 64 SHORT tile
        fence_regs(acc3);
        if constexpr (SPLIT) fence_regs(accx3);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t adv = (uint64_t)((k * 32) >> 4);
          if constexpr (SPLIT) {
            wgmma_m64n64k16_f16(accx3, da_lo + adv, d3_hi + adv, k != 0);
            wgmma_m64n64k16_f16(accx3, da_hi + adv, d3_lo + adv, 1u);
          }
          wgmma_m64n64k16_f16(acc3, da_hi + adv, d3_hi + adv, k != 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(acc3);
        if constexpr (SPLIT) fence_regs(accx3);
        if (s == C::SEGS - 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_a(sa));
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) acc3[i] = __fadd_rn(0.f, acc3[i]);   // SHORT's one flush (a -0 becomes +0)
        if constexpr (SPLIT) {
#pragma unroll
          for (int i = 0; i < 32; ++i) acc3[i] += accx3[i] * (1.0f / 2048.0f);
        }
        // v = acc + bias + residual (the slot, in the TMA box layout), staged over the residual or kept for the subsample
        mbar_wait(res_bar(wg, e), (uint32_t)(u >> 1) & 1u);
        uint8_t *brow = smem + C::RES_OFFSET + (2 * wg + e) * C::RES_SLOT + (frow - 64 * wg) * 128 + 8 * (lane & 1);
        const float *vsh = p.post_shift ? p.post_shift + 64 * s + fcol : nullptr;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const uint32_t piece = (uint32_t)(2 * (jj & 3) + ((lane & 3) >> 1)) ^ rsw;
          const float2 sh = vsh ? __ldg(reinterpret_cast<const float2 *>(vsh + 8 * jj)) : make_float2(0.f, 0.f);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!rok[h]) continue;
            float2 *f32 = reinterpret_cast<float2 *>(brow + h * 1024 + (jj >> 2) * BOX_BYTES + piece * 16);
            float y0 = acc3[4 * jj + 2 * h], y1 = acc3[4 * jj + 2 * h + 1];
            epi2_rn<true>(y0, y1, nullptr, make_float2(0.f, 0.f), vsh, sh, f32, 0);
            if (st32) *f32 = make_float2(y0, y1);
            acc3[4 * jj + 2 * h] = y0; acc3[4 * jj + 2 * h + 1] = y1;
          }
        }
        if (!st32) {                   // x[:, ::s, ::s] from registers
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int m = m0 + frow + 8 * h;
            if (m >= p.M) continue;
            const int n_img = m / hw, r = m - n_img * hw, oy = r / p.Wo, ox = r - oy * p.Wo;
            if (oy % p.out_sub != 0 || ox % p.out_sub != 0) continue;
            const int Hs = (p.Ho + p.out_sub - 1) / p.out_sub, Ws = (p.Wo + p.out_sub - 1) / p.out_sub;
            float *orow = p.out + ((size_t)((size_t)n_img * Hs + oy / p.out_sub) * Ws + ox / p.out_sub) * p.out_ld + 64 * s + fcol;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              *reinterpret_cast<float2 *>(orow + 8 * jj) = make_float2(acc3[4 * jj + 2 * h], acc3[4 * jj + 2 * h + 1]);
          }
        }
        // the pair of v = conv1's A operand for K chunk s.  The chunk was last read by this warpgroup's conv1 wgmmas of chunk s - 1
        // (waited for), or at s = 0 by the previous tile's conv1 output stores.
        if (s == 0 && ti > 0) {
          if (issuer) bulk_wait_read<0>();
          named_bar_sync(1 + wg, 128);
        }
        {
          const float *v2sc = p.post2_scale ? p.post2_scale + 64 * s + fcol : nullptr, *v2sh = p.post2_shift ? p.post2_shift + 64 * s + fcol : nullptr;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const float2 sc2 = v2sc ? __ldg(reinterpret_cast<const float2 *>(v2sc + 8 * jj)) : make_float2(0.f, 0.f);
            const float2 sh2 = v2sh ? __ldg(reinterpret_cast<const float2 *>(v2sh + 8 * jj)) : make_float2(0.f, 0.f);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float a0 = acc3[4 * jj + 2 * h], a1 = acc3[4 * jj + 2 * h + 1];
              epi2_rn(a0, a1, v2sc, sc2, v2sh, sh2, nullptr, p.post2_relu);
              uint32_t hh, ll;
              split_f16x2(a0, a1, hh, ll);
              uint32_t *hs = reinterpret_cast<uint32_t *>(pbrow + h * 1024 + (((uint32_t)jj ^ rsw) * 16));
              hs[0] = hh;
              if (SPLIT) hs[BOX_BYTES / 4] = ll;
            }
          }
        }
        fence_proxy_async();             // the slot's fp32 values -> TMA store, the pair chunk -> wgmma
        named_bar_sync(1 + wg, 128);
        if (issuer && st32) {
          if (r0 < p.M) {
            tma_store_2d(&tmap_out, slot_a(e), 64 * s, r0);
            tma_store_2d(&tmap_out, slot_a(e) + BOX_BYTES, 64 * s + 32, r0);
          }
          bulk_commit();
        }
        // conv1, K chunk s
        fence_regs(acc1);
        if constexpr (SPLIT) fence_regs(accx1);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t adv = (uint64_t)((k * 32) >> 4);
          if constexpr (SPLIT) {
            wgmma_m64n64k16_f16(accx1, dp_lo + adv, d1_hi + adv, (s | k) != 0);
            wgmma_m64n64k16_f16(accx1, dp_hi + adv, d1_lo + adv, 1u);
          }
          wgmma_m64n64k16_f16(acc1, dp_hi + adv, d1_hi + adv, !((s & 1) == 0 && k == 0));
        }
        wgmma_commit();
        if (issuer) {                    // under the wgmmas: the slot's store has read it; the next-but-one segment's residual
          bulk_wait_read<0>();
          load_res(u + 2);
        }
        wgmma_wait<0>();
        fence_regs(acc1);
        if constexpr (SPLIT) fence_regs(accx1);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_w(sw));
        if (s & 1) {
#pragma unroll
          for (int i = 0; i < 32; ++i) sums1[i] += acc1[i];
        }
      }
      if constexpr (SPLIT) {
#pragma unroll
        for (int i = 0; i < 32; ++i) sums1[i] += accx1[i] * (1.0f / 2048.0f);
      }
      // conv1's epilogue: its pair (post, then post2 where given) staged in the pair chunk and written by TMA
      named_bar_sync(1 + wg, 128);       // every warp's wgmmas of the last chunk have read the pair chunk
      {
        const float *vsc = q.post_scale ? q.post_scale + fcol : nullptr, *vsh = q.post_shift ? q.post_shift + fcol : nullptr;
        const float *v2sc = q.post2_scale ? q.post2_scale + fcol : nullptr, *v2sh = q.post2_shift ? q.post2_shift + fcol : nullptr;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const float2 sc = vsc ? __ldg(reinterpret_cast<const float2 *>(vsc + 8 * jj)) : make_float2(0.f, 0.f);
          const float2 sh = vsh ? __ldg(reinterpret_cast<const float2 *>(vsh + 8 * jj)) : make_float2(0.f, 0.f);
          const float2 sc2 = v2sc ? __ldg(reinterpret_cast<const float2 *>(v2sc + 8 * jj)) : make_float2(0.f, 0.f);
          const float2 sh2 = v2sh ? __ldg(reinterpret_cast<const float2 *>(v2sh + 8 * jj)) : make_float2(0.f, 0.f);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float a0 = sums1[4 * jj + 2 * h], a1 = sums1[4 * jj + 2 * h + 1];
            epi2_rn(a0, a1, vsc, sc, vsh, sh, nullptr, q.post_relu);
            epi2_rn(a0, a1, v2sc, sc2, v2sh, sh2, nullptr, q.post2_relu);
            uint32_t hh, ll;
            split_f16x2(a0, a1, hh, ll);
            uint32_t *hs = reinterpret_cast<uint32_t *>(pbrow + h * 1024 + (((uint32_t)jj ^ rsw) * 16));
            hs[0] = hh;
            if (SPLIT) hs[BOX_BYTES / 4] = ll;
          }
        }
      }
      fence_proxy_async();
      named_bar_sync(1 + wg, 128);
      if (issuer) {
        if (r0 < p.M) {
          tma_store_2d(&tmap_r1_hi, pb_a, 0, r0);
          if (SPLIT) tma_store_2d(&tmap_r1_lo, pb_a + BOX_BYTES, 0, r0);
        }
        bulk_commit();
      }
    }
    if (issuer) bulk_wait_all();         // the last stores have completed before the CTA exits
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void *ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(ptr);
    else (void)cudaGetLastError();
  }
  return fn;
}

constexpr int kMaxDevices = 64;

// Map over a row-major [rows, cols] activation matrix (row pitch ld_bytes) with the box of one warpgroup's epilogue: 128 bytes of
// columns x 64 rows, 128-byte swizzle.  gdim = {cols, rows}: TMA clips a partial box and never touches the pitch padding.
int encode_epilogue_map(CUtensorMap *tm, bool fp16, const void *base, int cols, int rows, long long ld_bytes, const char *what) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_last_error_text("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return HD_ERR_UNSUPPORTED; }
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld_bytes};
  const cuuint32_t box[2] = {fp16 ? 64u : 32u, 64u};
  const cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(tm, fp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void *>(base), gdim, gstride,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[96];
    snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled (%s) failed with CUresult %d", what, (int)r);
    set_last_error_text(msg);
    return HD_ERR_CUDA;
  }
  return HD_OK;
}

template <bool SPLIT, int PCH, bool HALF, bool GATHER = false, bool ASPLIT = false, int BN = 64, bool RES = false, bool SHORT = false,
          bool CM = false>
int launch_tc(const ConvParams &p, const hd_conv_desc *d, cudaStream_t st) {
  using C = Cfg<SPLIT, HALF, ASPLIT, BN, RES, SHORT, CM>;
  // function attributes and the SM count are per device: a process may drive several GPUs through this library
  static bool configured[kMaxDevices] = {};
  static int num_sms[kMaxDevices] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) { set_last_error_text("conv_gemm_tc: device ordinal out of range"); return HD_ERR_UNSUPPORTED; }
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(conv_gemm_tc_kernel<SPLIT, PCH, HALF, GATHER, ASPLIT, BN, RES, SHORT, CM>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) { set_last_error("conv_gemm_tc attr", e); return HD_ERR_CUDA; }
    cudaDeviceGetAttribute(&num_sms[dev], cudaDevAttrMultiProcessorCount, dev);
    if (num_sms[dev] <= 0) { set_last_error_text("conv_gemm_tc: no multiprocessor count"); return HD_ERR_CUDA; }
    configured[dev] = true;
  }
  // weight maps with the 64-row box (hd_make_weight_tmap accepts no other; a 128-wide N tile loads two boxes)
  alignas(64) CUtensorMap thi, tlo;
  const void *mhi = d->tmap_hi_n64 ? d->tmap_hi_n64 : d->tmap_hi;
  const void *mlo = d->tmap_hi_n64 ? d->tmap_lo_n64 : d->tmap_lo;
  memcpy(&thi, mhi, sizeof(CUtensorMap));
  memcpy(&tlo, mlo ? mlo : mhi, sizeof(CUtensorMap));     // mlo is null only without SPLIT, which never loads it (launch_conv_tc)
  // The residual and output maps are encoded here from p.res / p.out / p.out_hi / p.out_lo on every launch, never taken from the
  // descriptor's activation maps, so they always describe the buffers this launch reads and writes.  Maps not used stay copies
  // of the weight map.
  alignas(64) CUtensorMap tres, tout, tohi, tolo;
  memcpy(&tres, &thi, sizeof(CUtensorMap));
  memcpy(&tout, &thi, sizeof(CUtensorMap));
  memcpy(&tohi, &thi, sizeof(CUtensorMap));
  memcpy(&tolo, &thi, sizeof(CUtensorMap));
  int rc = HD_OK;
  if (RES) rc = encode_epilogue_map(&tres, false, p.res, p.Cout, p.M, p.res_ld * 4, "residual");
  // Pre-split layers stage outputs in shared memory for TMA stores, except those TMA cannot write: the strided subsample, and a
  // pair whose row pitch is not a multiple of 16 bytes (vec_out, checked by launch_conv_tc, gives aligned bases and fp32 pitches).
  int stage = 0;
  if (ASPLIT && p.out && !p.out_sub) {
    stage |= STAGE_OUT;
    if (rc == HD_OK) rc = encode_epilogue_map(&tout, false, p.out, p.Cout, p.M, p.out_ld * 4, "output");
  }
  if (ASPLIT && p.out_hi && p.out2_ld % 8 == 0) {
    stage |= STAGE_PAIR;
    if (rc == HD_OK) rc = encode_epilogue_map(&tohi, true, p.out_hi, p.Cout, p.M, p.out2_ld * 2, "output head");
    if (rc == HD_OK && SPLIT) rc = encode_epilogue_map(&tolo, true, p.out_lo, p.Cout, p.M, p.out2_ld * 2, "output remainder");
  }
  if (rc != HD_OK) return rc;
  const int num_tiles = ceil_div(p.M, C::TM) * ceil_div(p.Cout, BN);
  const int ctas = C::CTAS * num_sms[dev];       // persistent: one CTA per SM (SHORT: two) walks the tile list
  dim3 grid(num_tiles < ctas ? num_tiles : ctas);
  conv_gemm_tc_kernel<SPLIT, PCH, HALF, GATHER, ASPLIT, BN, RES, SHORT, CM>
      <<<grid, C::NUM_THREADS, C::SMEM_BYTES, st>>>(p, thi, tlo, tres, tout, tohi, tolo, stage);
  return check_launch("conv_gemm_tc_kernel");
}

// A 128-wide tile does the work of two 64-wide ones in less time, but there are half as many to spread over the SMs.  Take it
// unless that costs more than an eighth in whole waves of tiles (the small late layers of a small batch).
bool wide_n_tile(const ConvParams &p) {
  if (p.Cout <= 64) return false;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sms <= 0) return true;
  const long long m_tiles = ceil_div(p.M, BM);
  const long long w128 = (m_tiles * ceil_div(p.Cout, 128) + sms - 1) / sms, w64 = (m_tiles * ceil_div(p.Cout, 64) + sms - 1) / sms;
  return 16 * w128 <= 9 * w64;      // 2 w128 <= 1.125 w64
}

// The 64-channel x 256-pixel tile (CM) for the root conv1 over the planes (fp32 output alone, 32-bit input offsets for the lean
// plane loop), unless the halved tile count costs more than an eighth in whole waves, as in wide_n_tile.  Block 1's 3x3 Cout = 64
// layers measured slower on it than on the 128 x 64 tile: with two stages their consumers wait for data (DESIGN.md section 8).

bool cout_on_m(const ConvParams &p) {
  if (!p.planes || p.Cout != 64 || p.res || p.out_sub || p.out_hi || !p.out) return false;
  if ((long long)p.n_img * p.H * p.W * p.in_ld >= (1ll << 31)) return false;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sms <= 0) return true;
  const long long w256 = (ceil_div(p.M, 256) + sms - 1) / sms, w128 = (ceil_div(p.M, BM) + sms - 1) / sms;
  return 16 * w256 <= 9 * w128;     // 2 w256 <= 1.125 w128
}

// Whether the SHORT kernel runs two CTAs per SM on this device (checked once per device); if not, its layers keep the one-CTA kernels.
template <bool SPLIT, bool RES>
bool short_k_two_ctas() {
  using C = Cfg<SPLIT, true, true, 64, RES, true>;
  static int two[kMaxDevices] = {};      // 0 not checked yet, 1 yes, -1 no
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) return false;
  if (two[dev] == 0) {
    const auto kernel = conv_gemm_tc_kernel<SPLIT, 2, true, false, true, 64, RES, true, false>;
    int n = 0;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, C::NUM_THREADS, C::SMEM_BYTES) != cudaSuccess) {
      (void)cudaGetLastError();
      n = 0;
    }
    two[dev] = n >= 2 ? 1 : -1;
  }
  return two[dev] > 0;
}

// The fp16 paths: 3xFP16 (SPLIT, impl 3) or 1xFP16 (heads only, impl 4).  Both select the same kernel variant for a layer.
template <bool SPLIT>
int launch_conv_f16(const ConvParams &p, const hd_conv_desc *d, cudaStream_t st) {
  if (p.in_hi && p.planes) {           // resnet conv1 over padded RGBX fp16 planes (hd_pack_conv1_planes)
    if (p.Cin != 32 || p.KH != 8 || p.KW != 1 || p.stride != 2 || p.pad_t != 0 || p.pad_l != 0 || p.in_ld != 4 || p.Cout > 64 ||
        p.W % 2 != 0 || 2 * (p.Wo - 1) + 8 > p.W || 2 * (p.Ho - 1) + 7 > p.H || !aligned16(p.in_hi) || !aligned16(p.in_lo) || p.pre_scale) {
      set_last_error_text("hd_conv_gemm(tc planes): needs the conv1 plane geometry (Cin 32, KH 8, KW 1, stride 2, in_ld 4, even W)");
      return HD_ERR_INVALID;
    }
    return cout_on_m(p) ? launch_tc<SPLIT, 2, true, false, true, 64, false, false, true>(p, d, st) : launch_tc<SPLIT, 2, true, false, true>(p, d, st);
  }
  // drain every 2 chunks = 8 fp16 tensor-core accumulations between round-to-nearest adds (both modes: impl 4 then runs the
  // rounded operations impl 3 runs on zero remainders)
  if (p.in_hi) {                       // pre-split fp16 activations: cp.async producer
    if (p.Cin % 64 != 0 || p.K % 64 != 0 || p.in_ld % 8 != 0 || !aligned16(p.in_hi) || !aligned16(p.in_lo) || p.pre_scale) {
      set_last_error_text("hd_conv_gemm(tc split-A): needs Cin % 64 == 0, in_ld % 8 == 0, aligned in_hi/in_lo, no prologue");
      return HD_ERR_INVALID;
    }
    // A residual row-aligned with the output (row m of `res` belongs to output row m) is loaded by TMA into shared memory ahead of
    // the epilogue; vec_out (checked above) gives it the 16-byte aligned base and row pitch a tensor map needs.  Residual layers
    // have short K, so the 128-wide tile gives up its third stage for the slots.
    const bool res_rows = p.res && p.res_stride == 1 && p.res_H == p.Ho && p.res_W == p.Wo && p.K <= 8 * 64;
    // K <= 128 (one running-sum flush per tile), 1x1 windows with 32-bit input offsets (the lean producer loop): the
    // 64-wide tile two CTAs per SM, so one CTA's epilogue runs under the other's loads and MMAs.  Only for epilogues that add a
    // row-aligned residual or write the next layer's pair: a layer that writes the fp32 output alone (block 1's shortcut conv)
    // measured slower this way than on the 128-wide tile (DESIGN.md section 8).
    const bool short_k = p.K <= 2 * 64 && p.KH * p.KW == 1 && (long long)p.n_img * p.H * p.W * p.in_ld < (1ll << 31) &&
                         (p.res ? res_rows : p.out_hi != nullptr);
    if (short_k && (res_rows ? short_k_two_ctas<SPLIT, true>() : short_k_two_ctas<SPLIT, false>()))
      return res_rows ? launch_tc<SPLIT, 2, true, false, true, 64, true, true>(p, d, st)
                      : launch_tc<SPLIT, 2, true, false, true, 64, false, true>(p, d, st);
    if (wide_n_tile(p))
      return res_rows ? launch_tc<SPLIT, 2, true, false, true, 128, true>(p, d, st) : launch_tc<SPLIT, 2, true, false, true, 128>(p, d, st);
    return res_rows ? launch_tc<SPLIT, 2, true, false, true, 64, true>(p, d, st) : launch_tc<SPLIT, 2, true, false, true>(p, d, st);
  }
  if (p.Cin % 64 != 0) {               // ragged Cin (resnet conv1: 7x7x3): element-wise gather producer, K zero-padded
    const int segp = (p.KW * p.Cin + 7) & ~7;
    if (p.K_pad % 64 != 0 || p.K_pad < p.KH * segp || p.Cout > 64 || p.pre_scale || p.in_ld != p.Cin) {
      set_last_error_text("hd_conv_gemm(tc gather): needs K_pad % 64 == 0, K_pad >= KH*roundup8(KW*Cin), Cout <= 64, dense pixels, no prologue");
      return HD_ERR_INVALID;
    }
    return launch_tc<SPLIT, 2, true, true>(p, d, st);
  }
  if (!p.in || p.in_ld % 4 != 0 || !aligned16(p.in) || p.K % 64 != 0 ||
      (p.pre_scale && (!aligned16(p.pre_scale) || !aligned16(p.pre_shift) || p.pre_img_stride % 4 != 0))) {
    set_last_error_text("hd_conv_gemm(tc): needs Cin % 32 (tf32) / % 64 (fp16) == 0 and 16-byte aligned input / prologue vectors");
    return HD_ERR_INVALID;
  }
  return launch_tc<SPLIT, 2, true>(p, d, st);
}

}  // namespace

int launch_conv_tc(const ConvParams &p, const hd_conv_desc *d, cudaStream_t st) {
  const bool heads = d->impl == HD_IMPL_TC_1XF16;                     // 1xFP16: fp16 heads only (fill_params refuses remainders)
  const bool split_b = d->impl != HD_IMPL_TC_1XTF32 && !heads;       // 1xTF32 and 1xFP16 read no weight remainder
  if (!d->tmap_hi || (split_b && !d->tmap_lo) || (!d->tmap_hi_n64 && d->tmap_lo_n64) || (d->tmap_hi_n64 && split_b && !d->tmap_lo_n64)) {
    set_last_error_text("hd_conv_gemm(tc): missing tensor maps (tmap_hi/tmap_lo, and tmap_hi_n64/tmap_lo_n64 together or not at all)");
    return HD_ERR_INVALID;
  }
  const bool half = d->impl == HD_IMPL_TC_3XF16 || heads;
  // Compatibility gate, not a kernel limit: the register epilogue below writes the strided subsample for any descriptor, but
  // out_subsample keeps the acceptance rule of the C-ABI (hd_b200.h: pre-split input, Cout % 32 == 0, a plain residual, the
  // activation tensor maps given, HD_CONV_NO_TMA_EPILOGUE unset) so that a descriptor is accepted or refused as before.
  if (p.out_sub) {
    const bool res_plain = !p.res || (p.res_stride == 1 && p.res_H == p.Ho && p.res_W == p.Wo);
    const bool maps = (!p.res || d->tmap_res) && (!p.out_hi || (d->tmap_out_hi && (heads || d->tmap_out_lo)));
    if (!p.in_hi || p.planes || !maps || !res_plain || p.Cout % 32 != 0 || (d->flags & HD_CONV_NO_TMA_EPILOGUE)) {
      set_last_error_text("hd_conv_gemm: out_subsample needs the activation-map epilogue (pre-split input, Cout % 32 == 0, activation maps given)");
      return HD_ERR_UNSUPPORTED;
    }
  }
  if ((p.out_hi || p.in_hi) && (!half || !p.vec_out)) {
    set_last_error_text("hd_conv_gemm(tc): pre-split activations need impl 3 / 4 and 16-byte aligned, 4-column-multiple outputs");
    return HD_ERR_INVALID;
  }
  if (half) return heads ? launch_conv_f16<false>(p, d, st) : launch_conv_f16<true>(p, d, st);
  if (!p.in || p.Cin % 32 != 0 || p.in_ld % 4 != 0 || !aligned16(p.in) || p.K % 32 != 0 ||
      (p.pre_scale && (!aligned16(p.pre_scale) || !aligned16(p.pre_shift) || p.pre_img_stride % 4 != 0))) {
    set_last_error_text("hd_conv_gemm(tc): needs Cin % 32 (tf32) / % 64 (fp16) == 0 and 16-byte aligned input / prologue vectors");
    return HD_ERR_INVALID;
  }
  // 3xTF32: drain every 2 chunks = 8 tensor-core accumulations; 1xTF32 is ~1e-3 anyway: drain rarely
  return d->impl != HD_IMPL_TC_1XTF32 ? launch_tc<true, 2, false>(p, d, st) : launch_tc<false, 8, false>(p, d, st);
}

// Whether conv_chain_tc_kernel runs the pair (hd_b200.h, hd_conv_gemm_chain): shapes and pointers only, no device call.
int chain_check(const hd_conv_desc *a, const hd_conv_desc *b) {
  auto refuse = [](const char *why) {
    char msg[160];
    snprintf(msg, sizeof(msg), "hd_conv_gemm_chain: %s", why);
    set_last_error_text(msg);
    return HD_ERR_UNSUPPORTED;
  };
  if (!a || !b) return refuse("null descriptor");
  if (a->impl != b->impl || (a->impl != HD_IMPL_TC_3XF16 && a->impl != HD_IMPL_TC_1XF16)) return refuse("both convs need impl 3 or impl 4");
  const bool heads = a->impl == HD_IMPL_TC_1XF16;
  auto one_by_one = [heads](const hd_conv_desc *d) {
    return d->KH == 1 && d->KW == 1 && d->stride == 1 && d->pad_t == 0 && d->pad_l == 0 && d->Ho == d->H && d->Wo == d->W &&
           !d->pre_scale && !d->pre_shift && !(d->flags & HD_CONV_INPUT_PLANES) && d->K_pad == d->Cin && d->tmap_hi &&
           (heads ? !d->tmap_lo : d->tmap_lo != nullptr) && !d->tmap_hi_n64;
  };
  if (!one_by_one(a) || !one_by_one(b)) return refuse("both convs must be 1x1 stride 1 without prologue, with their weight maps");
  if (a->Cin != 64 || a->Cout != 256 || b->Cin != a->Cout || b->Cout != 64)
    return refuse("supported shape: conv3 64 -> 256 channels, then conv1 256 -> 64");
  if (!a->in_hi || (heads ? a->in_lo != nullptr : !a->in_lo) || a->in_ld % 8 != 0 || !aligned16(a->in_hi) || (a->in_lo && !aligned16(a->in_lo)) ||
      (long long)a->n_img * a->H * a->W * a->in_ld >= (1ll << 31))
    return refuse("the first conv reads an aligned pre-split pair with 32-bit element offsets");
  if (!a->res || a->res_stride != 1 || a->res_H != a->Ho || a->res_W != a->Wo || a->res_ld % 4 != 0 || !aligned16(a->res))
    return refuse("the first conv needs a row-aligned residual");
  if (!a->out || a->out_ld % 4 != 0 || !aligned16(a->out) || a->out_hi || a->out_lo || a->post_scale || a->post_relu ||
      (a->post_shift && !aligned16(a->post_shift)) || (a->post2_scale == nullptr) != (a->post2_shift == nullptr))
    return refuse("the first conv writes the fp32 output (or its subsample) and hands its post2 pair to the second");
  if (b->n_img != a->n_img || b->H != a->Ho || b->W != a->Wo || b->in || b->in_hi || b->in_lo || b->res || b->out ||
      b->out_subsample > 1 || !b->out_hi || (heads ? b->out_lo != nullptr : !b->out_lo) || b->out2_ld % 8 != 0 ||
      !aligned16(b->out_hi) || (b->out_lo && !aligned16(b->out_lo)))
    return refuse("the second conv reads the first's output rows and writes its pair alone");
  return HD_OK;
}

template <bool SPLIT>
int launch_chain(const ConvParams &p, const ConvParams &q, const hd_conv_desc *a, const hd_conv_desc *b, cudaStream_t st) {
  using C = ChainCfg<SPLIT>;
  static bool configured[kMaxDevices] = {};
  static int num_sms[kMaxDevices] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) { set_last_error_text("hd_conv_gemm_chain: device ordinal out of range"); return HD_ERR_UNSUPPORTED; }
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(conv_chain_tc_kernel<SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) { set_last_error("hd_conv_gemm_chain attr", e); return HD_ERR_CUDA; }
    cudaDeviceGetAttribute(&num_sms[dev], cudaDevAttrMultiProcessorCount, dev);
    if (num_sms[dev] <= 0) { set_last_error_text("hd_conv_gemm_chain: no multiprocessor count"); return HD_ERR_CUDA; }
    configured[dev] = true;
  }
  alignas(64) CUtensorMap w3h, w3l, w1h, w1l, tres, tout, r1h, r1l;
  memcpy(&w3h, a->tmap_hi, sizeof(CUtensorMap));
  memcpy(&w3l, SPLIT ? a->tmap_lo : a->tmap_hi, sizeof(CUtensorMap));
  memcpy(&w1h, b->tmap_hi, sizeof(CUtensorMap));
  memcpy(&w1l, SPLIT ? b->tmap_lo : b->tmap_hi, sizeof(CUtensorMap));
  memcpy(&tout, &w3h, sizeof(CUtensorMap));
  memcpy(&r1l, &w3h, sizeof(CUtensorMap));
  const int st32 = p.out_sub ? 0 : 1;
  int rc = encode_epilogue_map(&tres, false, p.res, p.Cout, p.M, p.res_ld * 4, "residual");
  if (rc == HD_OK && st32) rc = encode_epilogue_map(&tout, false, p.out, p.Cout, p.M, p.out_ld * 4, "output");
  if (rc == HD_OK) rc = encode_epilogue_map(&r1h, true, q.out_hi, q.Cout, q.M, q.out2_ld * 2, "second output head");
  if (rc == HD_OK && SPLIT) rc = encode_epilogue_map(&r1l, true, q.out_lo, q.Cout, q.M, q.out2_ld * 2, "second output remainder");
  if (rc != HD_OK) return rc;
  const int num_tiles = ceil_div(p.M, BM);
  dim3 grid(num_tiles < num_sms[dev] ? num_tiles : num_sms[dev]);
  conv_chain_tc_kernel<SPLIT><<<grid, C::NUM_THREADS, C::SMEM_BYTES, st>>>(p, q, w3h, w3l, w1h, w1l, tres, tout, r1h, r1l, st32);
  return check_launch("conv_chain_tc_kernel");
}

}  // namespace hd

extern "C" int hd_conv_gemm_chain_supported(const hd_conv_desc *first, const hd_conv_desc *second) {
  return hd::chain_check(first, second) == HD_OK ? 1 : 0;
}

extern "C" int hd_conv_gemm_chain(const hd_conv_desc *first, const hd_conv_desc *second, void *stream) {
  int rc = hd::chain_check(first, second);
  if (rc) return rc;
  hd::ConvParams p, q;
  if ((rc = hd::fill_params(first, p))) return rc;
  // the second conv's input is the first conv's pair, which never leaves the kernel: the first conv's input stands in for the
  // validation of fill_params (same rows, and the kernel never reads it)
  hd_conv_desc b = *second;
  b.in_hi = first->in_hi;
  b.in_lo = first->in_lo;
  if ((rc = hd::fill_params(&b, q))) return rc;
  if (!p.vec_out || !q.vec_out) {
    hd::set_last_error_text("hd_conv_gemm_chain: outputs and epilogue vectors must be 16-byte aligned");
    return HD_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  return first->impl == HD_IMPL_TC_3XF16 ? hd::launch_chain<true>(p, q, first, second, st) : hd::launch_chain<false>(p, q, first, second, st);
}

// K-major weight matrix [rows, k_pad] (fp32 for the tf32 path, fp16 for the fp16 path) -> CUtensorMap with a
// {128 bytes x box_rows} box and 128-byte swizzle.  box_rows must be 64: the kernel loads its 64- or 128-wide N tile as
// one or two such boxes.
extern "C" int hd_make_weight_tmap(const void *w_nk, int rows, int k_pad, int box_rows, int elem_bytes, void *tmap_out) {
  HD_REQUIRE(w_nk && tmap_out && rows > 0 && k_pad > 0 && (elem_bytes == 4 || elem_bytes == 2) && k_pad % (128 / elem_bytes) == 0 &&
                 box_rows == 64 && rows % box_rows == 0 && hd::aligned16(w_nk),
             "hd_make_weight_tmap: bad arguments");
  hd::EncodeTiledFn fn = hd::get_encode_fn();
  if (!fn) { hd::set_last_error_text("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return HD_ERR_UNSUPPORTED; }
  alignas(64) CUtensorMap tm;
  const cuuint64_t gdim[2] = {(cuuint64_t)k_pad, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)k_pad * (cuuint64_t)elem_bytes};
  const cuuint32_t box[2] = {(cuuint32_t)(128 / elem_bytes), (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(&tm, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(w_nk),
                  gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[96];
    snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    hd::set_last_error_text(msg);
    return HD_ERR_CUDA;
  }
  memcpy(tmap_out, &tm, sizeof(tm));
  return HD_OK;
}

// Row-major activation matrix [rows, cols] (leading dimension ld_elems; fp32 or fp16) -> CUtensorMap with a {32 columns x 128 rows}
// box: one 128-row x 32-column slab of the residual / outputs (the activation-map contract of hd_conv_desc).  fp32 slabs use the 128-byte swizzle, fp16 slabs the 64-byte one.
extern "C" int hd_make_act_tmap(const void *base, long long rows, int cols, long long ld_elems, int elem_bytes, void *tmap_out) {
  HD_REQUIRE(base && tmap_out && rows > 0 && cols > 0 && ld_elems >= cols && (elem_bytes == 4 || elem_bytes == 2) && hd::aligned16(base) &&
                 (ld_elems * elem_bytes) % 16 == 0,
             "hd_make_act_tmap: bad arguments (16-byte aligned base and row pitch required)");
  hd::EncodeTiledFn fn = hd::get_encode_fn();
  if (!fn) { hd::set_last_error_text("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return HD_ERR_UNSUPPORTED; }
  alignas(64) CUtensorMap tm;
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld_elems * (cuuint64_t)elem_bytes};
  const cuuint32_t box[2] = {32u, 128u};
  const cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(&tm, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(base), gdim,
                  gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, elem_bytes == 4 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[96];
    snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled (activation) failed with CUresult %d", (int)r);
    hd::set_last_error_text(msg);
    return HD_ERR_CUDA;
  }
  memcpy(tmap_out, &tm, sizeof(tm));
  return HD_OK;
}
