// Baseline JPEG decoding for sm_90a, bit for bit libjpeg's default decompression (oracle/jpeg_ref.py restates it):
//   hd_jpeg_parse          host C: markers and tables of one JPEG, every read bounds-checked;
//   jpeg_prep_kernel       one warp per image finds its restart markers (ballot over 32 bytes at a time) and checks its header
//                          against the call; extra blocks build each Huffman table's lookup (9-bit table + maxcode / valoffset);
//   jpeg_entropy_kernel    one thread per entropy-coded segment (an image, or one restart interval): sequential Huffman decoding,
//                          FF 00 unstuffing, dequantised int16 coefficients per block;
//   jpeg_idct_kernel       8 threads per 8x8 block: jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2) and its range-limit table;
//   jpeg_color_kernel      one thread per output pixel: fancy chroma upsampling (edges replicate the last real sample) and the
//                          jdcolor.c YCbCr -> RGB tables.
// Integer arithmetic only; each output byte depends only on its own image's data, so results do not depend on batching.
#include "common.cuh"

namespace {

constexpr int PREP_WARPS = 8;
constexpr int ENTROPY_THREADS = 32;
constexpr int IDCT_THREADS = 256;
constexpr int COLOR_THREADS = 256;
constexpr int LOOK_BITS = 9;

// T.81 Figure A.6 zig-zag -> natural order, with libjpeg's 16 guard entries for corrupt runs past k = 63
__constant__ unsigned char c_natural[80] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
    6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
    39, 46, 53, 60, 61, 54, 47, 55, 62, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};

struct DTable {                 // jdhuff.c's derived table, with a 9-bit lookahead
  unsigned short look[1 << LOOK_BITS];   // (length << 8) | symbol for codes of <= 9 bits, 0 otherwise
  int maxcode[18];              // largest code of each length, -1 if none; maxcode[17] is a sentinel
  int valoff[17];               // symbol index of a code of length l = valoff[l] + code
  unsigned char vals[256];
};

// The per-call geometry shared by the host entry and the kernels.
struct Geom {
  int N, H, W, hs, vs;
  int mcux, mcuy, n_mcu;
  int bwY, bhY, bwC, bhC;       // block grid of luma / each chroma component
  int bpi;                      // blocks per image
};

Geom make_geom(int N, int H, int W, int hs, int vs) {
  Geom g;
  g.N = N; g.H = H; g.W = W; g.hs = hs; g.vs = vs;
  g.mcux = (W + 8 * hs - 1) / (8 * hs);
  g.mcuy = (H + 8 * vs - 1) / (8 * vs);
  g.n_mcu = g.mcux * g.mcuy;
  g.bwY = g.mcux * hs; g.bhY = g.mcuy * vs;
  g.bwC = g.mcux; g.bhC = g.mcuy;
  g.bpi = g.bwY * g.bhY + 2 * g.bwC * g.bhC;
  return g;
}

struct Work {                   // workspace carve-up (256-byte aligned pieces)
  size_t coef, planes, seg, nseg, dtab, total;
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

Work carve(const Geom &g) {
  Work w;
  const size_t blocks = (size_t)g.N * g.bpi;
  w.coef = 0;
  w.planes = align256(w.coef + blocks * 64 * sizeof(short));
  w.seg = align256(w.planes + blocks * 64);
  w.nseg = align256(w.seg + (size_t)g.N * g.n_mcu * sizeof(int));
  w.dtab = align256(w.nseg + (size_t)g.N * sizeof(int));
  w.total = align256(w.dtab + (size_t)6 * g.N * sizeof(DTable));
  return w;
}

bool sampling_ok(int hs, int vs) { return (hs == 1 && vs == 1) || (hs == 2 && vs == 1) || (hs == 2 && vs == 2); }

constexpr long long MAX_INT = 0x7fffffffLL;

// The size contract of hd_jpeg_workspace_bytes / hd_jpeg_decode: pixel and byte offsets within one image fit in 32 bits
// (H * W <= 2^31 - 1), and every launch's grid fits in gridDim.x (N * H * W / 256, N * MCUs / 32 and N * blocks / 32 blocks).
bool size_ok(int N, int H, int W, int hs, int vs) {
  if (N < 1 || H < 1 || W < 1 || H > 65535 || W > 65535 || (long long)H * W > MAX_INT || !sampling_ok(hs, vs)) return false;
  const Geom g = make_geom(N, H, W, hs, vs);
  return ((long long)N * H * W + 255) / 256 <= MAX_INT && ((long long)N * g.n_mcu + 31) / 32 <= MAX_INT &&
         ((long long)N * g.bpi + 31) / 32 <= MAX_INT;
}

// ---------------------------------------------------------------------------------------------------------------- prep
__device__ void build_dtable(const hd_jpeg_huffman &h, DTable &t) {
  for (int i = 0; i < (1 << LOOK_BITS); ++i) t.look[i] = 0;
  for (int i = 0; i < 256; ++i) t.vals[i] = h.vals[i];
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    const int n = h.bits[l - 1];
    t.valoff[l] = k - code;
    for (int j = 0; j < n; ++j, ++k, ++code) {
      if (l <= LOOK_BITS && k < 256) {
        const int lo = code << (LOOK_BITS - l), cnt = 1 << (LOOK_BITS - l);
        for (int x = 0; x < cnt && lo + x < (1 << LOOK_BITS); ++x) t.look[lo + x] = (unsigned short)((l << 8) | h.vals[k]);
      }
    }
    t.maxcode[l] = n ? code - 1 : -1;
    code <<= 1;
  }
  t.maxcode[17] = 0x7fffffff;
  t.maxcode[0] = -1;
  t.valoff[0] = 0;
}

__global__ void jpeg_prep_kernel(const unsigned char *__restrict__ data, long long data_size, const hd_jpeg_header *__restrict__ hdrs,
                                 Geom g, int n_quant, const hd_jpeg_huffman *__restrict__ huff, int n_huff, int *__restrict__ seg_off,
                                 int *__restrict__ nseg, DTable *__restrict__ dtab, int *__restrict__ status, int img_blocks) {
  if ((int)blockIdx.x >= img_blocks) {               // Huffman lookup tables
    const int t = (blockIdx.x - img_blocks) * blockDim.x + threadIdx.x;
    if (t < n_huff) build_dtable(huff[t], dtab[t]);
    return;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int img = blockIdx.x * PREP_WARPS + warp;
  if (img >= g.N) return;
  const hd_jpeg_header h = hdrs[img];
  bool ok = h.width == g.W && h.height == g.H && h.h_samp == g.hs && h.v_samp == g.vs && h.restart_interval >= 0 &&
            h.data_offset >= 0 && h.data_bytes >= 0 && h.data_bytes <= MAX_INT && h.data_offset <= data_size &&
            h.data_bytes <= data_size - h.data_offset;
  for (int c = 0; c < 3; ++c)
    ok = ok && h.qt[c] >= 0 && h.qt[c] < n_quant && h.dc[c] >= 0 && h.dc[c] < n_huff && h.ac[c] >= 0 && h.ac[c] < n_huff;
  if (!ok) {
    if (lane == 0) { status[img] = HD_JPEG_BAD_HEADER; nseg[img] = 0; }
    return;
  }
  const int ri = h.restart_interval ? h.restart_interval : g.n_mcu;
  const int want = (g.n_mcu + ri - 1) / ri;
  int *off = seg_off + (size_t)img * g.n_mcu;
  const unsigned char *p = data + h.data_offset;
  const long long n = h.data_bytes;
  int count = 0;                                     // restart markers found so far
  if (want > 1) {
    for (long long base = 0; base < n; base += 32) {
      const long long i = base + lane;
      bool m = false;
      if (i + 1 < n && p[i] == 0xFF) {
        const unsigned char b = p[i + 1];
        m = b >= 0xD0 && b <= 0xD7;
      }
      const unsigned mask = __ballot_sync(0xffffffffu, m);
      if (m) {
        const int k = count + __popc(mask & ((1u << lane) - 1));      // 0-based marker ordinal: segment k + 1 starts after it
        if (k + 1 < want) off[k + 1] = (int)(i + 2);
      }
      count += __popc(mask);
    }
  }
  if (lane == 0) {
    off[0] = 0;
    nseg[img] = count + 1;
    status[img] = count + 1 == want ? 0 : HD_JPEG_MARKER;
  }
}

// ---------------------------------------------------------------------------------------------------------------- entropy
struct BitReader {
  const unsigned char *p, *end;
  unsigned long long buf;       // left-aligned
  int n;                        // valid bits in buf
  int phantom;                  // zero bytes appended past the segment
  int flags;

  __device__ __forceinline__ void fill() {
    while (n <= 56) {
      unsigned b = 0;
      if (p < end) {
        b = *p++;
        if (b == 0xFF) {
          if (p < end && *p == 0) {
            ++p;
          } else {                                   // a marker inside the segment: the data stops here
            flags |= HD_JPEG_MARKER;
            p = end;
            b = 0;
            ++phantom;
          }
        }
      } else {
        ++phantom;
      }
      buf |= (unsigned long long)b << (56 - n);
      n += 8;
    }
  }
  __device__ __forceinline__ unsigned get(int k) {               // k <= 16, needs n >= k
    if (k == 0) return 0;
    const unsigned v = (unsigned)(buf >> (64 - k));
    buf <<= k;
    n -= k;
    return v;
  }
};

// One Huffman symbol, or -1 for a bit pattern that starts no code.  Needs n >= 16.
__device__ __forceinline__ int decode_symbol(BitReader &br, const DTable &t) {
  const unsigned peek = (unsigned)(br.buf >> 48);
  const unsigned e = t.look[peek >> (16 - LOOK_BITS)];
  if (e >> 8) {
    br.get(e >> 8);
    return e & 255;
  }
#pragma unroll 1
  for (int l = LOOK_BITS + 1; l <= 16; ++l) {
    const int code = (int)(peek >> (16 - l));
    if (code <= t.maxcode[l]) {
      br.get(l);
      return t.vals[(t.valoff[l] + code) & 255];
    }
  }
  return -1;
}

__device__ __forceinline__ int extend(unsigned v, int s) { return (s && v < (1u << (s - 1))) ? (int)v - (1 << s) + 1 : (int)v; }

__global__ void __launch_bounds__(ENTROPY_THREADS, 16)
jpeg_entropy_kernel(const unsigned char *__restrict__ data, const hd_jpeg_header *__restrict__ hdrs, Geom g,
                    const unsigned short *__restrict__ quant, const DTable *__restrict__ dtab, const int *__restrict__ seg_off,
                    const int *__restrict__ nseg, short *__restrict__ coef, int *__restrict__ status) {
  __shared__ __align__(16) short blk[ENTROPY_THREADS][64];
  const long long t = (long long)blockIdx.x * ENTROPY_THREADS + threadIdx.x;
  const int img = (int)(t / g.n_mcu), seg = (int)(t % g.n_mcu);
  if (img >= g.N) return;
  const hd_jpeg_header h = hdrs[img];
  const int found = nseg[img];
  const int ri = h.restart_interval > 0 ? h.restart_interval : g.n_mcu;
  const int want = (g.n_mcu + ri - 1) / ri;
  if (found == 0 ? seg != 0 : seg >= want) return;   // found == 0: a bad header, its one thread zeroes the whole image
  const int m0 = found == 0 ? 0 : seg * ri;
  const int m1 = found == 0 ? g.n_mcu : min(g.n_mcu, m0 + ri);
  bool live = found > 0 && seg < found;
  int flags = 0;
  BitReader br;
  br.buf = 0; br.n = 0; br.phantom = 0; br.flags = 0;
  br.p = br.end = data;
  if (live) {
    const int *off = seg_off + (size_t)img * g.n_mcu;
    const long long s = off[seg];
    long long e = seg + 1 < min(found, want) ? off[seg + 1] - 2 : h.data_bytes;
    const unsigned char *base = data + h.data_offset;
    while (e > s && base[e - 1] == 0xFF) --e;          // fill bytes before the RST marker (T.81 B.1.1.2); data FFs are stuffed
    if (seg > 0 && base[s - 1] != 0xD0 + ((seg - 1) & 7)) flags |= HD_JPEG_MARKER;
    br.p = base + s;
    br.end = base + max(e, s);
    br.fill();
  } else if (found > 0) {
    flags |= HD_JPEG_MARKER;                         // missing restart markers: status already says so; the blocks are zeroed
  }
  // per-component state in registers (selected by component, not indexed, so nothing lives on the stack)
  const int dc0 = live ? h.dc[0] : 0, dc1 = live ? h.dc[1] : 0, dc2 = live ? h.dc[2] : 0;
  const int ac0 = live ? h.ac[0] : 0, ac1 = live ? h.ac[1] : 0, ac2 = live ? h.ac[2] : 0;
  const int qt0 = live ? h.qt[0] : 0, qt1 = live ? h.qt[1] : 0, qt2 = live ? h.qt[2] : 0;
  int pred0 = 0, pred1 = 0, pred2 = 0;
  short *cimg = coef + (size_t)img * g.bpi * 64;
  const int nY = g.bwY * g.bhY, nC = g.bwC * g.bhC;
  const int per_mcu = g.hs * g.vs + 2;
  short *b = blk[threadIdx.x];
#pragma unroll 1
  for (int m = m0; m < m1; ++m) {
    const int my = m / g.mcux, mx = m - my * g.mcux;
#pragma unroll 1
    for (int j = 0; j < per_mcu; ++j) {
      const int nl = g.hs * g.vs;
      const int c = j < nl ? 0 : j - nl + 1;
      size_t bi;
      if (c == 0) {
        const int yy = j / g.hs, xx = j - yy * g.hs;
        bi = (size_t)(my * g.vs + yy) * g.bwY + mx * g.hs + xx;
      } else {
        bi = (size_t)nY + (size_t)(c - 1) * nC + (size_t)my * g.bwC + mx;
      }
      uint4 *b4 = reinterpret_cast<uint4 *>(b);
#pragma unroll
      for (int i = 0; i < 8; ++i) b4[i] = make_uint4(0, 0, 0, 0);
      if (live) {
        const DTable &dt = dtab[c == 0 ? dc0 : c == 1 ? dc1 : dc2], &at = dtab[c == 0 ? ac0 : c == 1 ? ac1 : ac2];
        const unsigned short *q = quant + 64 * (c == 0 ? qt0 : c == 1 ? qt1 : qt2);
        if (br.n < 32) br.fill();
        const int sdc = decode_symbol(br, dt);
        if (sdc < 0 || sdc > 15) {
          flags |= HD_JPEG_BAD_CODE;
          live = false;
        } else {
          const int dc = (c == 0 ? pred0 : c == 1 ? pred1 : pred2) + extend(br.get(sdc), sdc);
          if (c == 0) pred0 = dc;
          else if (c == 1) pred1 = dc;
          else pred2 = dc;
          b[0] = (short)((short)dc * (int)q[0]);
#pragma unroll 1
          for (int k = 1; k < 64; ++k) {
            if (br.n < 32) br.fill();
            const int rs = decode_symbol(br, at);
            if (rs < 0) {
              flags |= HD_JPEG_BAD_CODE;
              live = false;
              break;
            }
            const int r = rs >> 4, sz = rs & 15;
            if (sz) {
              k += r;
              const int z = c_natural[k];
              b[z] = (short)(extend(br.get(sz), sz) * (int)q[z]);
            } else {
              if (r != 15) break;
              k += 15;
            }
          }
          if (!live) {
#pragma unroll
            for (int i = 0; i < 8; ++i) b4[i] = make_uint4(0, 0, 0, 0);
          }
        }
      }
      uint4 *dst = reinterpret_cast<uint4 *>(cimg + bi * 64);
#pragma unroll
      for (int i = 0; i < 8; ++i) dst[i] = b4[i];
    }
  }
  if (live && br.phantom * 8 > br.n) flags |= HD_JPEG_OVERRUN;
  flags |= br.flags;
  if (flags) atomicOr(status + img, flags);
}

// ---------------------------------------------------------------------------------------------------------------- IDCT
constexpr int FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433, FIX_0_765366865 = 6270;
constexpr int FIX_0_899976223 = 7373, FIX_1_175875602 = 9633, FIX_1_501321110 = 12299, FIX_1_847759065 = 15137;
constexpr int FIX_1_961570560 = 16069, FIX_2_053119869 = 16819, FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;
constexpr int CONST_BITS = 13, PASS1_BITS = 2;

// jpeg_idct_islow's butterflies on one column or row; o[k] before descaling.
__device__ __forceinline__ void idct_1d(const int (&s)[8], int (&o)[8]) {
  int z1 = (s[2] + s[6]) * FIX_0_541196100;
  const int tmp2 = z1 + s[6] * -FIX_1_847759065;
  const int tmp3 = z1 + s[2] * FIX_0_765366865;
  const int tmp0 = (s[0] + s[4]) * (1 << CONST_BITS);
  const int tmp1 = (s[0] - s[4]) * (1 << CONST_BITS);
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  int t0 = s[7], t1 = s[5], t2 = s[3], t3 = s[1];
  z1 = t0 + t3;
  int z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
  const int z5 = (z3 + z4) * FIX_1_175875602;
  t0 *= FIX_0_298631336; t1 *= FIX_2_053119869; t2 *= FIX_3_072711026; t3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447;
  z3 = z3 * -FIX_1_961570560 + z5;
  z4 = z4 * -FIX_0_390180644 + z5;
  t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
  o[0] = tmp10 + t3; o[7] = tmp10 - t3; o[1] = tmp11 + t2; o[6] = tmp11 - t2;
  o[2] = tmp12 + t1; o[5] = tmp12 - t1; o[3] = tmp13 + t0; o[4] = tmp13 - t0;
}

// range_limit[x & RANGE_MASK] with range_limit = sample_range_limit + CENTERJSAMPLE (jdmaster.c prepare_range_limit_table)
__device__ __forceinline__ unsigned idct_limit(int x) {
  const unsigned u = (unsigned)(x + 128) & 1023u;
  return u < 256 ? u : (u < 640 ? 255u : 0u);
}

__global__ void __launch_bounds__(IDCT_THREADS)
jpeg_idct_kernel(const short *__restrict__ coef, Geom g, unsigned char *__restrict__ planes, long long n_blocks) {
  constexpr int G = IDCT_THREADS / 8;
  __shared__ __align__(16) short cb[G][64];
  __shared__ int ws[G][8][9];
  const int grp = threadIdx.x >> 3, l = threadIdx.x & 7;
  const long long blk = (long long)blockIdx.x * G + grp;
  const bool on = blk < n_blocks;
  if (on) reinterpret_cast<uint4 *>(cb[grp])[l] = reinterpret_cast<const uint4 *>(coef + blk * 64)[l];
  __syncthreads();
  int s[8], o[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) s[r] = cb[grp][r * 8 + l];         // pass 1: column l
  idct_1d(s, o);
  constexpr int D1 = CONST_BITS - PASS1_BITS;
#pragma unroll
  for (int r = 0; r < 8; ++r) ws[grp][r][l] = (o[r] + (1 << (D1 - 1))) >> D1;
  __syncthreads();
  if (!on) return;
#pragma unroll
  for (int c = 0; c < 8; ++c) s[c] = ws[grp][l][c];               // pass 2: row l
  idct_1d(s, o);
  constexpr int D2 = CONST_BITS + PASS1_BITS + 3;
  unsigned lo = 0, hi = 0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    lo |= idct_limit((o[c] + (1 << (D2 - 1))) >> D2) << (8 * c);
    hi |= idct_limit((o[c + 4] + (1 << (D2 - 1))) >> D2) << (8 * c);
  }
  const int img = (int)(blk / g.bpi);
  int b = (int)(blk - (long long)img * g.bpi);
  const int nY = g.bwY * g.bhY, nC = g.bwC * g.bhC;
  int bw = g.bwY, first = 0;
  if (b >= nY) {
    first = nY + ((b - nY) / nC) * nC;
    bw = g.bwC;
  }
  const int local = b - first, by = local / bw, bx = local - by * bw;
  unsigned char *plane = planes + ((size_t)img * g.bpi + first) * 64;
  *reinterpret_cast<uint2 *>(plane + (size_t)(by * 8 + l) * (bw * 8) + bx * 8) = make_uint2(lo, hi);
}

// ---------------------------------------------------------------------------------------------------------------- colour
__device__ __forceinline__ int px(const unsigned char *p, int stride, int y, int x) { return p[(size_t)y * stride + x]; }

// One chroma sample of the output pixel (y, x): jdsample.c's fancy upsampling, or plain replication where the downsampled width <= 2.
__device__ __forceinline__ int chroma(const unsigned char *p, int stride, const Geom &g, int y, int x) {
  if (g.hs == 1) return px(p, stride, y, x);
  const int dw = (g.W + 1) >> 1, i = x >> 1;
  const bool even = !(x & 1);
  const int j = even ? max(i - 1, 0) : min(i + 1, dw - 1);
  if (g.vs == 1) {
    if (dw <= 2) return px(p, stride, y, i);
    return (3 * px(p, stride, y, i) + px(p, stride, y, j) + (even ? 1 : 2)) >> 2;
  }
  const int dh = (g.H + 1) >> 1, r = y >> 1;
  if (dw <= 2) return px(p, stride, r, i);
  const int far = (y & 1) ? min(r + 1, dh - 1) : max(r - 1, 0);
  const int csi = 3 * px(p, stride, r, i) + px(p, stride, far, i);
  const int csj = 3 * px(p, stride, r, j) + px(p, stride, far, j);
  return (3 * csi + csj + (even ? 8 : 7)) >> 4;
}

__device__ __forceinline__ unsigned char clamp255(int v) { return (unsigned char)min(max(v, 0), 255); }

__global__ void __launch_bounds__(COLOR_THREADS)
jpeg_color_kernel(const unsigned char *__restrict__ planes, Geom g, unsigned char *__restrict__ out) {
  const long long t = (long long)blockIdx.x * COLOR_THREADS + threadIdx.x;
  const long long hw = (long long)g.H * g.W;
  if (t >= hw * g.N) return;
  const int img = (int)(t / hw);
  const long long rem = t - img * hw;
  const int y = (int)(rem / g.W), x = (int)(rem - (long long)y * g.W);
  const unsigned char *pY = planes + (size_t)img * g.bpi * 64;
  const unsigned char *pCb = pY + (size_t)g.bwY * g.bhY * 64;
  const unsigned char *pCr = pCb + (size_t)g.bwC * g.bhC * 64;
  const int Y = px(pY, g.bwY * 8, y, x);
  const int cb = chroma(pCb, g.bwC * 8, g, y, x) - 128, cr = chroma(pCr, g.bwC * 8, g, y, x) - 128;
  // jdcolor.c build_ycc_rgb_table: FIX(x) = x * 2^16 rounded, ONE_HALF = 2^15
  const int r = Y + ((91881 * cr + 32768) >> 16);
  const int gg = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int b = Y + ((116130 * cb + 32768) >> 16);
  unsigned char *o = out + t * 3;
  o[0] = clamp255(r);
  o[1] = clamp255(gg);
  o[2] = clamp255(b);
}

// ---------------------------------------------------------------------------------------------------------------- host parse
struct Reader {
  const uint8_t *d;
  size_t n;
  int u16(size_t at) const { return (d[at] << 8) | d[at + 1]; }
};

int fail(int code, const char *msg) {
  hd::set_last_error_text(msg);
  return code;
}

// jdhuff.c jpeg_make_d_derived_tbl's checks: the code lengths fit (no length l reaches 2^l codes), DC symbols <= 15.
bool huffman_ok(const hd_jpeg_huffman &h, int count, bool dc) {
  long code = 0;
  for (int l = 1; l <= 16; ++l) {
    code += h.bits[l - 1];
    if (code > (1L << l)) return false;
    code <<= 1;
  }
  if (dc)
    for (int i = 0; i < count; ++i)
      if (h.vals[i] > 15) return false;
  return true;
}

}  // namespace

extern "C" {

int hd_jpeg_parse(const uint8_t *data, size_t len, hd_jpeg_header *hdr, hd_jpeg_tables *tables) {
  HD_REQUIRE(data && hdr && tables, "hd_jpeg_parse: null pointer");
  memset(hdr, 0, sizeof(*hdr));
  memset(tables, 0, sizeof(*tables));
  const Reader R{data, len};
  if (len < 4 || data[0] != 0xFF || data[1] != 0xD8) return fail(HD_ERR_INVALID, "hd_jpeg_parse: no SOI marker");
  size_t pos = 2;
  bool have_frame = false;
  int ids[3] = {0, 0, 0};
  int adobe_transform = -1;
  for (;;) {
    while (pos + 1 < len && data[pos] == 0xFF && data[pos + 1] == 0xFF) ++pos;      // fill bytes
    if (pos + 4 > len || data[pos] != 0xFF) return fail(HD_ERR_INVALID, "hd_jpeg_parse: truncated stream or a bad marker");
    const int m = data[pos + 1];
    const size_t seg_len = (size_t)R.u16(pos + 2);
    const size_t body = pos + 4, end = pos + 2 + seg_len;
    if (seg_len < 2 || end > len) return fail(HD_ERR_INVALID, "hd_jpeg_parse: truncated marker segment");
    const size_t sn = end - body;
    const uint8_t *s = data + body;
    if (m == 0xC0 || m == 0xC1) {
      if (have_frame) return fail(HD_ERR_INVALID, "hd_jpeg_parse: second SOF");
      if (sn < 6) return fail(HD_ERR_INVALID, "hd_jpeg_parse: short SOF");
      const int nc = s[5];
      if (sn < 6 + 3 * (size_t)nc) return fail(HD_ERR_INVALID, "hd_jpeg_parse: short SOF");
      if (s[0] != 8 || nc != 3) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: precision other than 8 or other than 3 components");
      hdr->height = (s[1] << 8) | s[2];
      hdr->width = (s[3] << 8) | s[4];
      if (hdr->height == 0 || hdr->width == 0) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: DNL height or zero width");
      if ((long long)hdr->height * hdr->width > MAX_INT) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: more than 2^31 - 1 pixels");
      hdr->h_samp = s[7] >> 4;
      hdr->v_samp = s[7] & 15;
      for (int c = 0; c < 3; ++c) {
        ids[c] = s[6 + 3 * c];
        if (c > 0 && s[7 + 3 * c] != 0x11) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: chroma sampling other than 1x1");
        if (s[8 + 3 * c] > 3) return fail(HD_ERR_INVALID, "hd_jpeg_parse: quantisation table id > 3");
        hdr->qt[c] = s[8 + 3 * c];
      }
      if (!sampling_ok(hdr->h_samp, hdr->v_samp)) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: luma sampling not 1x1, 2x1 or 2x2");
      if (ids[0] == 'R' && ids[1] == 'G' && ids[2] == 'B') return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: RGB components");
      have_frame = true;
    } else if ((m >= 0xC2 && m <= 0xCF) && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: progressive, lossless or arithmetic coding");
    } else if (m == 0xCC) {
      return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: arithmetic coding");
    } else if (m == 0xC4) {
      size_t p = 0;
      while (p < sn) {
        if (p + 17 > sn) return fail(HD_ERR_INVALID, "hd_jpeg_parse: short DHT");
        const int tc = s[p] >> 4, th = s[p] & 15;
        int cnt = 0;
        for (int i = 0; i < 16; ++i) cnt += s[p + 1 + i];
        if (tc > 1 || th > 3 || cnt > 256 || p + 17 + cnt > sn) return fail(HD_ERR_INVALID, "hd_jpeg_parse: bad DHT");
        hd_jpeg_huffman &h = tc == 0 ? tables->dc[th] : tables->ac[th];
        memset(&h, 0, sizeof(h));
        memcpy(h.bits, s + p + 1, 16);
        memcpy(h.vals, s + p + 17, cnt);
        if (!huffman_ok(h, cnt, tc == 0)) return fail(HD_ERR_INVALID, "hd_jpeg_parse: bad Huffman table");
        (tc == 0 ? tables->dc_defined : tables->ac_defined) |= 1 << th;
        p += 17 + cnt;
      }
    } else if (m == 0xDB) {
      size_t p = 0;
      while (p < sn) {
        const int pq = s[p] >> 4, tq = s[p] & 15;
        const size_t size = 64 * (pq + 1);
        if (pq > 1 || tq > 3 || p + 1 + size > sn) return fail(HD_ERR_INVALID, "hd_jpeg_parse: bad DQT");
        for (int k = 0; k < 64; ++k) {
          static const unsigned char zz[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                               41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                               30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
          tables->quant[tq][zz[k]] = (uint16_t)(pq ? R.u16(body + p + 1 + 2 * k) : s[p + 1 + k]);
        }
        tables->quant_defined |= 1 << tq;
        p += 1 + size;
      }
    } else if (m == 0xDD) {
      if (sn < 2) return fail(HD_ERR_INVALID, "hd_jpeg_parse: short DRI");
      hdr->restart_interval = (s[0] << 8) | s[1];
    } else if (m == 0xEE) {
      if (sn >= 12 && memcmp(s, "Adobe", 5) == 0) adobe_transform = s[11];
    } else if (m == 0xDA) {
      if (!have_frame) return fail(HD_ERR_INVALID, "hd_jpeg_parse: SOS before SOF");
      const int ns = sn ? s[0] : 0;
      if (ns != 3) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: a scan without all three components");
      if (sn < 1 + 2 * 3 + 3) return fail(HD_ERR_INVALID, "hd_jpeg_parse: short SOS");
      for (int c = 0; c < 3; ++c) {
        if (s[1 + 2 * c] != ids[c]) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: scan components out of frame order");
        hdr->dc[c] = s[2 + 2 * c] >> 4;
        hdr->ac[c] = s[2 + 2 * c] & 15;
        if (hdr->dc[c] > 3 || hdr->ac[c] > 3 || !(tables->dc_defined >> hdr->dc[c] & 1) || !(tables->ac_defined >> hdr->ac[c] & 1) ||
            !(tables->quant_defined >> hdr->qt[c] & 1))
          return fail(HD_ERR_INVALID, "hd_jpeg_parse: the scan uses an undefined table");
      }
      if (s[7] != 0 || s[8] != 63 || s[9] != 0) return fail(HD_ERR_INVALID, "hd_jpeg_parse: spectral selection in a sequential scan");
      if (adobe_transform == 0) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: Adobe RGB");
      size_t q = end;
      for (;;) {                                     // the scan ends at the first marker other than RSTn
        const void *f = q < len ? memchr(data + q, 0xFF, len - q) : NULL;
        if (!f) return fail(HD_ERR_INVALID, "hd_jpeg_parse: entropy-coded data runs to the end of the stream");
        q = (size_t)((const uint8_t *)f - data);
        if (q + 1 >= len) return fail(HD_ERR_INVALID, "hd_jpeg_parse: entropy-coded data runs to the end of the stream");
        const int nx = data[q + 1];
        if (nx == 0x00 || (nx >= 0xD0 && nx <= 0xD7)) q += 2;
        else if (nx == 0xFF) q += 1;
        else break;
      }
      if (data[q + 1] != 0xD9) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: more than one scan");
      size_t stop = q;                               // fill bytes before EOI are not data (a data FF is always stuffed)
      while (stop > end && data[stop - 1] == 0xFF) --stop;
      if (stop - end > (size_t)MAX_INT) return fail(HD_ERR_UNSUPPORTED, "hd_jpeg_parse: more than 2^31 - 1 bytes of entropy-coded data");
      hdr->data_offset = (long long)end;
      hdr->data_bytes = (long long)(stop - end);
      return HD_OK;
    } else if (m == 0xD9) {
      return fail(HD_ERR_INVALID, "hd_jpeg_parse: EOI before SOS");
    } else if ((m >= 0xD0 && m <= 0xD8) || m == 0x01 || m == 0x00) {
      return fail(HD_ERR_INVALID, "hd_jpeg_parse: a marker out of place");
    }
    pos = end;
  }
}

size_t hd_jpeg_workspace_bytes(int N, int H, int W, int h_samp, int v_samp) {
  if (!size_ok(N, H, W, h_samp, v_samp)) return 0;
  return carve(make_geom(N, H, W, h_samp, v_samp)).total;
}

int hd_jpeg_decode(const uint8_t *data, long long data_size, const hd_jpeg_header *hdrs, int N, int H, int W, int h_samp, int v_samp,
                   const uint16_t *quant, int n_quant, const hd_jpeg_huffman *huff, int n_huff, uint8_t *out, int *status,
                   void *workspace, size_t workspace_bytes, void *stream) {
  HD_REQUIRE(data && hdrs && quant && huff && out && status && workspace, "hd_jpeg_decode: null pointer");
  HD_REQUIRE(N >= 1 && H >= 1 && W >= 1 && H <= 65535 && W <= 65535 && data_size >= 0, "hd_jpeg_decode: N < 1 or H, W outside [1, 65535]");
  HD_REQUIRE(sampling_ok(h_samp, v_samp), "hd_jpeg_decode: luma sampling must be 1x1, 2x1 or 2x2");
  HD_REQUIRE((long long)H * W <= MAX_INT, "hd_jpeg_decode: H * W > 2^31 - 1");
  HD_REQUIRE(size_ok(N, H, W, h_samp, v_samp), "hd_jpeg_decode: N too large for one call (a grid would exceed 2^31 - 1 blocks)");
  HD_REQUIRE(n_quant >= 1 && n_huff >= 1 && (long long)n_huff <= 6LL * N, "hd_jpeg_decode: n_quant < 1 or n_huff outside [1, 6N]");
  HD_REQUIRE(((uintptr_t)workspace & 255) == 0, "hd_jpeg_decode: workspace not 256-byte aligned");
  const Geom g = make_geom(N, H, W, h_samp, v_samp);
  const Work w = carve(g);
  HD_REQUIRE(workspace_bytes >= w.total, "hd_jpeg_decode: workspace smaller than hd_jpeg_workspace_bytes");
  char *ws = static_cast<char *>(workspace);
  short *coef = reinterpret_cast<short *>(ws + w.coef);
  unsigned char *planes = reinterpret_cast<unsigned char *>(ws + w.planes);
  int *seg_off = reinterpret_cast<int *>(ws + w.seg);
  int *nseg = reinterpret_cast<int *>(ws + w.nseg);
  DTable *dtab = reinterpret_cast<DTable *>(ws + w.dtab);
  cudaStream_t st = (cudaStream_t)stream;

  const int img_blocks = hd::ceil_div(N, PREP_WARPS);
  jpeg_prep_kernel<<<img_blocks + hd::ceil_div(n_huff, 32 * PREP_WARPS), 32 * PREP_WARPS, 0, st>>>(
      data, data_size, hdrs, g, n_quant, huff, n_huff, seg_off, nseg, dtab, status, img_blocks);
  int rc = hd::check_launch("jpeg_prep_kernel");
  if (rc) return rc;
  jpeg_entropy_kernel<<<hd::ceil_div((long long)N * g.n_mcu, ENTROPY_THREADS), ENTROPY_THREADS, 0, st>>>(
      data, hdrs, g, quant, dtab, seg_off, nseg, coef, status);
  if ((rc = hd::check_launch("jpeg_entropy_kernel"))) return rc;
  const long long n_blocks = (long long)N * g.bpi;
  jpeg_idct_kernel<<<hd::ceil_div(n_blocks, IDCT_THREADS / 8), IDCT_THREADS, 0, st>>>(coef, g, planes, n_blocks);
  if ((rc = hd::check_launch("jpeg_idct_kernel"))) return rc;
  jpeg_color_kernel<<<hd::ceil_div((long long)N * H * W, COLOR_THREADS), COLOR_THREADS, 0, st>>>(planes, g, out);
  return hd::check_launch("jpeg_color_kernel");
}

}  // extern "C"
