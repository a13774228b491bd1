// Network-level entry points (SURVEY.md 8b): slim resnet_v2_50, f_movie and the IEF regressor as library-owned layer plans.
//
// Host-only code.  A plan packs the TF-named weights once (BatchNorm folded in double precision, K-major fp16 head / 2^11-scaled
// remainder written on the device by hd_pack_weight, TMA descriptors), owns its activation buffers, and `*_forward` is a fixed
// sequence of the per-layer entries of this library (hd_conv_gemm and friends) on the caller's stream: no allocation, no
// synchronisation.  The sequence, buffers and descriptors are the same as the Python host plans (human_dynamics_b200/nets.py:
// ResNetPlan in split mode, FMoviePlan / IEFPlan fast paths), so the results are bit-identical to them (tests/test_gpu_cplan.py).
//
// Reference functions replaced (graph-building Python + sess.run in the reference):
//   hd_resnet50_forward  encoder_resnet            src/models.py:50-77  (slim resnet_v2_50 [TF-ext], global pool, squeeze)
//   hd_fmovie_forward    az_fc2_groupnorm          src/models.py:121-228
//   hd_ief_forward       call_hmr_ief / hmr_ief    src/models.py:299-415 (+ encoder_fc3_dropout :80-116), use_optcam=True,
//                                                   use_delta_from_pred=True as wired by tester.py:196-207
#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <deque>
#include <functional>
#include <string>
#include <utility>
#include <vector>

struct hd_net {
  int kind = 0;                                   // 1 resnet, 2 f_movie, 3 ief
  hd_weight_fn get = nullptr;
  void *user = nullptr;
  std::vector<void *> allocs;                     // cudaMalloc'd, freed by hd_net_destroy
  std::deque<std::vector<unsigned char>> wmaps;   // 128-byte CUtensorMap blobs of the weights (stable addresses)
  std::deque<std::vector<unsigned char>> maps;    // ... of the activations (f_movie re-encodes them when the caller's pointers change)
  std::vector<std::function<int(cudaStream_t)>> steps;
  std::string err;
  // run-time pointers read by the step closures
  const float *in0 = nullptr;
  float *out0 = nullptr, *out1 = nullptr;
  // geometry
  int n = 0, size = 0, B = 0, T = 0, C = 0, layers = 0, N = 0, D = 0;
  // f_movie: descriptors depend on the caller's pointers -> rebuilt when they change
  const float *bound_in = nullptr;
  float *bound_out = nullptr;
  std::vector<void *> persist;                    // f_movie / ief device buffers referenced on rebuild
  std::vector<int> delta_t;
  float *theta0 = nullptr;                        // ief: mean_param tiled [N,85]
};

namespace {

using hd::set_last_error_text;

struct Pair { void *hi = nullptr, *lo = nullptr; };

struct PackedConv {                               // nets.py PackedConv (fp16 tensor-core packing) / PackedConv1Planes
  int KH = 1, KW = 1, Cin = 0, Cout = 0, K = 0, K_pad = 0, stride = 1, pad_t = 0, pad_l = 0;
  float *w_kn = nullptr;
  void *w_hi = nullptr, *w_lo = nullptr;
  float *post_scale = nullptr, *post_shift = nullptr;
  int post_relu = 0;
  void *tmap_hi = nullptr, *tmap_lo = nullptr;
};

struct Builder {
  hd_net *net;
  int rc = HD_OK;

  bool fail(int code, const std::string &msg) {
    if (rc == HD_OK) { rc = code; net->err = msg; set_last_error_text(msg.c_str()); }
    return false;
  }

  const float *weight(const std::string &name, long long expect) {
    long long numel = -1;
    const float *p = net->get ? net->get(net->user, name.c_str(), &numel) : nullptr;
    if (!p) { fail(HD_ERR_INVALID, "weight '" + name + "' not provided"); return nullptr; }
    if (numel != expect) {
      fail(HD_ERR_INVALID, "weight '" + name + "' has " + std::to_string(numel) + " elements, expected " + std::to_string(expect));
      return nullptr;
    }
    return p;
  }

  void *dev_alloc(size_t bytes, bool zero = false) {
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes ? bytes : 16);
    if (e != cudaSuccess) { hd::set_last_error("cudaMalloc", e); rc = rc ? rc : HD_ERR_CUDA; return nullptr; }
    net->allocs.push_back(p);
    if (zero && cudaMemset(p, 0, bytes) != cudaSuccess) { fail(HD_ERR_CUDA, "cudaMemset failed"); return nullptr; }
    return p;
  }

  template <typename Tv>
  void *upload(const std::vector<Tv> &v) {
    void *p = dev_alloc(v.size() * sizeof(Tv));
    if (!p) return nullptr;
    cudaError_t e = cudaMemcpy(p, v.data(), v.size() * sizeof(Tv), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { hd::set_last_error("cudaMemcpy(H2D)", e); rc = rc ? rc : HD_ERR_CUDA; return nullptr; }
    return p;
  }

  Pair pair(size_t count) { return Pair{dev_alloc(count * 2), dev_alloc(count * 2)}; }

  void *new_map(bool weight = false) {
    auto &q = weight ? net->wmaps : net->maps;
    q.emplace_back(128);
    return q.back().data();
  }

  // fold_bn (nets.py): s = gamma / sqrt(var + eps), shift = beta - mean * s, evaluated in double, stored as float
  bool fold_bn(const std::string &prefix, int C, std::vector<float> &s, std::vector<float> &b) {
    const float *g = weight(prefix + "/gamma", C), *be = weight(prefix + "/beta", C);
    const float *m = weight(prefix + "/moving_mean", C), *v = weight(prefix + "/moving_variance", C);
    if (!g || !be || !m || !v) return false;
    s.resize(C); b.resize(C);
    for (int c = 0; c < C; ++c) {
      const double sd = (double)g[c] / std::sqrt((double)v[c] + 1e-5);
      s[c] = (float)sd;
      b[c] = (float)((double)be[c] - (double)m[c] * sd);
    }
    return true;
  }

  // K-major [roundup64(Cout), K_pad] fp16 head / 2^11-scaled remainder of the device weight w [KH, Cin, Cout] (hd_pack_weight on the
  // default stream; sync() completes it) + TMA descriptors (box 64 rows: the kernel loads a 64/128-wide N tile as one or two, conv_tc.cu)
  bool pack(PackedConv &c, const float *w, int KH, int Cin) {
    const int rows = (c.Cout + 63) / 64 * 64;
    c.w_hi = dev_alloc((size_t)rows * c.K_pad * 2); c.w_lo = dev_alloc((size_t)rows * c.K_pad * 2);
    if (!c.w_hi || !c.w_lo) return false;
    c.tmap_hi = new_map(true); c.tmap_lo = new_map(true);
    int r = hd_pack_weight(w, KH, Cin, c.Cout, HD_PACK_FORWARD, 2, c.w_hi, c.w_lo, rows, c.K_pad, nullptr);
    if (!r) r = hd_make_weight_tmap(c.w_hi, rows, c.K_pad, 64, 2, c.tmap_hi);
    if (!r) r = hd_make_weight_tmap(c.w_lo, rows, c.K_pad, 64, 2, c.tmap_lo);
    if (r) { rc = rc ? rc : r; return false; }
    return true;
  }

  // waits for the packing queued by pack(): a plan's weights are then ready on any stream
  bool sync() {
    if (rc != HD_OK) return false;
    const cudaError_t e = cudaStreamSynchronize(nullptr);
    if (e != cudaSuccess) { hd::set_last_error("cudaStreamSynchronize", e); rc = HD_ERR_CUDA; return false; }
    return true;
  }

  // conv / FC weights in TF layout HWIO (FC: [in, out] = 1x1 HWIO); w != nullptr overrides the lookup (sliced FC weights)
  bool make_conv(PackedConv &c, const std::string &wname, int KH, int KW, int Cin, int Cout, int stride, int pad_t, int pad_l,
                 const std::vector<float> *scale, const std::vector<float> *shift, int relu, const float *w = nullptr, bool tc = true) {
    c.KH = KH; c.KW = KW; c.Cin = Cin; c.Cout = Cout; c.K = KH * KW * Cin; c.K_pad = c.K;
    c.stride = stride; c.pad_t = pad_t; c.pad_l = pad_l; c.post_relu = relu;
    if (!w) w = weight(wname, (long long)c.K * Cout);
    if (!w) return false;
    std::vector<float> w_kn(w, w + (size_t)c.K * Cout);
    c.w_kn = (float *)upload(w_kn);
    if (scale) c.post_scale = (float *)upload(*scale);
    if (shift) c.post_shift = (float *)upload(*shift);
    if (!c.w_kn || (scale && !c.post_scale) || (shift && !c.post_shift)) return false;
    if (!tc) return true;
    if (Cin % 64 != 0) return fail(HD_ERR_UNSUPPORTED, "layer '" + wname + "': Cin % 64 != 0 has no fp16 tensor-core packing");
    return pack(c, c.w_kn, KH * KW, Cin);
  }

  bool bias_vec(const std::string &name, int C, std::vector<float> &v) {
    const float *b = weight(name, C);
    if (!b) return false;
    v.assign(b, b + C);
    return true;
  }

  // nets.py PackedConv.bind + ConvOp.encode_act_maps for a pre-split (fp16 pair) input
  struct Bind {
    int n = 0, H = 0, W = 0;
    Pair in;
    float *out = nullptr;
    Pair out2;
    const float *post2_scale = nullptr, *post2_shift = nullptr;
    int post2_relu = 0;
    const float *res = nullptr;
    long long res_ld = 0;
    int res_H = 0, res_W = 0, res_stride = 1;
    int out_subsample = 0;
  };

  bool bind(const PackedConv &c, const Bind &b, hd_conv_desc &d) {
    memset(&d, 0, sizeof(d));
    const int Ho = c.KH > 1 ? (b.H + 2 * c.pad_t - c.KH) / c.stride + 1 : (b.H - 1) / c.stride + 1;
    const int Wo = c.KW > 1 ? (b.W + 2 * c.pad_l - c.KW) / c.stride + 1 : (b.W - 1) / c.stride + 1;
    d.in_ld = c.Cin;
    d.in_hi = b.in.hi; d.in_lo = b.in.lo;
    d.n_img = b.n; d.H = b.H; d.W = b.W; d.Cin = c.Cin; d.Ho = Ho; d.Wo = Wo; d.KH = c.KH; d.KW = c.KW;
    d.stride = c.stride; d.pad_t = c.pad_t; d.pad_l = c.pad_l;
    d.w_kn = c.w_kn; d.Cout = c.Cout; d.K_pad = c.K_pad;
    d.post_scale = c.post_scale; d.post_shift = c.post_shift; d.post_relu = c.post_relu;
    if (b.res) { d.res = b.res; d.res_ld = b.res_ld; d.res_H = b.res_H; d.res_W = b.res_W; d.res_stride = b.res_stride; }
    d.out = b.out; d.out_ld = c.Cout;
    d.out_subsample = b.out ? b.out_subsample : 0;
    if (b.out2.hi) {
      d.out_hi = b.out2.hi; d.out_lo = b.out2.lo; d.out2_ld = c.Cout;
      d.post2_scale = b.post2_scale; d.post2_shift = b.post2_shift; d.post2_relu = b.post2_relu;
    }
    d.impl = HD_IMPL_TC_3XF16;
    d.w_nk_hi = c.w_hi; d.w_nk_lo = c.w_lo; d.tmap_hi = c.tmap_hi; d.tmap_lo = c.tmap_lo;
    return encode_act_maps(d);
  }

  bool encode_act_maps(hd_conv_desc &d) {
    d.tmap_res = d.tmap_out = d.tmap_out_hi = d.tmap_out_lo = nullptr;
    const bool ok = d.impl == HD_IMPL_TC_3XF16 && d.in_hi && d.Cout % 32 == 0 &&
                    (!d.res || (d.res_stride == 1 && d.res_H == d.Ho && d.res_W == d.Wo));
    if (!ok) return true;
    const long long M = (long long)d.n_img * d.Ho * d.Wo;
    struct F { const void *ptr; long long ld; int eb; const void **slot; };
    F f[4] = {{d.res, d.res_ld, 4, &d.tmap_res}, {d.out, d.out_ld, 4, &d.tmap_out}, {d.out_hi, d.out2_ld, 2, &d.tmap_out_hi},
              {d.out_lo, d.out2_ld, 2, &d.tmap_out_lo}};
    for (auto &x : f) {
      if (!x.ptr || (x.slot == &d.tmap_out && d.out_subsample > 1)) continue;
      if (((uintptr_t)x.ptr % 16) || (x.ld * x.eb) % 16) {
        d.tmap_res = d.tmap_out = d.tmap_out_hi = d.tmap_out_lo = nullptr;
        return true;
      }
      void *m = new_map();
      const int r = hd_make_act_tmap(x.ptr, M, d.Cout, x.ld, x.eb, m);
      if (r) { rc = rc ? rc : r; return false; }
      *x.slot = m;
    }
    return true;
  }

  void conv_step(const hd_conv_desc &d) {
    net->steps.push_back([d](cudaStream_t st) { return hd_conv_gemm(&d, (void *)st); });
  }
};

const int kBlocks[4][3] = {{64, 3, 2}, {128, 4, 2}, {256, 6, 2}, {512, 3, 1}};      // (base depth, units, stride of the LAST unit)

struct Unit {
  int stride, base, depth, d_in;
  bool has_shortcut = false;
  float *pre_scale = nullptr, *pre_shift = nullptr;
  PackedConv shortcut, conv1, conv2, conv3;
};

int run_steps(hd_net *net, cudaStream_t st) {
  for (auto &s : net->steps) {
    const int r = s(st);
    if (r) return r;
  }
  return HD_OK;
}

// ------------------------------------------------------------------------------------------------ f_movie (re)binding
int bind_fmovie(hd_net *net, const float *x, float *out) {
  Builder b{net};
  net->steps.clear();
  net->maps.clear();
  net->bound_in = nullptr;             // a failure below must not leave a half-built plan looking bound
  net->bound_out = nullptr;
  const int B = net->B, T = net->T, C = net->C, L = net->layers;
  // persist layout: [0] act.hi [1] act.lo [2] mid [3] buf0 [4] buf1, then per block: gn1 gamma, gn1 beta, gn2 gamma, gn2 beta
  Pair act{net->persist[0], net->persist[1]};
  float *mid = (float *)net->persist[2];
  float *bufs[2] = {(float *)net->persist[3], (float *)net->persist[4]};
  const PackedConv *convs = (const PackedConv *)net->persist[5];
  const float *cur = x;
  for (int i = 0; i < L; ++i) {
    float *o = (i == L - 1) ? out : bufs[i % 2];
    const float *g1 = (const float *)net->persist[6 + 4 * i], *b1 = (const float *)net->persist[7 + 4 * i];
    const float *g2 = (const float *)net->persist[8 + 4 * i], *b2 = (const float *)net->persist[9 + 4 * i];
    const float *src = cur;
    net->steps.push_back([=](cudaStream_t st) { return hd_groupnorm_relu_split(src, g1, b1, act.hi, act.lo, B, T, C, 32, 1e-6f, (void *)st); });
    hd_conv_desc d;
    Builder::Bind bd;
    bd.n = B; bd.H = T; bd.W = 1; bd.in = act; bd.out = mid;
    if (!b.bind(convs[2 * i], bd, d)) { net->steps.clear(); return b.rc; }
    b.conv_step(d);
    net->steps.push_back([=](cudaStream_t st) { return hd_groupnorm_relu_split(mid, g2, b2, act.hi, act.lo, B, T, C, 32, 1e-6f, (void *)st); });
    Builder::Bind be;
    be.n = B; be.H = T; be.W = 1; be.in = act; be.out = o; be.res = cur; be.res_ld = C; be.res_H = T; be.res_W = 1; be.res_stride = 1;
    if (!b.bind(convs[2 * i + 1], be, d)) { net->steps.clear(); return b.rc; }
    b.conv_step(d);
    cur = o;
  }
  if (b.rc != HD_OK) { net->steps.clear(); return b.rc; }
  net->bound_in = x;
  net->bound_out = out;
  return HD_OK;
}

}  // namespace

extern "C" {

void hd_net_destroy(hd_net *net) {
  if (!net) return;
  for (void *p : net->allocs) cudaFree(p);
  if (net->kind == 2 && net->persist.size() > 5) delete[] (PackedConv *)net->persist[5];
  delete net;
}

const char *hd_net_error(const hd_net *net) { return net ? net->err.c_str() : ""; }
long long hd_net_num_launches(const hd_net *net) { return net ? (long long)net->steps.size() : 0; }

// ------------------------------------------------------------------------------------------------------------ ResNet
int hd_resnet50_create(hd_weight_fn get, void *user, int n_frames, int size, hd_net **out_net) {
  HD_REQUIRE(get && out_net && n_frames > 0 && size >= 32 && size % 2 == 0, "hd_resnet50_create: bad arguments (even size >= 32)");
  *out_net = nullptr;
  hd_net *net = new hd_net();
  net->kind = 1; net->get = get; net->user = user; net->n = n_frames; net->size = size;
  Builder b{net};
  const std::string p = "resnet_v2_50";
  const int n = n_frames;

  // ---- pack (nets.py PackedResNet) ----
  PackedConv conv1;                        // PackedConv1Planes: HWIO [ky(8), kx(8), c(4), co] with zero weights in the padding taps
  {
    const float *w = b.weight(p + "/conv1/weights", 7 * 7 * 3 * 64);
    std::vector<float> bias;
    if (w && b.bias_vec(p + "/conv1/biases", 64, bias)) {
      conv1.Cout = 64; conv1.K = conv1.K_pad = 256;
      std::vector<float> wp((size_t)256 * 64, 0.0f);
      for (int ky = 0; ky < 7; ++ky)
        for (int kx = 0; kx < 7; ++kx)
          for (int c = 0; c < 3; ++c) memcpy(&wp[(size_t)((ky * 8 + kx) * 4 + c) * 64], w + ((ky * 7 + kx) * 3 + c) * 64, 64 * sizeof(float));
      conv1.post_shift = (float *)b.upload(bias);
      const float *wd = (const float *)b.upload(wp);
      if (conv1.post_shift && wd) b.pack(conv1, wd, 8, 32);
    }
  }
  std::vector<Unit> units;
  int d_in = 64;
  for (int bi = 0; bi < 4 && b.rc == HD_OK; ++bi) {
    const int base = kBlocks[bi][0], nu = kBlocks[bi][1], bstride = kBlocks[bi][2], depth = 4 * base;
    for (int u = 1; u <= nu && b.rc == HD_OK; ++u) {
      const std::string q = p + "/block" + std::to_string(bi + 1) + "/unit_" + std::to_string(u) + "/bottleneck_v2";
      units.emplace_back();
      Unit &un = units.back();
      un.stride = (u == nu) ? bstride : 1; un.base = base; un.depth = depth; un.d_in = d_in;
      std::vector<float> s, sh, bias;
      if (!b.fold_bn(q + "/preact", d_in, s, sh)) break;
      un.pre_scale = (float *)b.upload(s); un.pre_shift = (float *)b.upload(sh);
      if (d_in != depth) {
        un.has_shortcut = true;
        if (!b.bias_vec(q + "/shortcut/biases", depth, bias)) break;
        if (!b.make_conv(un.shortcut, q + "/shortcut/weights", 1, 1, d_in, depth, un.stride, 0, 0, nullptr, &bias, 0)) break;
      }
      if (!b.fold_bn(q + "/conv1/BatchNorm", base, s, sh)) break;
      if (!b.make_conv(un.conv1, q + "/conv1/weights", 1, 1, d_in, base, 1, 0, 0, &s, &sh, 1)) break;
      if (!b.fold_bn(q + "/conv2/BatchNorm", base, s, sh)) break;
      // conv2d_same: stride 1 -> SAME (pad 1); stride 2 -> explicit pad 1+1 then VALID  (A.2)
      if (!b.make_conv(un.conv2, q + "/conv2/weights", 3, 3, base, base, un.stride, 1, 1, &s, &sh, 1)) break;
      if (!b.bias_vec(q + "/conv3/biases", depth, bias)) break;
      if (!b.make_conv(un.conv3, q + "/conv3/weights", 1, 1, base, depth, 1, 0, 0, nullptr, &bias, 0)) break;
      d_in = depth;
    }
  }
  float *post_scale = nullptr, *post_shift = nullptr;
  if (b.rc == HD_OK) {
    std::vector<float> s, sh;
    if (b.fold_bn(p + "/postnorm", d_in, s, sh)) { post_scale = (float *)b.upload(s); post_shift = (float *)b.upload(sh); }
  }
  b.sync();
  if (b.rc != HD_OK) { const int r = b.rc; hd_net_destroy(net); return r; }

  // ---- plan (nets.py ResNetPlan, split mode, root + all units + tail) ----
  const int H1 = size / 2, H2 = (H1 + 1) / 2;
  long long mx_io = (long long)H2 * H2 * 64, mx_r = 0;
  {
    int h = H2;
    for (const Unit &un : units) {
      const int ho = (h - 1) / un.stride + 1;
      if (un.has_shortcut) mx_io = std::max(mx_io, (long long)h * h * un.depth);
      mx_io = std::max(mx_io, (long long)ho * ho * un.depth);
      mx_r = std::max(mx_r, (long long)h * h * un.base);
      h = ho;
    }
    mx_io = std::max(mx_io, (long long)H1 * H1 * 64);
  }
  float *bufA = (float *)b.dev_alloc((size_t)n * mx_io * 4), *bufB = (float *)b.dev_alloc((size_t)n * mx_io * 4);
  float *bufS = (float *)b.dev_alloc((size_t)n * mx_io * 4);
  Pair xs = b.pair((size_t)n * mx_io), ys = b.pair((size_t)n * mx_io), r1 = b.pair((size_t)n * mx_r), r2 = b.pair((size_t)n * mx_r);
  const int WP = (size + 8 + 1) / 2 * 2;
  const size_t plane_elems = (size_t)n * (size + 6) * WP * 4;
  void *plane_hi = b.dev_alloc(plane_elems * 2, true), *plane_lo = b.dev_alloc(plane_elems * 2, true);   // zero border, never rewritten
  if (b.rc != HD_OK) { const int r = b.rc; hd_net_destroy(net); return r; }

  net->steps.push_back([=](cudaStream_t st) { return hd_pack_conv1_planes(net->in0, plane_hi, plane_lo, n, size, size, WP, (void *)st); });
  {
    hd_conv_desc d;
    memset(&d, 0, sizeof(d));
    d.in_hi = plane_hi; d.in_lo = plane_lo; d.in_ld = 4;
    d.n_img = n; d.H = size + 6; d.W = WP; d.Cin = 32; d.Ho = d.Wo = H1;
    d.KH = 8; d.KW = 1; d.stride = 2; d.pad_t = 0; d.pad_l = 0; d.Cout = 64; d.K_pad = 256;
    d.post_shift = conv1.post_shift; d.out = bufS; d.out_ld = 64; d.impl = HD_IMPL_TC_3XF16;
    d.w_nk_hi = conv1.w_hi; d.w_nk_lo = conv1.w_lo; d.tmap_hi = conv1.tmap_hi; d.tmap_lo = conv1.tmap_lo;
    d.flags = HD_CONV_INPUT_PLANES;
    if (!b.encode_act_maps(d)) { const int r = b.rc; hd_net_destroy(net); return r; }
    b.conv_step(d);
  }
  {
    // pool1 + the first unit's pre-activation as an fp16 pair; its fp32 output is dead (unit 1's shortcut is a conv of the pre-activation)
    const float *ps = units[0].pre_scale, *pb = units[0].pre_shift;
    float *pool_out = units[0].has_shortcut ? nullptr : bufA;
    net->steps.push_back([=](cudaStream_t st) { return hd_maxpool3x3s2_same(bufS, pool_out, n, H1, H1, 64, ps, pb, xs.hi, xs.lo, (void *)st); });
  }
  float *x = bufA, *y = bufB;
  int H = H2;
  bool sub_ready = false;              // bufS already holds x[:, ::s, ::s] of the current unit's input
  hd_conv_desc prev3;                  // the previous unit's conv3, the last step pushed when the loop reaches the next unit's conv1
  bool has_prev3 = false;
  for (size_t ui = 0; ui < units.size() && b.rc == HD_OK; ++ui) {
    const Unit &un = units[ui];
    const int s = un.stride, Ho = (H - 1) / s + 1;
    const float *res = nullptr;
    hd_conv_desc d;
    if (un.has_shortcut) {
      Builder::Bind bs; bs.n = n; bs.H = H; bs.W = H; bs.in = xs; bs.out = bufS;
      if (!b.bind(un.shortcut, bs, d)) break;
      b.conv_step(d);
      res = bufS;
    } else if (s > 1) {                                  // strided identity shortcut: dense subsampled copy (row-aligned residual),
      if (!sub_ready) {                                  // written by the previous unit's conv3 epilogue (out_subsample) when possible
        const float *src = x;
        const int Hh = H, Cc = un.depth;
        net->steps.push_back([=](cudaStream_t st) { return hd_subsample(src, bufS, n, Hh, Hh, Cc, s, (void *)st); });
      }
      res = bufS;
    } else {
      res = x;
    }
    Builder::Bind b1; b1.n = n; b1.H = H; b1.W = H; b1.in = xs; b1.out2 = r1;
    if (!b.bind(un.conv1, b1, d)) break;
    // an identity unit's conv1 reads only the pair the previous conv3 writes: one launch for both where the library runs the pair
    // (nets.py ResNetPlan, ChainOp)
    bool chained = false;
    if (has_prev3 && !un.has_shortcut && !(s > 1 && !sub_ready)) {
      hd_conv_desc c3 = prev3, c1 = d;
      c3.out_hi = c3.out_lo = nullptr;
      c3.tmap_out_hi = c3.tmap_out_lo = nullptr;
      c1.in_hi = c1.in_lo = nullptr;
      if (hd_conv_gemm_chain_supported(&c3, &c1) == 1) {
        net->steps.back() = [c3, c1](cudaStream_t st) { return hd_conv_gemm_chain(&c3, &c1, (void *)st); };
        chained = true;
      }
    }
    if (!chained) b.conv_step(d);
    Builder::Bind b2; b2.n = n; b2.H = H; b2.W = H; b2.in = r1; b2.out2 = r2;
    if (!b.bind(un.conv2, b2, d)) break;
    b.conv_step(d);
    const bool last = ui + 1 == units.size();
    Builder::Bind b3; b3.n = n; b3.H = Ho; b3.W = Ho; b3.in = r2;
    b3.res = res; b3.res_ld = un.depth; b3.res_H = Ho; b3.res_W = Ho; b3.res_stride = 1;
    sub_ready = false;
    if (!last) {
      b3.out2 = ys; b3.post2_scale = units[ui + 1].pre_scale; b3.post2_shift = units[ui + 1].pre_shift; b3.post2_relu = 1;
      // the fp32 block output only feeds an IDENTITY shortcut; skip it when the next unit's shortcut is a conv
      b3.out = units[ui + 1].has_shortcut ? nullptr : y;
      // ... and when that identity shortcut is strided only x[:, ::s, ::s] is ever read: write just those pixels, densely, into bufS
      if (b3.out && units[ui + 1].stride > 1 && !un.has_shortcut && s == 1) {
        sub_ready = true;
        b3.out = bufS; b3.out_subsample = units[ui + 1].stride;
      }
    } else {
      b3.out = y;
    }
    if (!b.bind(un.conv3, b3, d)) break;
    b.conv_step(d);
    prev3 = d;
    has_prev3 = true;
    std::swap(x, y);
    std::swap(xs, ys);
    H = Ho;
  }
  if (b.rc != HD_OK) { const int r = b.rc; hd_net_destroy(net); return r; }
  {
    const float *fin = x;
    const int HW = H * H, Cc = d_in;
    net->steps.push_back([=](cudaStream_t st) { return hd_bnrelu_avgpool(fin, post_scale, post_shift, net->out0, n, HW, Cc, (void *)st); });
  }
  *out_net = net;
  return HD_OK;
}

int hd_resnet50_forward(hd_net *net, const float *images, float *phi, void *stream) {
  HD_REQUIRE(net && net->kind == 1 && images && phi, "hd_resnet50_forward: bad arguments");
  net->in0 = images; net->out0 = phi;
  return run_steps(net, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------------------ f_movie
int hd_fmovie_create(hd_weight_fn get, void *user, int B, int T, int num_conv_layers, hd_net **out_net) {
  HD_REQUIRE(get && out_net && B > 0 && T > 0 && num_conv_layers > 0, "hd_fmovie_create: bad arguments");
  const int C = 2048;
  HD_REQUIRE(T * (C / 32) <= 1280, "hd_fmovie_create: T * C/groups <= 1280 (T <= 20) is what hd_groupnorm_relu_split supports");
  *out_net = nullptr;
  hd_net *net = new hd_net();
  net->kind = 2; net->get = get; net->user = user; net->B = B; net->T = T; net->C = C; net->layers = num_conv_layers;
  Builder b{net};
  Pair act = b.pair((size_t)B * T * C);
  net->persist = {act.hi, act.lo, b.dev_alloc((size_t)B * T * C * 4), b.dev_alloc((size_t)B * T * C * 4), b.dev_alloc((size_t)B * T * C * 4)};
  PackedConv *convs = new PackedConv[2 * num_conv_layers];
  net->persist.push_back(convs);
  for (int i = 0; i < num_conv_layers && b.rc == HD_OK; ++i) {
    const std::string name = "block_" + std::to_string(i);
    for (int k = 1; k <= 2; ++k) {
      const std::string gn = "AZ_FC_block_preact_gn" + std::to_string(k) + name, cv = "AZ_FC_block2_conv" + std::to_string(k) + name;
      std::vector<float> g, be, bias;
      if (!b.bias_vec(gn + "/gamma", C, g) || !b.bias_vec(gn + "/beta", C, be) || !b.bias_vec(cv + "/biases", C, bias)) break;
      net->persist.push_back(b.upload(g));
      net->persist.push_back(b.upload(be));
      // temporal conv: kernel [3,1] over NT1C, SAME  (models.py:173-184,209-221)
      if (!b.make_conv(convs[2 * i + k - 1], cv + "/weights", 3, 1, C, C, 1, 1, 0, nullptr, &bias, 0)) break;
    }
  }
  b.sync();
  if (b.rc != HD_OK) { const int r = b.rc; hd_net_destroy(net); return r; }
  *out_net = net;
  return HD_OK;
}

int hd_fmovie_forward(hd_net *net, const float *phi, float *out, void *stream) {
  HD_REQUIRE(net && net->kind == 2 && phi && out && phi != out, "hd_fmovie_forward: bad arguments (in-place is not supported)");
  if (net->bound_in != phi || net->bound_out != out) {      // descriptors / tensor maps carry the caller's pointers: host work only
    const int r = bind_fmovie(net, phi, out);
    if (r) return r;
  }
  return run_steps(net, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------------------ IEF
int hd_ief_create(hd_weight_fn get, void *user, int N, const int *delta_t, int num_delta, hd_net **out_net) {
  HD_REQUIRE(get && out_net && N > 0 && num_delta >= 0 && (num_delta == 0 || delta_t), "hd_ief_create: bad arguments");
  *out_net = nullptr;
  hd_net *net = new hd_net();
  net->kind = 3; net->get = get; net->user = user; net->N = N;
  Builder b{net};
  for (int i = 0; i < num_delta; ++i)
    if (delta_t[i] != 0) net->delta_t.push_back(delta_t[i]);
  std::sort(net->delta_t.begin(), net->delta_t.end());
  const int D = (int)net->delta_t.size();
  net->D = D;
  const int feat = 2048, Hd = 1024, num_stage = 3;
  float *P = (float *)b.dev_alloc((size_t)N * Hd * 4), *h2 = (float *)b.dev_alloc((size_t)N * Hd * 4);
  Pair phi_split = b.pair((size_t)N * feat), h1_split = b.pair((size_t)N * Hd);
  {
    const float *mp = b.weight("mean_param", 85);
    if (mp) {
      std::vector<float> t0((size_t)N * 85);
      for (int i = 0; i < N; ++i) memcpy(&t0[(size_t)i * 85], mp, 85 * sizeof(float));
      net->theta0 = (float *)b.upload(t0);
    }
  }
  net->steps.push_back([=](cudaStream_t st) { return hd_split_f16(net->in0, phi_split.hi, phi_split.lo, (long long)N * feat, (void *)st); });

  // one hmr_ief head: fc1 split into phi.W1[:2048] (hoisted, tensor cores) + theta.W1[2048:] (per stage), fc2 on the tensor cores, fc3 small
  auto head = [&](const std::string &scope, int d, std::function<const float *()> start, int start_ld, std::function<float *()> state, int ld) {
    const std::string q = scope + "/3D_module";
    const float *W1 = b.weight(q + "/fc1/weights", (long long)(feat + d) * Hd);
    std::vector<float> b1, b2, b3;
    if (!W1 || !b.bias_vec(q + "/fc1/biases", Hd, b1) || !b.bias_vec(q + "/fc2/biases", Hd, b2) || !b.bias_vec(q + "/fc3/biases", d, b3)) return;
    PackedConv fc1_phi, fc1_theta, fc2, fc3;
    if (!b.make_conv(fc1_phi, q + "/fc1/weights[:2048]", 1, 1, feat, Hd, 1, 0, 0, nullptr, &b1, 0, W1)) return;
    if (!b.make_conv(fc1_theta, q + "/fc1/weights[2048:]", 1, 1, d, Hd, 1, 0, 0, nullptr, nullptr, 1, W1 + (size_t)feat * Hd, false)) return;
    if (!b.make_conv(fc2, q + "/fc2/weights", 1, 1, Hd, Hd, 1, 0, 0, nullptr, &b2, 1)) return;
    if (!b.make_conv(fc3, q + "/fc3/weights", 1, 1, Hd, d, 1, 0, 0, nullptr, &b3, 0, nullptr, false)) return;
    hd_conv_desc dd;
    Builder::Bind bp; bp.n = N; bp.H = 1; bp.W = 1; bp.in = phi_split; bp.out = P;
    if (!b.bind(fc1_phi, bp, dd)) return;
    b.conv_step(dd);
    hd_conv_desc d2;
    Builder::Bind b2d; b2d.n = N; b2d.H = 1; b2d.W = 1; b2d.in = h1_split; b2d.out = h2;
    if (!b.bind(fc2, b2d, d2)) return;
    const float *Wt = fc1_theta.w_kn, *W3 = fc3.w_kn, *bias3 = fc3.post_shift;
    for (int s = 0; s < num_stage; ++s) {
      const bool first = s == 0;
      net->steps.push_back([=](cudaStream_t st) {
        const float *prev = first ? start() : state();
        return hd_ief_fc1_theta(P, prev, first ? start_ld : ld, Wt, d, Hd, h1_split.hi, h1_split.lo, nullptr, N, (void *)st);
      });
      b.conv_step(d2);
      net->steps.push_back([=](cudaStream_t st) {
        const float *prev = first ? start() : state();
        return hd_ief_fc3(h2, W3, bias3, prev, first ? start_ld : ld, state(), ld, N, Hd, d, (void *)st);
      });
    }
  };
  const std::string scope = "single_view_ief";
  head(scope, 85, [net]() { return (const float *)net->theta0; }, 85, [net]() { return net->out0; }, 85);
  for (int i = 0; i < D && b.rc == HD_OK; ++i) {
    const int dt = net->delta_t[i];
    const std::string sc = scope + (dt > 0 ? "_future" + std::to_string(dt) : "_past" + std::to_string(-dt));
    // models.py:349-371: the delta head starts from the main prediction's pose ([:, 3:75]), output = [1, 0, 0 | pose | beta]
    net->steps.push_back([=](cudaStream_t st) { return hd_ief_delta_init(net->out0, net->out1 + (size_t)i * 85, D * 85, N, (void *)st); });
    auto view = [net, i]() { return net->out1 + (size_t)i * 85 + 3; };
    head(sc, 72, [view]() { return (const float *)view(); }, D * 85, view, D * 85);
  }
  b.sync();
  if (b.rc != HD_OK) { const int r = b.rc; hd_net_destroy(net); return r; }
  *out_net = net;
  return HD_OK;
}

int hd_ief_forward(hd_net *net, const float *phi, float *theta, float *deltas, void *stream) {
  HD_REQUIRE(net && net->kind == 3 && phi && theta && (net->D == 0 || deltas), "hd_ief_forward: bad arguments");
  net->in0 = phi; net->out0 = theta; net->out1 = deltas;
  return run_steps(net, (cudaStream_t)stream);
}

}  // extern "C"
