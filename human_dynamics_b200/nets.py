"""Host-side layer plans for the three networks on the path: slim ResNet-v2-50, f_movie, IEF.

A *plan* is a list of pre-filled C descriptors (hd_conv_desc) over pre-allocated device buffers, so a
forward pass is a sequence of ctypes calls with no Python-side tensor math and no allocation.
Weights come in as a dict of numpy arrays keyed by TF variable names (SURVEY.md A.6).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import lib, check, fptr, current_stream, ConvDesc

RESNET_BLOCKS = ((64, 3, 2), (128, 4, 2), (256, 6, 2), (512, 3, 1))
BN_EPS = 1e-5        # resnet_arg_scope batch_norm_epsilon [TF-ext]
# Training-mode batch norm [TF-ext] (slim batch_norm with is_training=True; TF 1.8 takes its fused kernel for 4-D NHWC input): a map is
# normalised with its batch mean and BIASED batch variance over frames x H x W, and the layer's UPDATE_OPS move the moving statistics
# by one step of assign_moving_average, m -= (m - v) * (1 - BN_DECAY), with v = the batch mean and the BESSEL-CORRECTED batch variance
# var_b * rows / (rows - 1) (the variance output of the fused kernel).  The fused op also raises an epsilon below 1.001e-5 to that
# value; both trunks here use BN_EPS, as the inference trunk always has.  Pinned only through the TF stand-in (oracle/ref_exec).
BN_DECAY = 0.997     # resnet_arg_scope batch_norm_decay [TF-ext]
# Trunk backward conventions [TF-ext]: ReluGrad is 0 at 0; MaxPoolGrad of pool1 (3x3 stride 2 SAME) sends each window's gradient to its
# FIRST maximum in scan order (ky, then kx), as TF's CPU kernel does (hd_maxpool3x3s2_same_backward).
GN_EPS = 1e-6        # tf.contrib.layers.group_norm epsilon [TF-ext]
GN_GROUPS = 32


# impl names whose networks run on the fp16 formats (pre-split activations, conv1 planes, fast heads).  'tc1h' is the half-precision
# inference mode (HD_IMPL_TC_1XF16): the fp16 heads alone, one MMA per product, and no remainder buffers at all.
F16_IMPLS = ('auto', 'tc3h', 'tc1h')


def heads_only(impl):
    """True for the half-precision inference mode: activation pairs are (head, None) and every descriptor leaves the remainders unset."""
    return impl == 'tc1h'


def f16_pair(shape, device, impl):
    """The fp16 A-operand buffers of one activation: (head, remainder), or (head, None) in the half-precision mode."""
    hi = torch.empty(shape, dtype=torch.float16, device=device)
    return (hi, None) if heads_only(impl) else (hi, torch.empty(shape, dtype=torch.float16, device=device))


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def require_training_impl(impl, who):
    """The training paths run FP32-class arithmetic (their backward passes and the saved activations they read): refuse 'tc1h'."""
    if heads_only(impl):
        raise _lib.HDError("%s: impl 'tc1h' is an inference-only half-precision mode; training runs FP32-class ('auto' / 'tc3h')" % who)


# Precision of the training backward passes' tensor-core GEMMs (weight and data gradients; the forward passes never change):
#   'fp32'  3xTF32 (HD_IMPL_TC_3XTF32), FP32-class
#   'tf32'  1xTF32 (HD_IMPL_TC_1XTF32): one TF32 MMA per product on round-to-nearest heads, no remainder operand (DESIGN.md section 2)
GRAD_PRECISIONS = ('fp32', 'tf32')


def grad_one_pass(grad_precision, who):
    """True for 'tf32' (single-pass TF32 gradients), False for 'fp32'; any other value raises HDError."""
    if not isinstance(grad_precision, str) or grad_precision not in GRAD_PRECISIONS:
        raise _lib.HDError("%s: grad_precision must be 'fp32' or 'tf32', got %r" % (who, grad_precision))
    return grad_precision == 'tf32'


def _dev(a, device, dtype=np.float32):
    if isinstance(a, torch.Tensor):           # already on the device (TemporalModel's parameters): used in place
        return a
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(device)


def pack_weight(src, KH, Cin, Cout, hi, lo, stream):
    """hd_pack_weight (forward): the fp32 weight src [KH, Cin, Cout] on the device -> K-major head / remainder hi, lo [rows, k_pad]
    (fp16 tensors: fp16 head + 2^11-scaled remainder; fp32 tensors: TF32 pair), zero past the matrix.  Runs on `stream`."""
    check(lib.hd_pack_weight(C.c_void_p(src.data_ptr()), KH, Cin, Cout, _lib.HD_PACK_FORWARD, hi.element_size(), C.c_void_p(hi.data_ptr()),
                             C.c_void_p(lo.data_ptr()), hi.shape[0], hi.shape[1], stream), 'hd_pack_weight')


def weight_tmap(t):
    """128-byte TMA descriptor of a packed [rows, k_pad] weight half (box 64 rows: the kernel loads a 64- or 128-wide N tile as one or
    two boxes, conv_tc.cu)."""
    m = (C.c_ubyte * 128)()
    check(lib.hd_make_weight_tmap(C.c_void_p(t.data_ptr()), t.shape[0], t.shape[1], 64, t.element_size(), C.cast(m, C.c_void_p)),
          'hd_make_weight_tmap')
    return m


def _packs_on(device):
    """Packing is a kernel launch, so only a CUDA device runs it.  Host-side plan logic on another device (the CPU wiring tests) gets
    its pack tensors and descriptors, but the packs stay unwritten."""
    return torch.device(device).type == 'cuda'


def sync_packing(device):
    """Wait for the packing queued on `device`'s current stream: a constructor's weights are then complete on any stream."""
    if _packs_on(device):
        torch.cuda.current_stream(device).synchronize()


def fold_bn(w, prefix):
    """BN inference -> (scale, shift): y = x*scale + shift  (A.5)."""
    g = w[prefix + '/gamma'].astype(np.float64)
    b = w[prefix + '/beta'].astype(np.float64)
    m = w[prefix + '/moving_mean'].astype(np.float64)
    v = w[prefix + '/moving_variance'].astype(np.float64)
    s = g / np.sqrt(v + BN_EPS)
    return s.astype(np.float32), (b - m * s).astype(np.float32)


class PackedConv(object):
    """Device-resident weights (+ epilogue vectors) of one conv / FC layer.

    w_hwio: TF HWIO (FC: [in, out]) float32, a host array or a contiguous device tensor whose storage the layer then reads in place
    (as post_scale / post_shift may be).  The tensor-core packs (K-major head / remainder, rows padded to 64; DESIGN.md 3) are written
    from it on the device by hd_pack_weight, on the current stream."""

    def __init__(self, w_hwio, device, post_scale=None, post_shift=None, post_relu=False, stride=1, pad=(0, 0),
                 tc=False):
        if not isinstance(w_hwio, torch.Tensor):
            w_hwio = np.asarray(w_hwio, np.float32)
        shape = tuple(w_hwio.shape)
        self.KH, self.KW, self.Cin, self.Cout = (1, 1) + shape if len(shape) == 2 else shape
        self.K = self.KH * self.KW * self.Cin
        self.stride = stride
        self.pad_t, self.pad_l = pad
        self.device = device
        self.w_kn = _dev(w_hwio.reshape(self.K, self.Cout), device)
        self.post_scale = _dev(post_scale, device) if post_scale is not None else None
        self.post_shift = _dev(post_shift, device) if post_shift is not None else None
        self.post_relu = bool(post_relu)
        self.tc = False            # False | 'f16' | 'tf32': which tensor-core packing this layer carries
        self.K_pad = 0
        want = {True: 'f16', 'auto': 'f16', 'tc3h': 'f16', 'tc1h': 'f16', 'tc3': 'tf32', 'tc1': 'tf32'}.get(tc, tc)
        gather = want == 'f16' and self.Cin % 32 != 0 and self.Cout <= 64   # conv1: row-segment gather producer
        if want == 'f16' and self.Cin % 64 != 0 and not gather:
            want = 'tf32'
        self.gather = bool(gather)
        if want in ('f16', 'tf32') and (self.Cin % 32 == 0 or gather):
            seg = self.KW * self.Cin
            segp = (seg + 7) // 8 * 8                        # gather layout: each kernel row's KW*Cin floats padded to x8
            self.K_pad = (self.KH * segp + 63) // 64 * 64 if gather else self.K
            if gather:                                       # K index = ky*segp + (kx*Cin + ci)   (conv_tc.cu GATHER producer)
                src = torch.zeros((self.KH, segp, self.Cout), dtype=torch.float32, device=device)
                src[:, :seg] = self.w_kn.view(self.KH, seg, self.Cout)
                self.pack_src = (src, self.KH, segp)
            else:
                self.pack_src = (self.w_kn, self.KH * self.KW, self.Cin)
            rows = (self.Cout + 63) // 64 * 64
            dt = torch.float16 if want == 'f16' else torch.float32
            self.w_nk_hi = torch.empty((rows, self.K_pad), dtype=dt, device=device)
            self.w_nk_lo = torch.empty((rows, self.K_pad), dtype=dt, device=device)
            if _packs_on(device):
                self.repack(current_stream())
            self.tmap_hi, self.tmap_lo = weight_tmap(self.w_nk_hi), weight_tmap(self.w_nk_lo)
            self.tc = want

    def repack(self, stream):
        """Rewrite w_nk_hi / w_nk_lo on `stream` from the fp32 source `pack_src` (w_kn; for the gather layout its zero-padded copy
        [KH, segp, Cout] made at construction)."""
        src, KH, Cin = self.pack_src
        if self.gather:                    # the zero-padded copy follows w_kn (a trainable weight changes in place)
            src[:, :self.KW * self.Cin].copy_(self.w_kn.view(self.KH, self.KW * self.Cin, self.Cout))
        pack_weight(src, KH, Cin, self.Cout, self.w_nk_hi, self.w_nk_lo, stream)

    def bind(self, inp, n_img, H, W, out, in_ld=None, out_ld=None, pre=None, res=None, res_geom=None, impl='auto',
             inp_split=None, out_split=None, post2=None, out_subsample=0, post=None):
        """Fill a descriptor.  inp/out/res: CUDA float32 tensors (only their data_ptr is used).

        pre = (scale, shift, img_stride, relu); res_geom = (res_ld, res_H, res_W, res_stride).
        post = (scale|None, shift|None, relu): epilogue vectors in place of the layer's own (the training-mode trunk writes conv1 /
        conv2 raw, post = (None, None, False), and normalises them with batch statistics in the next layer's prologue).
        out_subsample = s > 1: `out` is the dense [n, ceil(Ho/s), ceil(Wo/s), Cout] tensor x[:, ::s, ::s] (hd_b200.h);
        inp_split = (hi, lo) fp16 tensors: pre-activated, pre-split A operand (then `inp` may be None);
        out_split = (hi, lo) fp16 tensors + post2 = (scale|None, shift|None, relu): second output (then `out` may be None).
        impl 'tc1h' (half precision, HD_IMPL_TC_1XF16): the pairs are (hi, None) and no remainder pointer is set.
        """
        d = ConvDesc()
        Ho = (H + 2 * self.pad_t - self.KH) // self.stride + 1 if self.KH > 1 else (H - 1) // self.stride + 1
        Wo = (W + 2 * self.pad_l - self.KW) // self.stride + 1 if self.KW > 1 else (W - 1) // self.stride + 1
        d.in_ = inp.data_ptr() if inp is not None else None
        d.in_ld = self.Cin if in_ld is None else in_ld
        heads = heads_only(impl)
        if inp_split is not None:
            d.in_hi = inp_split[0].data_ptr()
            if not heads:
                d.in_lo = inp_split[1].data_ptr()
        d.n_img, d.H, d.W, d.Cin = n_img, H, W, self.Cin
        d.Ho, d.Wo, d.KH, d.KW = Ho, Wo, self.KH, self.KW
        d.stride, d.pad_t, d.pad_l = self.stride, self.pad_t, self.pad_l
        d.w_kn = self.w_kn.data_ptr()
        d.Cout = self.Cout
        d.K_pad = self.K_pad
        if pre is not None:
            d.pre_scale, d.pre_shift = pre[0].data_ptr(), pre[1].data_ptr()
            d.pre_img_stride, d.pre_relu = int(pre[2]), int(pre[3])
        post_scale, post_shift, post_relu = (self.post_scale, self.post_shift, self.post_relu) if post is None else post
        if post_scale is not None:
            d.post_scale = post_scale.data_ptr()
        if post_shift is not None:
            d.post_shift = post_shift.data_ptr()
        d.post_relu = int(post_relu)
        if res is not None:
            d.res = res.data_ptr()
            if res_geom is None:
                res_geom = (self.Cout, Ho, Wo, 1)
            d.res_ld, d.res_H, d.res_W, d.res_stride = res_geom
        d.out = out.data_ptr() if out is not None else None
        d.out_ld = self.Cout if out_ld is None else out_ld
        d.out_subsample = int(out_subsample) if out is not None else 0
        if out_split is not None:
            d.out_hi, d.out2_ld = out_split[0].data_ptr(), self.Cout
            if not heads:
                d.out_lo = out_split[1].data_ptr()
            if post2 is not None:
                if post2[0] is not None:
                    d.post2_scale = post2[0].data_ptr()
                if post2[1] is not None:
                    d.post2_shift = post2[1].data_ptr()
                d.post2_relu = int(post2[2])
        # ragged layers (Cin % 32 != 0, unaligned views) always run on the exact-FP32 SIMT kernel
        use_tc = bool(self.tc) and impl in ('auto', 'tc3', 'tc1', 'tc3h', 'tc1h') and \
            (self.gather or inp_split is not None or ((d.in_ld % 4 == 0) and (inp.data_ptr() % 16 == 0)))
        if (inp_split is not None or out_split is not None) and not (use_tc and self.tc == 'f16'):
            raise _lib.HDError('pre-split activations need the fp16 tensor-core packing (impl auto / tc3h / tc1h, Cin % 64 == 0)')
        if use_tc:
            if self.tc == 'f16':
                d.impl = _lib.HD_IMPL_TC_1XF16 if heads else _lib.HD_IMPL_TC_3XF16
            else:
                d.impl = _lib.HD_IMPL_TC_1XTF32 if impl in ('tc1', 'tc1h') else _lib.HD_IMPL_TC_3XTF32
            d.w_nk_hi = self.w_nk_hi.data_ptr()
            d.tmap_hi = C.cast(self.tmap_hi, C.c_void_p)
            if not heads:
                d.w_nk_lo = self.w_nk_lo.data_ptr()
                d.tmap_lo = C.cast(self.tmap_lo, C.c_void_p)
        else:
            d.impl = _lib.HD_IMPL_SIMT
        op = ConvOp(d, (self, inp, out, pre, res, inp_split, out_split, post2, post), (Ho, Wo))
        op.encode_act_maps()
        return op


class BackwardDataPack(object):
    """PackedConv's backward twin: the transposed, tap-flipped weight of a conv whose conv is dX, written on the device from the fp32
    weight [KH, Cin, Cout] (KH: the conv's taps; FC: 1) by hd_pack_weight(HD_PACK_BACKWARD_DATA): TF32 head / remainder
    [roundup64(Cin), KH*Cout] for impl tc3, the B operand of dgrad_op."""

    def __init__(self, weight, KH, Cin, Cout):
        self.src, self.src_shape = weight, (KH, Cin, Cout)
        self.Cout, self.K = Cin, KH * Cout
        if self.K % 32 != 0:
            raise _lib.HDError('BackwardDataPack: K = %d does not fit the TF32 packing' % self.K)
        self.w_nk_hi = torch.empty(((Cin + 63) // 64 * 64, self.K), dtype=torch.float32, device=weight.device)
        self.w_nk_lo = torch.empty_like(self.w_nk_hi)
        self.tmap_hi, self.tmap_lo = weight_tmap(self.w_nk_hi), weight_tmap(self.w_nk_lo)

    def repack(self, stream):
        KH, Cin, Cout = self.src_shape
        check(lib.hd_pack_weight(fptr(self.src), KH, Cin, Cout, _lib.HD_PACK_BACKWARD_DATA, 4, _vp(self.w_nk_hi), _vp(self.w_nk_lo),
                                 self.w_nk_hi.shape[0], self.K, stream), 'hd_pack_weight')


def dgrad_op(pack, inp, n, H, W, KH, KW, out, res=None, one_pass=False):
    """A backward GEMM as an hd_conv_gemm op in its 3xTF32 mode (one_pass: 1xTF32 on the pack's head alone): out[n, H, W, pack.Cout]
    (+ res) = the stride-1 SAME KH x KW conv of inp [n, H, W, Cin] with the B operand `pack`, Cin = pack.K / (KH*KW).

    pack: a BackwardDataPack (the data gradient of a conv, or over the zero-inserted gradient of a strided conv2d_same 3x3; f_movie's
    3x1 conv over n clips of H = T frames; an FC layer, H = W = KH = KW = 1), or any operand with its fields w_nk_hi / w_nk_lo /
    tmap_hi / tmap_lo / Cout / K (a weight gradient's stacked upstream gradient).  The op holds `pack` and the tensors until it is
    dropped."""
    Cin, Cout = pack.K // (KH * KW), pack.Cout
    d = ConvDesc()
    d.in_, d.in_ld = inp.data_ptr(), Cin
    d.n_img, d.H, d.W, d.Cin = n, H, W, Cin
    d.Ho, d.Wo, d.KH, d.KW, d.stride, d.pad_t, d.pad_l = H, W, KH, KW, 1, KH // 2, KW // 2
    d.w_kn = pack.w_nk_hi.data_ptr()
    d.w_nk_hi = pack.w_nk_hi.data_ptr()
    d.Cout, d.K_pad = Cout, pack.K
    if res is not None:
        d.res, d.res_ld, d.res_H, d.res_W, d.res_stride = res.data_ptr(), Cout, H, W, 1
    d.out, d.out_ld = out.data_ptr(), Cout
    d.tmap_hi = C.cast(pack.tmap_hi, C.c_void_p)
    if one_pass:
        d.impl = _lib.HD_IMPL_TC_1XTF32
    else:
        d.impl = _lib.HD_IMPL_TC_3XTF32
        d.w_nk_lo, d.tmap_lo = pack.w_nk_lo.data_ptr(), C.cast(pack.tmap_lo, C.c_void_p)
    return ConvOp(d, (pack, inp, out, res), (H, W))


class SubsampleOp(object):
    """x[:, ::s, ::s, :] into a dense buffer (slim's max_pool2d(1x1, stride) shortcut): one op in a plan's op list."""
    __slots__ = ('src', 'dst', 'geom', 'd')

    def __init__(self, src, dst, n, H, C, stride):
        self.src, self.dst, self.geom, self.d = src, dst, (n, H, H, C, stride), None

    def rebind(self, field, tensor):
        self.src = tensor

    def encode_act_maps(self):
        pass

    def run(self, stream):
        n, H, W, Cc, s = self.geom
        check(lib.hd_subsample(fptr(self.src), fptr(self.dst), n, H, W, Cc, s, stream), 'hd_subsample')


class ConvOp(object):
    __slots__ = ('d', 'keep', 'out_hw', 'ref', 'dyn', 'maps')

    def __init__(self, d, keep, out_hw):
        self.d, self.keep, self.out_hw = d, keep, out_hw
        self.ref = C.byref(d)
        self.dyn = {}           # descriptor field -> tensor it currently points at (rebinding overwrites, never appends)
        self.maps = None

    def encode_act_maps(self):
        """(Re-)encode the activation tensor maps (hd_conv_desc.tmap_res etc.) for the pointers currently in the descriptor.
        The sm_90a kernel does not read them; hd_conv_gemm accepts out_subsample only with them (and HD_CONV_NO_TMA_EPILOGUE unset),
        the C-ABI rule of hd_b200.h.  Layers that qualify: fp16-split input, Cout % 32 == 0, residual row == output row."""
        d = self.d
        K = d.KH * d.KW * d.Cin
        ok = (d.impl in (_lib.HD_IMPL_TC_3XF16, _lib.HD_IMPL_TC_1XF16) and d.in_hi and d.Cout % 32 == 0 and
              (not d.res or (d.res_stride == 1 and d.res_H == d.Ho and d.res_W == d.Wo)))
        for f in ('tmap_res', 'tmap_out', 'tmap_out_hi', 'tmap_out_lo'):
            setattr(d, f, None)
        if not ok:
            return
        M = d.n_img * d.Ho * d.Wo
        if self.maps is None:
            self.maps = {f: (C.c_ubyte * 128)() for f in ('res', 'out', 'out_hi', 'out_lo')}
        for f, ptr, ld, eb in (('res', d.res, d.res_ld, 4), ('out', d.out, d.out_ld, 4), ('out_hi', d.out_hi, d.out2_ld, 2),
                               ('out_lo', d.out_lo, d.out2_ld, 2)):
            if not ptr or (f == 'out' and d.out_subsample > 1):
                continue
            if ptr % 16 or (ld * eb) % 16:
                for g in ('tmap_res', 'tmap_out', 'tmap_out_hi', 'tmap_out_lo'):
                    setattr(d, g, None)
                return
            check(lib.hd_make_act_tmap(C.c_void_p(ptr), M, d.Cout, ld, eb, C.cast(self.maps[f], C.c_void_p)), 'hd_make_act_tmap')
            setattr(d, 'tmap_' + f, C.cast(self.maps[f], C.c_void_p))

    def rebind(self, field, tensor):
        """Point one descriptor field at another tensor (stage input / output of a cached plan)."""
        setattr(self.d, field, tensor.data_ptr())
        self.dyn[field] = tensor

    def run(self, stream):
        rc = lib.hd_conv_gemm(self.ref, stream)
        if rc:
            check(rc, 'hd_conv_gemm')


class ChainOp(object):
    """conv3 of a unit and conv1 of the identity unit after it in one launch (hd_conv_gemm_chain): the pre-activated pair conv3 hands to
    conv1 stays in shared memory.  `d` / `ref` are conv3's descriptor, so the op reads as that conv to code that walks a plan's convs."""
    __slots__ = ('first', 'second', 'd', 'ref')

    def __init__(self, first, second):
        self.first, self.second = first, second
        self.d, self.ref = first.d, first.ref

    @staticmethod
    def bind(first, second):
        """The chain of two bound ConvOps (conv3 writing the pair that conv1 reads), or None when the library does not run the pair as
        one launch; then both ops are left as they were."""
        d3, d1 = first.d, second.d
        saved = (d3.out_hi, d3.out_lo, d1.in_hi, d1.in_lo)
        d3.out_hi = d3.out_lo = d1.in_hi = d1.in_lo = None
        if lib.hd_conv_gemm_chain_supported(first.ref, second.ref) == 1:
            first.encode_act_maps()
            return ChainOp(first, second)
        d3.out_hi, d3.out_lo, d1.in_hi, d1.in_lo = saved
        return None

    def rebind(self, field, tensor):
        self.first.rebind(field, tensor)

    def encode_act_maps(self):
        self.first.encode_act_maps()
        self.second.encode_act_maps()

    def run(self, stream):
        rc = lib.hd_conv_gemm_chain(self.first.ref, self.second.ref, stream)
        if rc:
            check(rc, 'hd_conv_gemm_chain')


class PackedConv1Planes(object):
    """ResNet root conv1 (7x7 stride 2, explicit pad 3+3, bias; A.2) on the tensor cores, reading its input as two padded
    RGBX fp16 planes [n, S+6, WP, 4] (head / remainder, hd_pack_conv1_planes): every (output pixel, kernel row) needs 8
    consecutive pixels = 64 contiguous, 16-byte-aligned bytes per plane, which four cp.async move straight into the swizzled
    A tile.  GEMM view: K = 8 kernel rows x 8 pixels x 4 channels = 256 (the 8th row / pixel / channel carry zero weights)."""

    def __init__(self, w_hwio, bias, device):
        # w_hwio: a host array, or a device tensor (a trainable weight) that `repack` reads again
        w = w_hwio if isinstance(w_hwio, torch.Tensor) else torch.from_numpy(np.asarray(w_hwio, np.float32))
        assert tuple(w.shape) == (7, 7, 3, 64), tuple(w.shape)
        self.device = device
        self.w = w
        self.Cout, self.K = 64, 256
        self.wp = torch.zeros((8, 8, 4, 64), dtype=torch.float32, device=device)    # [ky, kx, c, co]: K index ky*32 + kx*4 + c
        self.w_nk_hi = torch.empty((64, 256), dtype=torch.float16, device=device)
        self.w_nk_lo = torch.empty((64, 256), dtype=torch.float16, device=device)
        if _packs_on(device):
            self.repack(current_stream())
        self.bias = _dev(bias, device)
        self.tmap_hi, self.tmap_lo = weight_tmap(self.w_nk_hi), weight_tmap(self.w_nk_lo)

    def repack(self, stream):
        """Rewrite the packs on `stream` from the current weight (through the zero-padded [8, 8, 4, 64] layout)."""
        self.wp[:7, :7, :3].copy_(self.w)
        pack_weight(self.wp, 8, 32, 64, self.w_nk_hi, self.w_nk_lo, stream)

    @staticmethod
    def plane_width(size):
        return (size + 8 + 1) // 2 * 2

    def alloc_planes(self, n, size, impl='auto'):
        """Zero-initialised planes: the 3-pixel border (and the spare columns) must be zero and is never written again.  'tc1h': the
        head plane alone, (hi, None)."""
        shape = (n, size + 6, self.plane_width(size), 4)
        hi = torch.zeros(shape, dtype=torch.float16, device=self.device)
        return (hi, None) if heads_only(impl) else (hi, torch.zeros(shape, dtype=torch.float16, device=self.device))

    def bind(self, planes, n, size, out, impl='auto'):
        d = ConvDesc()
        WP = self.plane_width(size)
        heads = heads_only(impl)
        d.in_hi = planes[0].data_ptr()
        if not heads:
            d.in_lo = planes[1].data_ptr()
        d.in_ld = 4
        d.n_img, d.H, d.W, d.Cin = n, size + 6, WP, 32
        d.Ho = d.Wo = size // 2
        d.KH, d.KW, d.stride, d.pad_t, d.pad_l = 8, 1, 2, 0, 0
        d.Cout, d.K_pad = 64, 256
        d.post_shift = self.bias.data_ptr()
        d.out, d.out_ld = out.data_ptr(), 64
        d.impl = _lib.HD_IMPL_TC_1XF16 if heads else _lib.HD_IMPL_TC_3XF16
        d.w_nk_hi, d.tmap_hi = self.w_nk_hi.data_ptr(), C.cast(self.tmap_hi, C.c_void_p)
        if not heads:
            d.w_nk_lo, d.tmap_lo = self.w_nk_lo.data_ptr(), C.cast(self.tmap_lo, C.c_void_p)
        d.flags = _lib.HD_CONV_INPUT_PLANES
        op = ConvOp(d, (self, planes, out), (size // 2, size // 2))
        op.encode_act_maps()
        return op


# ------------------------------------------------------------------------------------------------
# ResNet-v2-50 (slim)  -- src/models.py:50-77
# ------------------------------------------------------------------------------------------------
class PackedResNet(object):
    def __init__(self, w, device, tc=False, blocks=RESNET_BLOCKS):
        p = 'resnet_v2_50'
        self.device = device
        self.blocks = blocks
        w1 = w[p + '/conv1/weights']          # a device tensor (a trainable weight) is read in place, like PackedConv's
        self.conv1_w = w1.reshape(147, 64) if isinstance(w1, torch.Tensor) else _dev(np.asarray(w1, np.float32).reshape(147, 64), device)
        self.conv1_b = _dev(w[p + '/conv1/biases'], device)
        # conv2d_same(7x7, stride 2): explicit pad 3+3 then VALID (A.2); tensor-core path gathers the ragged K=147 element-wise
        self.conv1 = PackedConv(w[p + '/conv1/weights'], device, post_shift=w[p + '/conv1/biases'], stride=2, pad=(3, 3), tc=tc)
        want = {True: 'f16', 'auto': 'f16', 'tc3h': 'f16', 'tc1h': 'f16'}.get(tc, None)
        self.conv1_planes = PackedConv1Planes(w[p + '/conv1/weights'], w[p + '/conv1/biases'], device) if want == 'f16' else None
        self.units = []
        d_in = 64
        for b, (base, units, bstride) in enumerate(blocks, start=1):
            depth = 4 * base
            for u in range(1, units + 1):
                q = '%s/block%d/unit_%d/bottleneck_v2' % (p, b, u)
                stride = bstride if u == units else 1
                ps, pb = fold_bn(w, q + '/preact')
                unit = {'stride': stride, 'base': base, 'depth': depth, 'd_in': d_in,
                        'pre': (_dev(ps, device), _dev(pb, device))}
                if d_in != depth:
                    unit['shortcut'] = PackedConv(w[q + '/shortcut/weights'], device,
                                                  post_shift=w[q + '/shortcut/biases'], stride=stride, tc=tc)
                s1, b1 = fold_bn(w, q + '/conv1/BatchNorm')
                unit['conv1'] = PackedConv(w[q + '/conv1/weights'], device, s1, b1, True, tc=tc)
                s2, b2 = fold_bn(w, q + '/conv2/BatchNorm')
                # conv2d_same: stride 1 -> SAME (pad 1); stride 2 -> explicit pad 1+1 then VALID  (A.2)
                unit['conv2'] = PackedConv(w[q + '/conv2/weights'], device, s2, b2, True, stride=stride, pad=(1, 1), tc=tc)
                unit['conv3'] = PackedConv(w[q + '/conv3/weights'], device, post_shift=w[q + '/conv3/biases'], tc=tc)
                self.units.append(unit)
                d_in = depth
        s, b = fold_bn(w, p + '/postnorm')
        self.post = (_dev(s, device), _dev(b, device))
        self.out_dim = d_in
        sync_packing(device)


def bind_root_conv1(packed: PackedResNet, n, size, impl, out):
    """The root conv1 of a trunk plan writing `out` (the plan's root_buf) -> (planes, op): in the fp16 impls at an even size, the
    padded fp16 planes and their PackedConv1Planes op; else, when conv1 has a tensor-core packing and impl is not 'simt', (None, the
    row-segment gather op, the only tensor-core conv1 at odd sizes; its `in_` is set per run); else (None, None): hd_conv1_7x7s2."""
    if packed.conv1_planes is not None and impl in F16_IMPLS and size % 2 == 0:
        planes = packed.conv1_planes.alloc_planes(n, size, impl)
        return planes, packed.conv1_planes.bind(planes, n, size, out, impl)
    if packed.conv1.tc and impl != 'simt':
        return None, packed.conv1.bind(out, n, size, size, out, in_ld=3, impl=impl)
    return None, None


def run_root_conv1(plan, images, st):
    """Run the root conv1 that bind_root_conv1 gave `plan` (its planes, conv1_op, root_buf) over images (n,size,size,3) contiguous
    float32; images None: the planes were filled by the caller (uint8 frames through hd_process_image)."""
    n, size = plan.n, plan.size
    if plan.planes is not None:
        if images is not None:
            check(lib.hd_pack_conv1_planes(fptr(images), _vp(plan.planes[0]), _vp(plan.planes[1]), n, size, size,
                                           plan.planes[0].shape[2], st), 'hd_pack_conv1_planes')
        plan.conv1_op.run(st)
    elif plan.conv1_op is not None:
        plan.conv1_op.d.in_ = images.data_ptr()
        plan.conv1_op.run(st)
    else:
        check(lib.hd_conv1_7x7s2(fptr(images), fptr(plan.p.conv1_w), fptr(plan.p.conv1_b), fptr(plan.root_buf), n, size, size, st),
              'hd_conv1_7x7s2')


class ResNetPlan(object):
    """Forward plan for a fixed number of frames n (activation buffers are reused across chunks).

    `units=(lo, hi)` restricts the plan to bottleneck units [lo, hi) so the trunk can be run in two stages with
    different frame counts: the early blocks have thousands of tiles per layer at any batch, the late blocks
    (14x14 / 7x7 maps) only fill the 132 SMs when many frames are batched (wave quantisation, DESIGN.md).
    root=True prepends conv1 + pool1; tail=True appends postnorm + global mean.
    """

    def __init__(self, packed: PackedResNet, n, size=224, impl='auto', units=None, root=True, tail=True, next_pre=None,
                 next_has_shortcut=False):
        self.p = packed
        self.n = n
        self.size = size
        self.root, self.tail = root, tail
        dev = packed.device
        lo, hi = units if units is not None else (0, len(packed.units))
        H1 = size // 2                        # conv1 output (explicit pad 3, stride 2)
        H2 = (H1 + 1) // 2                    # pool1 SAME
        self.H1, self.H2 = H1, H2
        # spatial size / depth entering unit `lo`
        H, d_in = H2, 64
        for unit in packed.units[:lo]:
            H = (H - 1) // unit['stride'] + 1
            d_in = unit['depth']
        self.in_hw, self.in_depth = H, d_in
        # buffer sizes (floats per frame) needed by units [lo, hi)
        mx_io, mx_r = H * H * d_in, 0
        h = H
        for unit in packed.units[lo:hi]:
            ho = (h - 1) // unit['stride'] + 1
            mx_io = max(mx_io, h * h * unit['depth'] if 'shortcut' in unit else 0, ho * ho * unit['depth'])
            mx_r = max(mx_r, h * h * unit['base'])
            h = ho
        if root:
            mx_io = max(mx_io, H1 * H1 * 64)
        f32 = dict(dtype=torch.float32, device=dev)
        f16 = dict(dtype=torch.float16, device=dev)
        # split mode: every conv reads its A operand as a pre-activated fp16 head/remainder pair written by the producing
        # epilogue (cp.async straight into the swizzled tile, DESIGN.md 4.1); fp32 copies exist only where a residual needs them
        self.impl = impl
        self.split = impl in F16_IMPLS and all(
            c.tc == 'f16' and not c.gather for u in packed.units[lo:hi] for k, c in u.items() if isinstance(c, PackedConv))
        self.bufA = torch.empty(n * mx_io, **f32)
        self.bufB = torch.empty(n * mx_io, **f32)
        self.bufS = torch.empty(n * mx_io, **f32)
        self.ops = []
        self.root_buf = self.bufS             # conv1 output, read by pool1
        self.planes, self.conv1_op = bind_root_conv1(packed, n, size, impl, self.root_buf) if root else (None, None)
        self.in_refs = []                     # (op, field) descriptor fields that read the stage input
        self.pool_split = None
        self.pool_f32_dead = False
        x, y = self.bufA, self.bufB
        units = packed.units[lo:hi]
        if self.split:
            def pair(count):                  # 'tc1h': heads only, (hi, None)
                return f16_pair(max(1, count), dev, impl)
            xs, ys = pair(n * mx_io), pair(n * mx_io)
            r1, r2 = pair(n * mx_r), pair(n * mx_r)
            self.in_split = xs
            if root:
                self.pool_split = (units[0]['pre'][0], units[0]['pre'][1], xs)
                self.pool_f32_dead = 'shortcut' in units[0]
            self.out_split = None
            sub_ready = False                 # bufS already holds x[:, ::s, ::s] of this unit's input (written by the previous conv3)
            for ui, unit in enumerate(units):
                s = unit['stride']
                Ho = (H - 1) // s + 1
                if 'shortcut' in unit:
                    self.ops.append(unit['shortcut'].bind(None, n, H, H, self.bufS, inp_split=xs, impl=impl))
                    if ui == 0:
                        self.in_refs += self._split_refs(self.ops[-1])
                    res, res_geom = self.bufS, (unit['depth'], Ho, Ho, 1)
                elif s > 1:
                    # strided identity shortcut: a dense subsampled copy so conv3's residual is row-aligned (TMA slab loads) -- written by
                    # the previous unit's conv3 epilogue when that unit is in this plan, else by one hd_subsample pass
                    if not sub_ready:
                        self.ops.append(SubsampleOp(x, self.bufS[:n * Ho * Ho * unit['depth']], n, H, unit['depth'], s))
                        if ui == 0:
                            self.in_refs.append((self.ops[-1], 'res', 2))
                    res, res_geom = self.bufS, (unit['depth'], Ho, Ho, 1)
                else:
                    res, res_geom = x, (unit['depth'], H, H, 1)
                conv1 = unit['conv1'].bind(None, n, H, H, None, inp_split=xs, out_split=r1, impl=impl)
                # an identity unit's conv1 reads only the pair the previous conv3 writes: one launch for both where the library runs it
                chain = ChainOp.bind(self.ops[-1], conv1) if ui > 0 and 'shortcut' not in unit and isinstance(self.ops[-1], ConvOp) else None
                if chain is not None:
                    self.ops[-1] = chain
                else:
                    self.ops.append(conv1)
                if ui == 0:
                    self.in_refs += self._split_refs(self.ops[-1])
                self.ops.append(unit['conv2'].bind(None, n, H, H, None, inp_split=r1, out_split=r2, impl=impl))
                last = ui == len(units) - 1
                nxt = units[ui + 1]['pre'] if not last else next_pre        # the next unit's pre-activation BN (+ReLU)
                osplit = ys if nxt is not None else None
                # the fp32 block output only feeds an IDENTITY shortcut: when the next unit changes depth (first unit of a block) its
                # shortcut is a conv of the pre-activation, and the fp32 copy would be written for nobody
                nxt_conv_shortcut = ('shortcut' in units[ui + 1]) if not last else bool(next_has_shortcut)
                y_out = None if nxt_conv_shortcut else y
                # the next unit is a strided identity unit: the only reader of this unit's fp32 output is that shortcut, x[:, ::s, ::s]
                # -- write just those pixels, densely, into bufS (free here: this unit's own residual is not in bufS)
                s_next = units[ui + 1]['stride'] if not last else 1
                sub_ready = not last and s_next > 1 and not nxt_conv_shortcut and 'shortcut' not in unit and s == 1
                if sub_ready:
                    y_out = self.bufS
                self.ops.append(unit['conv3'].bind(None, n, Ho, Ho, y_out, inp_split=r2, res=res, res_geom=res_geom, impl=impl,
                                                   out_split=osplit, post2=(nxt[0], nxt[1], 1) if nxt is not None else None,
                                                   out_subsample=s_next if sub_ready else 0))
                if ui == 0 and 'shortcut' not in unit and s == 1:
                    self.in_refs.append((self.ops[-1], 'res', 2))
                if last:
                    self.out_split = osplit
                x, y = y, x
                xs, ys = ys, xs
                H = Ho
                d_in = unit['depth']
        else:
            self.bufR1 = torch.empty(max(1, n * mx_r), **f32)
            self.bufR2 = torch.empty(max(1, n * mx_r), **f32)
            for ui, unit in enumerate(units):
                s = unit['stride']
                Ho = (H - 1) // s + 1
                pre = (unit['pre'][0], unit['pre'][1], 0, 1)
                if 'shortcut' in unit:
                    self.ops.append(unit['shortcut'].bind(x, n, H, H, self.bufS, pre=pre, impl=impl))
                    if ui == 0:
                        self.in_refs.append((self.ops[-1], 'in_', 2))
                    res, res_geom = self.bufS, (unit['depth'], Ho, Ho, 1)
                else:
                    res, res_geom = x, (unit['depth'], H, H, s)      # identity, or max_pool2d(1x1, stride) = subsample
                self.ops.append(unit['conv1'].bind(x, n, H, H, self.bufR1, pre=pre, impl=impl))
                if ui == 0:
                    self.in_refs.append((self.ops[-1], 'in_', 2))
                self.ops.append(unit['conv2'].bind(self.bufR1, n, H, H, self.bufR2, impl=impl))
                self.ops.append(unit['conv3'].bind(self.bufR2, n, Ho, Ho, y, res=res, res_geom=res_geom, impl=impl))
                if ui == 0 and 'shortcut' not in unit:
                    self.in_refs.append((self.ops[-1], 'res', 2))
                x, y = y, x
                H = Ho
                d_in = unit['depth']
        self.final = x
        self.final_hw = H * H
        self.out_hw, self.out_depth = H, d_in
        self.in_buf = self.bufA               # stage input when root=False

    def _split_refs(self, op):
        """in_refs entries of a conv that reads the stage input's pair (its head only in the 'tc1h' mode)."""
        return [(op, 'in_hi', 0)] + ([] if heads_only(self.impl) else [(op, 'in_lo', 1)])

    def set_input(self, t, t_split=None):
        """Point the stage at an external input feature map [n, in_hw, in_hw, in_depth] (fp32 `t`, and in split mode its
        pre-activated fp16 pair `t_split`); no copy."""
        srcs = (t_split[0] if t_split else None, t_split[1] if t_split else None, t)
        for op, field, which in self.in_refs:
            src = srcs[which]
            if src is None:
                raise _lib.HDError('stage input %s missing' % field)
            op.rebind(field, src)
        for op in {id(o): o for o, _, _ in self.in_refs}.values():
            op.encode_act_maps()

    def set_output(self, t, t_split=None):
        """Let the last unit write its output feature map [n, out_hw, out_hw, out_depth] straight into `t` (and, in split
        mode, the next stage's pre-activated pair into `t_split`)."""
        op = self.ops[-1]
        if op.d.out:                          # (no fp32 output when the consumer's shortcut is a conv)
            op.rebind('out', t)
        if t_split is not None:
            op.rebind('out_hi', t_split[0])
            if t_split[1] is not None:
                op.rebind('out_lo', t_split[1])
        op.encode_act_maps()
        self.final = t

    def run(self, images, out, stream=None):
        """root=True: images (n,size,size,3) contiguous float32 CUDA view; else `images` is ignored and the stage
        input must already be in `in_buf` ([n, in_hw, in_hw, in_depth]).  tail=True: out = phi (n,2048) view;
        else the stage output feature map is left in `self.final`."""
        st = current_stream() if stream is None else stream
        n, p = self.n, self.p
        if self.root:
            run_root_conv1(self, images, st)
            ps = self.pool_split
            check(lib.hd_maxpool3x3s2_same(fptr(self.root_buf), None if self.pool_f32_dead else fptr(self.bufA), n, self.H1, self.H1, 64,
                                           fptr(ps[0]) if ps else None, fptr(ps[1]) if ps else None,
                                           _vp(ps[2][0]) if ps else None, _vp(ps[2][1]) if ps else None, st), 'hd_maxpool3x3s2_same')
        for op in self.ops:
            op.run(st)
        if self.tail:
            check(lib.hd_bnrelu_avgpool(fptr(self.final), fptr(p.post[0]), fptr(p.post[1]), fptr(out), n, self.final_hw,
                                        p.out_dim, st), 'hd_bnrelu_avgpool')

    @property
    def num_launches(self):
        return ((3 if self.planes is not None else 2) if self.root else 0) + len(self.ops) + (1 if self.tail else 0)


# ------------------------------------------------------------------------------------------------
# ResNet-v2-50 in training mode (is_training=True: batch statistics) -- src/models.py:50-77 as trainer_sequence_fc.py:562-575 calls it
# ------------------------------------------------------------------------------------------------
def resnet_bn_scopes(blocks=RESNET_BLOCKS):
    """The trunk's 49 batch-norm scopes in the order a forward pass meets them: per unit preact, conv1/BatchNorm, conv2/BatchNorm; then
    postnorm."""
    p = 'resnet_v2_50'
    out = []
    for b, (_, units, _) in enumerate(blocks, start=1):
        for u in range(1, units + 1):
            q = '%s/block%d/unit_%d/bottleneck_v2' % (p, b, u)
            out += [q + '/preact', q + '/conv1/BatchNorm', q + '/conv2/BatchNorm']
    return out + [p + '/postnorm']


class ResNetBatchNorm(object):
    """gamma, beta and the moving statistics of the trunk's batch-norm layers, each a flat device vector with one slice per scope
    (`scopes` order, `offsets`).  Training-mode plans read gamma / beta and step moving_mean / moving_variance in place."""

    def __init__(self, w, device, blocks=RESNET_BLOCKS):
        self.device = device
        self.scopes = resnet_bn_scopes(blocks)
        missing = [s + '/' + k for s in self.scopes for k in ('gamma', 'beta', 'moving_mean', 'moving_variance') if s + '/' + k not in w]
        if missing:
            raise _lib.HDError('training-mode ResNet: weights lack %d batch-norm variables, e.g. %s' % (len(missing), missing[0]))
        self.sizes = [int(np.size(w[s + '/gamma'])) for s in self.scopes]
        self.offsets = [0] + [int(v) for v in np.cumsum(self.sizes)]

        def flat(k):
            return _dev(np.concatenate([np.asarray(w[s + '/' + k], np.float32).reshape(-1) for s in self.scopes]), device)
        self.gamma, self.beta = flat('gamma'), flat('beta')
        self.moving_mean, self.moving_variance = flat('moving_mean'), flat('moving_variance')

    def view(self, t, i):
        return t[self.offsets[i]:self.offsets[i + 1]]

    def moving(self):
        """{'<scope>/moving_mean' | '<scope>/moving_variance': float32 ndarray}, copied to the host."""
        mm, mv = self.moving_mean.cpu().numpy(), self.moving_variance.cpu().numpy()
        out = {}
        for i, s in enumerate(self.scopes):
            a, b = self.offsets[i], self.offsets[i + 1]
            out[s + '/moving_mean'], out[s + '/moving_variance'] = mm[a:b].copy(), mv[a:b].copy()
        return out


class BatchStatsOp(object):
    """hd_bn_batch_stats over one [rows, C] map: one op in a training plan's op list, writing the scale / shift the next layers'
    prologue (or the tail) applies and the layer's batch mean / biased variance."""
    __slots__ = ('x', 'rows', 'C', 'gamma', 'beta', 'scale', 'shift', 'mean', 'var', 'ws', 'd')

    def __init__(self, x, rows, C, gamma, beta, scale, shift, mean, var, ws):
        self.x, self.rows, self.C = x, rows, C
        self.gamma, self.beta, self.scale, self.shift, self.mean, self.var, self.ws = gamma, beta, scale, shift, mean, var, ws
        self.d = None

    def encode_act_maps(self):
        pass

    def run(self, stream):
        check(lib.hd_bn_batch_stats(fptr(self.x), self.rows, self.C, self.C, fptr(self.gamma), fptr(self.beta), BN_EPS, fptr(self.scale),
                                    fptr(self.shift), fptr(self.mean), fptr(self.var), None, None, 0.0, C.c_void_p(self.ws.data_ptr()),
                                    self.ws.numel(), stream), 'hd_bn_batch_stats')


class ResNetTrainPlan(object):
    """Training-mode forward of the whole trunk over n frames (slim resnet_v2_50 with is_training=True, no dropout on this path): every
    batch norm normalises with the moments of the current batch over all n frames x H x W.  The fp32 layer chain of ResNetPlan with
    the batch statistics of each map taken right before the layers that apply them:

      root   conv1 + pool1 exactly as in the inference plan (no batch norm there)
      unit   stats(x) -> preact scale/shift, applied (+ReLU) in the A producer of the shortcut conv and of conv1; conv1 writes raw fp32;
             stats -> conv2's prologue (padded 3x3, strided in a block's last unit); conv2 writes raw; stats -> conv3's prologue;
             conv3 adds its bias and the residual (the identity shortcut reads the raw unit input, as slim does)
      tail   stats(final map) -> hd_bnrelu_avgpool's scale / shift

    49 BatchStatsOps.  The scale / shift / mean / variance vectors are plan-owned device buffers rewritten on every run, so the
    descriptors never change.  `run` leaves the moving statistics alone; `apply_moving_update` takes the one step of the update ops
    from this run's moments.

    keep=True (training the trunk, freeze_phi=False): the layer chain writes every map the backward reads into its own buffer -- the root
    conv1 output, each unit's input and its raw conv1 / conv2 outputs -- instead of ping-ponging (about 32 MB per frame at 224 x 224);
    the kernels, descriptors and arithmetic are the same, so the phis are bit-identical to keep=False.  `backward(dphi, images)` then
    walks the units in reverse (csrc/resnet_grad.cu + hd_conv_gemm 3xTF32); it needs a `bwd` data-gradient pack on every conv but the
    root's (trunk.TrainableResNet sets them).  grad_precision='tf32' runs the backward's weight and data gradients in 1xTF32 instead
    (GRAD_PRECISIONS); the forward is the same either way."""

    def __init__(self, packed: PackedResNet, bn: ResNetBatchNorm, n, size=224, impl='auto', keep=False, grad_precision='fp32'):
        require_training_impl(impl, 'ResNetTrainPlan')
        self.one_pass = grad_one_pass(grad_precision, 'ResNetTrainPlan')
        self.grad_precision = grad_precision
        self.p, self.bn, self.n, self.size, self.keep = packed, bn, n, size, bool(keep)
        self.generation = 0                   # runs so far: a recorded graph checks that its saved maps are still the plan's
        dev = packed.device
        H1 = size // 2
        H2 = (H1 + 1) // 2
        self.H1, self.H2 = H1, H2
        mx_io, mx_r, h = max(H1 * H1 * 64, H2 * H2 * 64), 0, H2
        for unit in packed.units:
            ho = (h - 1) // unit['stride'] + 1
            mx_io = max(mx_io, h * h * unit['depth'], ho * ho * unit['depth'])
            mx_r = max(mx_r, h * h * unit['base'])
            h = ho
        f32 = dict(dtype=torch.float32, device=dev)
        self.mx_io, self.mx_r = mx_io, mx_r
        if self.keep:                         # one buffer per kept map; bufS only carries the shortcut convs' outputs
            self.bufS = torch.empty(n * mx_io, **f32)
            self.root_out = torch.empty(n * H1 * H1 * 64, **f32)
            self.xs, self.r1s, self.r2s, h = [torch.empty(n * H2 * H2 * 64, **f32)], [], [], H2
            for unit in packed.units:
                ho = (h - 1) // unit['stride'] + 1
                self.r1s.append(torch.empty(n * h * h * unit['base'], **f32))
                self.r2s.append(torch.empty(n * ho * ho * unit['base'], **f32))
                self.xs.append(torch.empty(n * ho * ho * unit['depth'], **f32))
                h = ho
        else:
            self.bufA, self.bufB, self.bufS = (torch.empty(n * mx_io, **f32) for _ in range(3))
            self.bufR1, self.bufR2 = torch.empty(n * mx_r, **f32), torch.empty(n * mx_r, **f32)
        self.root_buf = self.root_out if self.keep else self.bufS
        L = bn.offsets[-1]
        self.scale, self.shift, self.mean, self.var = (torch.empty(L, **f32) for _ in range(4))
        self.planes, self.conv1_op = bind_root_conv1(packed, n, size, impl, self.root_buf)
        self.ops, self.stats = [], []
        shapes = []                           # (map, rows, C) of every normalised map, in scope order
        h = H2
        for unit in packed.units:
            ho = (h - 1) // unit['stride'] + 1
            shapes += [(n * h * h, unit['d_in']), (n * h * h, unit['base']), (n * ho * ho, unit['base'])]
            h = ho
        shapes.append((n * h * h, packed.out_dim))
        ws_bytes = max(int(lib.hd_bn_stats_workspace_bytes(rows, Cc)) for rows, Cc in shapes)
        self.ws = torch.empty(max(16, ws_bytes), dtype=torch.uint8, device=dev)

        def stats(x, rows, Cc):
            i = len(self.stats)
            assert (rows, Cc) == shapes[i], (i, rows, Cc, shapes[i])
            v = lambda t: bn.view(t, i)          # noqa: E731
            op = BatchStatsOp(x, rows, Cc, v(bn.gamma), v(bn.beta), v(self.scale), v(self.shift), v(self.mean), v(self.var), self.ws)
            self.ops.append(op)
            self.stats.append(op)
            return (op.scale, op.shift, 0, 1)

        raw = (None, None, False)
        x, y, H = (self.xs[0], None, H2) if self.keep else (self.bufA, self.bufB, H2)
        self.pool_out = x
        for ui, unit in enumerate(packed.units):
            s = unit['stride']
            Ho = (H - 1) // s + 1
            if self.keep:
                x, y, self.bufR1, self.bufR2 = self.xs[ui], self.xs[ui + 1], self.r1s[ui], self.r2s[ui]
            pre = stats(x, n * H * H, unit['d_in'])
            if 'shortcut' in unit:
                self.ops.append(unit['shortcut'].bind(x, n, H, H, self.bufS, pre=pre, impl=impl))
                res, res_geom = self.bufS, (unit['depth'], Ho, Ho, 1)
            else:
                res, res_geom = x, (unit['depth'], H, H, s)      # identity, or max_pool2d(1x1, stride) = subsample, of the raw input
            self.ops.append(unit['conv1'].bind(x, n, H, H, self.bufR1, pre=pre, impl=impl, post=raw))
            pre1 = stats(self.bufR1, n * H * H, unit['base'])
            self.ops.append(unit['conv2'].bind(self.bufR1, n, H, H, self.bufR2, pre=pre1, impl=impl, post=raw))
            pre2 = stats(self.bufR2, n * Ho * Ho, unit['base'])
            self.ops.append(unit['conv3'].bind(self.bufR2, n, Ho, Ho, y, pre=pre2, res=res, res_geom=res_geom, impl=impl))
            x, y = y, x
            H = Ho
        self.final, self.final_hw = x, H * H
        self.tail = stats(x, n * H * H, packed.out_dim)
        assert len(self.stats) == len(bn.scopes)
        self._bwd = None

    def run(self, images, out, stream=None):
        """images (n,size,size,3) contiguous float32 CUDA NHWC in [-1, 1] (None: the conv1 planes were filled by the caller) -> out
        (n,2048) float32 view: the phis with batch statistics.  The moving statistics are not touched."""
        st = current_stream() if stream is None else stream
        n, p = self.n, self.p
        run_root_conv1(self, images, st)
        check(lib.hd_maxpool3x3s2_same(fptr(self.root_buf), fptr(self.pool_out), n, self.H1, self.H1, 64, None, None, None, None, st),
              'hd_maxpool3x3s2_same')
        self.generation += 1
        for op in self.ops:
            op.run(st)
        check(lib.hd_bnrelu_avgpool(fptr(self.final), fptr(self.tail[0]), fptr(self.tail[1]), fptr(out), n, self.final_hw, p.out_dim, st),
              'hd_bnrelu_avgpool')

    def apply_moving_update(self, decay=BN_DECAY, stream=None):
        """One step of the 49 layers' update ops from the moments of the last `run`: bn.moving_mean / moving_variance in place."""
        st = current_stream() if stream is None else stream
        bn = self.bn
        for i, op in enumerate(self.stats):
            check(lib.hd_bn_moving_update(fptr(op.mean), fptr(op.var), op.rows, op.C, float(decay), fptr(bn.view(bn.moving_mean, i)),
                                          fptr(bn.view(bn.moving_variance, i)), st), 'hd_bn_moving_update')

    def moments(self):
        """{scope: (batch mean, biased batch variance)} of the last `run`, device views."""
        return {s: (op.mean, op.var) for s, op in zip(self.bn.scopes, self.stats)}

    @property
    def num_launches(self):
        return (3 if self.planes is not None else 2) + sum(2 if isinstance(op, BatchStatsOp) else 1 for op in self.ops) + 1

    # ---------------------------------------------------------------------------------------------------------------------------- backward
    def unit_scopes(self):
        """The variable scope of every bottleneck unit, in order."""
        return ['resnet_v2_50/block%d/unit_%d/bottleneck_v2' % (b, u) for b, (_, units, _) in enumerate(self.p.blocks, start=1)
                for u in range(1, units + 1)]

    @property
    def num_backward_launches(self):
        """Kernel launches of one `backward`: 3 per batch-norm backward, 2 per weight gradient, 1 per data-gradient GEMM, zero
        insertion and pool1 backward."""
        out = 3 + 1 + 2                       # the tail's batch norm; pool1; the root conv's weight gradient
        for unit in self.p.units:
            out += 3 * 3 + 3 * 2 + 3 + (1 if unit['stride'] > 1 else 0) + (3 if 'shortcut' in unit else 0)
        return out

    def _backward_state(self):
        """Scratch maps, workspaces and the data-gradient descriptors of `backward` (hd_conv_gemm over each conv's `bwd` pack),
        made on the first call; every pointer is plan-owned, so the descriptors never change."""
        if self._bwd is not None:
            return self._bwd
        if not self.keep:
            raise _lib.HDError('ResNetTrainPlan.backward needs a plan built with keep=True (the maps the backward reads)')
        p, n = self.p, self.n
        f32 = dict(dtype=torch.float32, device=p.device)
        G = [torch.empty(n * self.mx_io, **f32) for _ in range(2)]        # gradients of the unit outputs / inputs, alternating
        D1, D2, Z = (torch.empty(n * self.mx_r, **f32) for _ in range(3))
        P = torch.empty(n * self.mx_io, **f32)
        ws_w = lib.hd_conv_wgrad_workspace_bytes(n * self.H1 * self.H1, 147, 64, 1)
        ws_b = max(int(lib.hd_bn_relu_backward_workspace_bytes(op.rows, op.C)) for op in self.stats)
        ops, H, U = [], self.H2, len(p.units)
        for ui, unit in enumerate(p.units):
            s, base, depth, d_in = unit['stride'], unit['base'], unit['depth'], unit['d_in']
            Ho = (H - 1) // s + 1
            for c in ('conv1', 'conv2', 'conv3', 'shortcut'):
                if c in unit and getattr(unit[c], 'bwd', None) is None:
                    raise _lib.HDError('ResNetTrainPlan.backward: %s of unit %d has no data-gradient pack' % (c, ui))
            if 'shortcut' in unit and s != 1:
                raise _lib.HDError('ResNetTrainPlan.backward: a strided shortcut conv is not part of resnet_v2_50')
            k = U - 1 - ui
            gy, gx = G[k % 2], G[(k + 1) % 2]
            for pix, K, Cout, bias in ((Ho * Ho, base, depth, 1), (Ho * Ho, 9 * base, base, 0), (H * H, d_in, base, 0),
                                       (H * H, d_in, depth, 1)):
                ws_w = max(ws_w, lib.hd_conv_wgrad_workspace_bytes(n * pix, K, Cout, bias))
            u = {'gy': gy, 'gx': gx, 'H': H, 'Ho': Ho}
            op = self.one_pass
            u['conv3'] = dgrad_op(unit['conv3'].bwd, gy, n, Ho, Ho, 1, 1, D1, one_pass=op)
            u['conv2'] = dgrad_op(unit['conv2'].bwd, D2 if s == 1 else Z, n, H, H, 3, 3, D1, one_pass=op)
            if 'shortcut' in unit:
                u['shortcut'] = dgrad_op(unit['shortcut'].bwd, gy, n, H, H, 1, 1, P, one_pass=op)
                u['conv1'] = dgrad_op(unit['conv1'].bwd, D2, n, H, H, 1, 1, P, res=P, one_pass=op)
            else:
                u['conv1'] = dgrad_op(unit['conv1'].bwd, D2, n, H, H, 1, 1, P, one_pass=op)
            ops.append(u)
            H = Ho
        self._bwd = dict(G=G, D1=D1, D2=D2, Z=Z, P=P, units=ops, ws_w=torch.empty(max(16, int(ws_w)), dtype=torch.uint8, device=p.device),
                         ws_b=torch.empty(max(16, ws_b), dtype=torch.uint8, device=p.device))
        return self._bwd

    def _bn_backward(self, i, dz, out, dgamma, dbeta, group=1, addend=None, add_geom=(0, 0, 0), stream=None):
        op, bn, ws = self.stats[i], self.bn, self._bwd['ws_b']
        check(lib.hd_bn_relu_backward(fptr(op.x), fptr(dz), int(group), op.rows, op.C, fptr(op.scale), fptr(op.shift), fptr(op.var),
                                      fptr(op.gamma), BN_EPS, fptr(addend) if addend is not None else None, add_geom[0], add_geom[1],
                                      add_geom[2], fptr(out), fptr(bn.view(dgamma, i)), fptr(bn.view(dbeta, i)),
                                      C.c_void_p(ws.data_ptr()), ws.numel(), stream), 'hd_bn_relu_backward')

    def _wgrad(self, x, geom, pre, dy, Cout, dw, db, stream, one_pass=False):
        """hd_conv_wgrad (one_pass: hd_conv_wgrad_ex in 1xTF32); geom = (n, H, W, Cin, Ho, Wo, KH, KW, stride, pad_t, pad_l); pre = a
        stats op (relu(bn(x))) or None."""
        n, H, W, Cin, Ho, Wo, KH, KW, s, pt, pl = geom
        ws = self._bwd['ws_w']
        args = (fptr(x), Cin, n, H, W, Cin, Ho, Wo, KH, KW, s, pt, pl, fptr(pre.scale) if pre is not None else None,
                fptr(pre.shift) if pre is not None else None, fptr(dy), Cout, Cout, fptr(dw), fptr(db) if db is not None else None,
                C.c_void_p(ws.data_ptr()), ws.numel())
        if one_pass:
            check(lib.hd_conv_wgrad_ex(*args, _lib.HD_IMPL_TC_1XTF32, stream), 'hd_conv_wgrad_ex')
        else:
            check(lib.hd_conv_wgrad(*args, stream), 'hd_conv_wgrad')

    def backward(self, dphi, images, stream=None):
        """Gradients of sum(phis * dphi) after the last `run` (keep=True), images (n,size,size,3) being that run's input: returns
        {TF variable name: gradient} for the 53 conv weights (HWIO) and 21 biases, plus 'gamma' / 'beta': the batch-norm gradients as
        flat vectors laid out like bn.gamma / bn.beta.  The images get no gradient.  Deterministic; `num_backward_launches` launches."""
        st = current_stream() if stream is None else stream
        S = self._backward_state()
        p, n, bn = self.p, self.n, self.bn
        dev = p.device
        f32 = dict(dtype=torch.float32, device=dev)
        L = bn.offsets[-1]
        dgamma, dbeta = torch.empty(L, **f32), torch.empty(L, **f32)
        grads = {'gamma': dgamma, 'beta': dbeta}
        G, D1, D2, Z, P = S['G'], S['D1'], S['D2'], S['Z'], S['P']
        U = len(p.units)
        # postnorm + ReLU + mean over H x W
        self._bn_backward(3 * U, dphi.contiguous(), G[0], dgamma, dbeta, group=self.final_hw, stream=st)
        scopes = self.unit_scopes()
        for ui in range(U - 1, -1, -1):
            unit, u, q = p.units[ui], S['units'][ui], scopes[ui]
            s, base, depth, d_in, H, Ho = unit['stride'], unit['base'], unit['depth'], unit['d_in'], u['H'], u['Ho']
            gy, gx = u['gy'], u['gx']
            st0, st1, st2 = self.stats[3 * ui], self.stats[3 * ui + 1], self.stats[3 * ui + 2]
            dW3, db3 = torch.empty((1, 1, base, depth), **f32), torch.empty(depth, **f32)
            self._wgrad(self.r2s[ui], (n, Ho, Ho, base, Ho, Ho, 1, 1, 1, 0, 0), st2, gy, depth, dW3, db3, st, self.one_pass)
            u['conv3'].run(st)                                                          # d relu(bn(conv2 out)) -> D1
            self._bn_backward(3 * ui + 2, D1, D2, dgamma, dbeta, stream=st)             # d conv2 out -> D2
            dW2 = torch.empty((3, 3, base, base), **f32)
            self._wgrad(self.r1s[ui], (n, H, H, base, Ho, Ho, 3, 3, s, 1, 1), st1, D2, base, dW2, None, st, self.one_pass)
            if s > 1:
                check(lib.hd_zero_insert(fptr(D2), fptr(Z), n, Ho, Ho, base, s, H, H, st), 'hd_zero_insert')
            u['conv2'].run(st)                                                          # d relu(bn(conv1 out)) -> D1
            self._bn_backward(3 * ui + 1, D1, D2, dgamma, dbeta, stream=st)             # d conv1 out -> D2
            dW1 = torch.empty((1, 1, d_in, base), **f32)
            self._wgrad(self.xs[ui], (n, H, H, d_in, H, H, 1, 1, 1, 0, 0), st0, D2, base, dW1, None, st, self.one_pass)
            addend, geom = None, (0, 0, 0)
            if 'shortcut' in unit:
                dWs, dbs = torch.empty((1, 1, d_in, depth), **f32), torch.empty(depth, **f32)
                self._wgrad(self.xs[ui], (n, H, H, d_in, H, H, 1, 1, 1, 0, 0), st0, gy, depth, dWs, dbs, st, self.one_pass)
                u['shortcut'].run(st)                                                   # d preact, shortcut path -> P
                grads[q + '/shortcut/weights'], grads[q + '/shortcut/biases'] = dWs, dbs
            else:
                addend, geom = gy, ((0, 0, 0) if s == 1 else (H, H, s))
            u['conv1'].run(st)                                                          # d preact (+ the shortcut's, in the epilogue) -> P
            self._bn_backward(3 * ui, P, gx, dgamma, dbeta, addend=addend, add_geom=geom, stream=st)
            grads[q + '/conv1/weights'], grads[q + '/conv2/weights'], grads[q + '/conv3/weights'] = dW1, dW2, dW3
            grads[q + '/conv3/biases'] = db3
        # pool1, then the root conv (7x7 stride 2, explicit pad 3) over the images
        check(lib.hd_maxpool3x3s2_same_backward(fptr(self.root_buf), fptr(G[U % 2]), fptr(P), n, self.H1, self.H1, 64, st),
              'hd_maxpool3x3s2_same_backward')
        dW, db = torch.empty((7, 7, 3, 64), **f32), torch.empty(64, **f32)
        self._wgrad(images, (n, self.size, self.size, 3, self.H1, self.H1, 7, 7, 2, 3, 3), None, P, 64, dW, db, st, self.one_pass)
        grads['resnet_v2_50/conv1/weights'], grads['resnet_v2_50/conv1/biases'] = dW, db
        return grads


# ------------------------------------------------------------------------------------------------
# f_movie temporal encoder -- src/models.py:121-228
# ------------------------------------------------------------------------------------------------
class PackedFMovie(object):
    def __init__(self, w, device, num_conv_layers=3, tc=False):
        self.device = device
        self.blocks = []
        for i in range(num_conv_layers):
            name = 'block_%d' % i
            blk = {}
            for k in (1, 2):
                blk['gn%d' % k] = (_dev(w['AZ_FC_block_preact_gn%d%s/gamma' % (k, name)], device),
                                   _dev(w['AZ_FC_block_preact_gn%d%s/beta' % (k, name)], device))
                blk['conv%d' % k] = PackedConv(w['AZ_FC_block2_conv%d%s/weights' % (k, name)], device,
                                               post_shift=w['AZ_FC_block2_conv%d%s/biases' % (k, name)], pad=(1, 0), tc=tc)
            self.blocks.append(blk)
        self.C = self.blocks[0]['conv1'].Cin if self.blocks else 2048
        sync_packing(device)


class FMoviePlan(object):
    """az_fc2_groupnorm over (B,T,C).  keep=True (training): each block writes its conv1 output and its output into buffers of its own
    instead of one `mid` and two ping-pong buffers, and `saved` = [(block input, conv1 output)] per block is what the backward reads;
    the launches and their arguments are the same, so the outputs are bit-identical to keep=False."""

    def __init__(self, packed: PackedFMovie, B, T, impl='auto', keep=False):
        self.p, self.B, self.T = packed, B, T
        dev, Cc = packed.device, packed.C
        self.gain = torch.empty((B, Cc), dtype=torch.float32, device=dev)
        self.offset = torch.empty((B, Cc), dtype=torch.float32, device=dev)
        nb = len(packed.blocks)
        bufs = [torch.empty((B, T, Cc), dtype=torch.float32, device=dev) for _ in range(2 * nb if keep else 3)]
        self.mids = bufs[:nb] if keep else [bufs[2]] * nb
        self.outs = bufs[nb:] if keep else [bufs[i % 2] for i in range(nb)]
        self.saved = []
        self.impl = impl
        self._bound_for = None

    def _bind_fast(self, x):
        """impl auto / tc3h / tc1h: GroupNorm + ReLU + split in one kernel (hd_groupnorm_relu_split), then the temporal conv reads its A
        operand as the pre-split pair (cp.async producer) instead of running GroupNorm in the register-staged producer."""
        dev, Cc = self.p.device, self.p.C
        B, T = self.B, self.T
        if not hasattr(self, 'act'):
            self.act = f16_pair((B * T, Cc), dev, self.impl)
        steps, cur, self.saved = [], x, []
        for blk, mid, out in zip(self.p.blocks, self.mids, self.outs):
            steps.append(('gns', cur, blk['gn1']))
            steps.append(('conv', blk['conv1'].bind(None, B, T, 1, mid, inp_split=self.act, impl=self.impl)))
            steps.append(('gns', mid, blk['gn2']))
            steps.append(('conv', blk['conv2'].bind(None, B, T, 1, out, inp_split=self.act, res=cur, res_geom=(Cc, T, 1, 1), impl=self.impl)))
            self.saved.append((cur, mid))
            cur = out
        self.steps, self.out = steps, cur
        self._bound_for = x.data_ptr()

    def _bind(self, x):
        if self.impl in F16_IMPLS and self.p.blocks and all(b[k].tc == 'f16' for b in self.p.blocks for k in ('conv1', 'conv2')) \
                and self.T * (self.p.C // GN_GROUPS) <= 1280:
            return self._bind_fast(x)
        steps, cur, self.saved = [], x, []
        pre = (self.gain, self.offset, self.p.C, 1)
        B, T = self.B, self.T
        for blk, mid, out in zip(self.p.blocks, self.mids, self.outs):
            steps.append(('gn', cur, blk['gn1']))
            steps.append(('conv', blk['conv1'].bind(cur, B, T, 1, mid, pre=pre, impl=self.impl)))
            steps.append(('gn', mid, blk['gn2']))
            steps.append(('conv', blk['conv2'].bind(mid, B, T, 1, out, pre=pre, res=cur,
                                                    res_geom=(self.p.C, T, 1, 1), impl=self.impl)))
            self.saved.append((cur, mid))
            cur = out
        self.steps, self.out = steps, cur
        self._bound_for = x.data_ptr()

    def run(self, x, stream=None):
        """x (B,T,C) contiguous float32 CUDA -> (B,T,C) (a plan-owned buffer; x itself if there are no blocks)."""
        st = current_stream() if stream is None else stream
        if self._bound_for != x.data_ptr():
            self._bind(x)
        for s in self.steps:
            if s[0] == 'gn':
                check(lib.hd_groupnorm_stats(fptr(s[1]), fptr(s[2][0]), fptr(s[2][1]), fptr(self.gain), fptr(self.offset),
                                             self.B, self.T, self.p.C, GN_GROUPS, GN_EPS, st), 'hd_groupnorm_stats')
            elif s[0] == 'gns':
                check(lib.hd_groupnorm_relu_split(fptr(s[1]), fptr(s[2][0]), fptr(s[2][1]), _vp(self.act[0]), _vp(self.act[1]),
                                                  self.B, self.T, self.p.C, GN_GROUPS, GN_EPS, st),
                      'hd_groupnorm_relu_split')
            else:
                s[1].run(st)
        return self.out

    @property
    def num_launches(self):
        return 4 * len(self.p.blocks)


# ------------------------------------------------------------------------------------------------
# IEF regressor -- src/models.py:80-116, 299-415
# ------------------------------------------------------------------------------------------------
class PackedIEFHead(object):
    def __init__(self, w, scope, device, feat=2048, tc=False):
        q = scope + '/3D_module'
        W1 = _dev(w[q + '/fc1/weights'], device)            # a device tensor (a trainable weight) is read in place, like PackedConv's
        self.d = W1.shape[0] - feat
        self.feat = feat
        # state = concat[phi, theta] (models.py:402): split fc1 so phi.W1[:feat] is computed once per window
        self.fc1_phi = PackedConv(W1[:feat], device, post_shift=w[q + '/fc1/biases'], tc=tc)
        self.fc1_theta = PackedConv(W1[feat:], device, post_relu=True)
        self.fc2 = PackedConv(w[q + '/fc2/weights'], device, post_shift=w[q + '/fc2/biases'], post_relu=True, tc=tc)
        self.fc3 = PackedConv(w[q + '/fc3/weights'], device, post_shift=w[q + '/fc3/biases'], tc=tc)   # ragged N: scalar epilogue path


class PackedIEF(object):
    def __init__(self, w, device, scope='single_view_ief', delta_t_values=(-5, 5), tc=False):
        self.device = device
        self.main = PackedIEFHead(w, scope, device, tc=tc)
        self.deltas = {}
        for dt in delta_t_values:
            dt = int(dt)
            if dt == 0:
                continue
            sc = scope + ('_future%d' % dt if dt > 0 else '_past%d' % abs(dt))
            self.deltas[dt] = PackedIEFHead(w, sc, device, tc=tc)
        self.mean_param = _dev(w['mean_param'], device).reshape(1, 85)
        sync_packing(device)


class IEFPlan(object):
    """call_hmr_ief for N rows: main 85-d head + 72-d delta heads started from the main prediction
    (use_delta_from_pred=True, use_optcam=True as wired by tester.py:196-207).

    keep=True (training, fast heads only): every head writes each stage's h1 in fp32 (hd_ief_fc1_theta's out_f32) and h2 into buffers of
    its own, and its stages other than the last into separate outputs instead of updating the state in place; each delta head writes an
    (N,85) output of its own instead of a slot of delta_all.  `saved` = per head, in the order main, delta_keys: (h1 [S,N,1024],
    h2 [S,N,1024], the outputs of stages 0 .. S-2) -- what the backward reads.  The launches are the same, so are the outputs' bits.

    dropout=(seed, step, call, keep_prob) (training, keep=True): slim.dropout(keep_prob) after the ReLU of fc1 and fc2 at every stage of
    every head, as the reference trains (src/models.py:101-105, is_training=True).  The masks are drawn in hd_ief_fc1_theta_dropout and
    hd_ief_fc3_dropout from (seed, step, site, row, column) alone (csrc/dropout.cuh), site = ief_dropout_site(call, head, stage, layer)
    with head 0 = main and 1.. = the packed delta heads in ascending dt; the saved h1 / h2 are the masked activations.  keep_prob 1 or
    dropout=None: today's launches."""

    def __init__(self, packed: PackedIEF, N, num_stage=3, delta_keys=None, impl='auto', keep=False, dropout=None):
        self.p, self.N, self.num_stage, self.keep = packed, N, num_stage, bool(keep)
        self.dropout = ief_dropout(dropout, len(packed.deltas) + 1, num_stage)
        if self.dropout is not None and not self.keep:
            raise _lib.HDError('IEFPlan: dropout is a training mode and needs keep=True')
        self.dropout_p = self.dropout[3] if self.dropout is not None else None
        self._head_index = {id(packed.main): 0}
        self._head_index.update({id(packed.deltas[k]): 1 + i for i, k in enumerate(sorted(packed.deltas))})
        dev = packed.device
        f32 = dict(dtype=torch.float32, device=dev)
        self.P = torch.empty((N, 1024), **f32)
        self.h1 = torch.empty((N, 1024), **f32)
        self.h2 = torch.empty((N, 1024), **f32)
        self.theta = torch.empty((N, 85), **f32)
        self.delta_keys = sorted(packed.deltas.keys()) if delta_keys is None else [k for k in delta_keys if k != 0]
        if self.keep:
            self.delta_out = {dt: torch.empty((N, 85), **f32) for dt in self.delta_keys}
        else:
            D = max(1, len(self.delta_keys))
            self.delta_all = torch.empty((N, D, 85), **f32)          # [N, D, 85]: the stacking of tester.py:252-253
            self.delta_out = {dt: self.delta_all[:, i, :] for i, dt in enumerate(self.delta_keys)}
        self.impl = impl
        self._bound_for = None
        self.saved = []
        heads = [packed.main] + [packed.deltas[k] for k in self.delta_keys]
        self.fast = impl in F16_IMPLS and all(h.fc1_phi.tc == 'f16' and h.fc2.tc == 'f16' for h in heads)
        if self.keep and not self.fast:
            raise _lib.HDError('IEFPlan: keep=True needs the fast heads (impl auto / tc3h / tc1h and fp16 packs)')
        if self.fast:
            self.phi_split = f16_pair((N, heads[0].feat), dev, impl)
            self.h1_split = f16_pair((N, 1024), dev, impl)

    def _head_ops_fast(self, head, start_view, state_view):
        """impl auto / tc3h / tc1h.  phi arrives once as a pre-split pair (hd_split_f16); per stage: hd_ief_fc1_theta (K = 85 / 72, writes h1
        pre-split) -> fc2 on the tensor cores (cp.async producer) -> hd_ief_fc3 (D = 85 / 72 + the IEF update).  The
        generic kernels ran fc1-theta on 40 SIMT blocks (50 us) and fc3 as ONE 128-row tile per 128 poses on 5 CTAs (80 us)."""
        N, S = self.N, self.num_stage
        ops = [('conv', head.fc1_phi.bind(None, N, 1, 1, self.P, inp_split=self.phi_split, impl=self.impl))]
        if self.keep:
            f32 = dict(dtype=torch.float32, device=self.p.device)
            h1, h2 = torch.empty((S, N, 1024), **f32), torch.empty((S, N, 1024), **f32)
            outs = [torch.empty((N, head.d), **f32) for _ in range(S - 1)] + [state_view]
            self.saved.append((h1, h2) + tuple(outs[:-1]))
        else:
            h1, h2, outs = [None] * S, [self.h2] * S, [state_view] * S
        prev = start_view
        sites = [(None, None)] * S
        if self.dropout is not None:
            hi = self._head_index[id(head)]
            sites = [tuple(ief_dropout_site(self.dropout[2], hi, s, layer) for layer in (0, 1)) for s in range(S)]
        for s in range(S):
            ops.append(('fc1t', prev, prev.stride(0), head, h1[s], sites[s][0]))
            ops.append(('conv', head.fc2.bind(None, N, 1, 1, h2[s], inp_split=self.h1_split, impl=self.impl)))
            ops.append(('fc3', prev, prev.stride(0), outs[s], outs[s].stride(0), head, h2[s], sites[s][1]))
            prev = outs[s]
        return ops

    def _run_ops(self, ops, st):
        N = self.N
        for op in ops:
            kind = op[0] if isinstance(op, tuple) else None
            if kind is None:
                op.run(st)
            elif kind == 'conv':
                op[1].run(st)
            elif kind == 'fc1t':
                _, prev, prev_ld, head, h1, site = op
                if site is None:
                    check(lib.hd_ief_fc1_theta(fptr(self.P), fptr(prev), prev_ld, fptr(head.fc1_theta.w_kn), head.d, 1024,
                                               _vp(self.h1_split[0]), _vp(self.h1_split[1]), _vp(h1), N, st),
                          'hd_ief_fc1_theta')
                else:
                    seed, step, _, p = self.dropout
                    check(lib.hd_ief_fc1_theta_dropout(fptr(self.P), fptr(prev), prev_ld, fptr(head.fc1_theta.w_kn), head.d, 1024,
                                                       _vp(self.h1_split[0]), _vp(self.h1_split[1]), _vp(h1), N, seed, step, site, p, st),
                          'hd_ief_fc1_theta_dropout')
            else:
                _, prev, prev_ld, out, out_ld, head, h2, site = op
                if site is None:
                    check(lib.hd_ief_fc3(fptr(h2), fptr(head.fc3.w_kn), fptr(head.fc3.post_shift), fptr(prev), prev_ld, fptr(out), out_ld,
                                         N, 1024, head.d, st), 'hd_ief_fc3')
                else:
                    seed, step, _, p = self.dropout
                    check(lib.hd_ief_fc3_dropout(fptr(h2), fptr(head.fc3.w_kn), fptr(head.fc3.post_shift), fptr(prev), prev_ld, fptr(out),
                                                 out_ld, N, 1024, head.d, seed, step, site, p, st), 'hd_ief_fc3_dropout')

    def _head_ops(self, head, phi, start_view, state_view):
        """ops for one hmr_ief: start_view = theta_prev of stage 0, state_view = in-place theta afterwards."""
        if self.fast:
            return self._head_ops_fast(head, start_view, state_view)
        return ief_head_ops(head, phi, start_view, state_view, self.P, self.h1, self.h2, self.num_stage, self.impl)

    def _bind(self, phi, theta0):
        self.saved = []
        self.main_ops = self._head_ops(self.p.main, phi, theta0, self.theta)
        self.delta_ops = {}
        for dt in self.delta_keys:
            view = self.delta_out[dt][:, 3:75]
            self.delta_ops[dt] = self._head_ops(self.p.deltas[dt], phi, view, view)
        self._bound_for = (phi.data_ptr(), theta0.data_ptr())

    def run_main(self, phi, theta0, stream=None):
        """Main 85-d head only: phi (N,2048), theta0 (N,85) contiguous -> theta (N,85)."""
        st = current_stream() if stream is None else stream
        if self._bound_for != (phi.data_ptr(), theta0.data_ptr()):
            self._bind(phi, theta0)
        if self.fast:
            check(lib.hd_split_f16(fptr(phi), _vp(self.phi_split[0]), _vp(self.phi_split[1]), phi.numel(), st), 'hd_split_f16')
        self._run_ops(self.main_ops, st)
        return self.theta

    def run_deltas(self, stream=None):
        """Delta heads, started from the main prediction (run_main must have run): {dt: (N,85) output, a view of delta_all[:, i] unless
        keep}."""
        st = current_stream() if stream is None else stream
        for dt in self.delta_keys:
            check(lib.hd_ief_delta_init(fptr(self.theta), fptr(self.delta_out[dt]), self.delta_out[dt].stride(0), self.N, st),
                  'hd_ief_delta_init')
            self._run_ops(self.delta_ops[dt], st)
        return self.delta_out

    def run(self, phi, theta0, stream=None):
        """phi (N,2048), theta0 (N,85) contiguous -> (theta (N,85), run_deltas())."""
        theta = self.run_main(phi, theta0, stream)
        return theta, self.run_deltas(stream)

    @property
    def num_launches(self):
        per = 1 + 3 * self.num_stage
        return per + len(self.delta_keys) * (per + 1) + (1 if self.fast else 0)


def ief_dropout_site(call, head, stage, layer):
    """The dropout site of one IEF call's layer: call 0 = the pred strips, 1 = the hal strips; head 0 = main, then the delta heads in
    ascending dt; stage 0..3; layer 0 = dropout1 (after fc1), 1 = dropout2 (after fc2)."""
    return ((call * 8 + head) * 4 + stage) * 2 + layer


def nn_keep_prob(keep_prob):
    """The float32 keep_prob TF 1.8's nn.dropout computes with for slim.dropout(keep_prob): core_layers.Dropout keeps rate = 1 -
    keep_prob and calls nn.dropout(1 - rate), a Python float64 that becomes a float32 tensor."""
    return float(np.float32(1.0 - (1.0 - float(keep_prob))))


def ief_dropout(spec, num_heads, num_stage):
    """IEFPlan's dropout argument -> (seed, step, call, nn.dropout's float32 keep_prob), or None for the identity (None, keep_prob 1)."""
    if spec is None:
        return None
    seed, step, call, p = spec
    p = float(p)
    if not 0.0 < p <= 1.0:
        raise _lib.HDError('IEF dropout: keep_prob must be in (0, 1], got %r' % (p,))
    seed, step, call = int(seed), int(step), int(call)
    if not (0 <= seed < 2 ** 64 and 0 <= step < 2 ** 64 and call >= 0):
        raise _lib.HDError('IEF dropout: need 0 <= seed, step < 2^64 and call >= 0, got %r' % (spec,))
    if num_heads > 8 or num_stage > 4 or ief_dropout_site(call + 1, 0, 0, 0) > 2 ** 31:
        raise _lib.HDError('IEF dropout: at most 8 heads and 4 stages per call')
    p32 = nn_keep_prob(p)
    if p32 <= 0.0:
        raise _lib.HDError('IEF dropout: keep_prob %r is 0 in float32' % (p,))
    return None if p32 == 1.0 else (seed, step, call, p32)


def ief_head_ops(head: PackedIEFHead, phi, start, state, P, h1, h2, num_stage, impl):
    """The generic kernels of one hmr_ief head, as ops: phi.W1[:feat] once into P, then per stage fc1-theta (SIMT, + P) into h1 -> fc2
    into h2 -> fc3 + the IEF update into `state`.  start: theta_prev of stage 0; later stages update `state` in place (row strides
    from the views)."""
    N = state.shape[0]
    ops = [head.fc1_phi.bind(phi, N, 1, 1, P, impl=impl)]
    for s in range(num_stage):
        prev = start if s == 0 else state
        ops.append(head.fc1_theta.bind(prev, N, 1, 1, h1, in_ld=prev.stride(0), res=P, res_geom=(1024, 1, 1, 1), impl='simt'))
        ops.append(head.fc2.bind(h1, N, 1, 1, h2, impl=impl))
        ops.append(head.fc3.bind(h2, N, 1, 1, state, out_ld=state.stride(0), res=prev, res_geom=(prev.stride(0), 1, 1, 1), impl=impl))
    return ops


def run_ief_head(head: PackedIEFHead, phi, start, num_stage=3, impl='auto', stream=None, out=None):
    """hmr_ief for one head from an arbitrary start: phi (N,feat), start (N,d) (unit inner stride) -> (N,d).

    The generic kernels (ief_head_ops), bound per call; the Tester path uses the cached IEFPlan instead.
    """
    st = current_stream() if stream is None else stream
    N, d = phi.shape[0], head.d
    if start.shape[0] != N or start.shape[1] != d or start.stride(1) != 1:
        raise _lib.HDError('hmr_ief: omega_start must be (N,%d) with unit inner stride' % d)
    f32 = dict(dtype=torch.float32, device=phi.device)
    P, h1, h2 = torch.empty((N, 1024), **f32), torch.empty((N, 1024), **f32), torch.empty((N, 1024), **f32)
    theta = torch.empty((N, d), **f32) if out is None else out
    for op in ief_head_ops(head, phi, start, theta, P, h1, h2, num_stage, impl):
        op.run(st)
    return theta


class PackedHal(object):
    """fc2_res hallucinator (models.py:270-296): x + fc3(relu(fc2(relu(fc1(x)))))."""

    def __init__(self, w, device, tc=False, name='fc2_res'):
        self.fc1 = PackedConv(w[name + '/fc1/weights'], device, post_shift=w[name + '/fc1/biases'], post_relu=True, tc=tc)
        self.fc2 = PackedConv(w[name + '/fc2/weights'], device, post_shift=w[name + '/fc2/biases'], post_relu=True, tc=tc)
        self.fc3 = PackedConv(w[name + '/fc3/weights'], device, post_shift=w[name + '/fc3/biases'], tc=tc)
        sync_packing(device)

    def run(self, x, h1, h2, out, impl='auto', stream=None):
        """x (N,2048) contiguous -> out (N,2048); h1 / h2 (N,2048) receive the two hidden activations."""
        st = current_stream() if stream is None else stream
        N = x.shape[0]
        self.fc1.bind(x, N, 1, 1, h1, impl=impl).run(st)
        self.fc2.bind(h1, N, 1, 1, h2, impl=impl).run(st)
        self.fc3.bind(h2, N, 1, 1, out, res=x, res_geom=(2048, 1, 1, 1), impl=impl).run(st)
        return out
