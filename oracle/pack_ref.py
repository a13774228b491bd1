"""numpy restatement of the tensor-core weight packing (hd_pack_weight, forward mode): what the device packs are compared against.

A conv / FC weight in TF HWIO is laid out K-major as w_nk [roundup64(Cout), K_pad] (K index (ky, kx, ci); zero rows and columns past
the matrix), then split into a head and a remainder: fp16 head + 2^11-scaled fp16 remainder, or a TF32 pair in fp32 storage.
"""
import numpy as np


def tf32_split(w):
    """w (float32) -> (hi, lo), both exactly representable in TF32 (low 13 mantissa bits zero, which is all the
    tensor core reads): hi = w rounded to nearest TF32, lo = (w - hi) rounded to nearest TF32.  Rounding (not
    truncating) keeps the representation error zero-mean, so it does not build up over the 53 layers."""
    def rn_tf32(x):
        b = np.ascontiguousarray(x, np.float32).view(np.uint32)
        return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
    w = np.ascontiguousarray(w, np.float32)
    hi = rn_tf32(w)
    lo = rn_tf32((w - hi).astype(np.float32))
    return hi, lo


def f16_split(w):
    """w (float32) -> (hi, lo) float16: hi = RN_f16(w), lo = RN_f16((w - hi) * 2^11).  Same 11+11 significant bits as the
    TF32 split at twice the tensor-core rate; the 2^11 scale keeps the remainder of small weights out of the fp16
    subnormal range (the kernel accumulates the scaled cross terms separately and rescales once)."""
    w = np.ascontiguousarray(w, np.float32)
    hi = w.astype(np.float16)
    lo = ((w - hi.astype(np.float32)) * np.float32(2048.0)).astype(np.float16)
    return hi, lo


def nk_layout(w_hwio, gather=False):
    """TF HWIO (FC: [in, out]) -> w_nk [roundup64(Cout), K_pad] float32.  gather: the row-segment layout of a ragged conv1 (each
    kernel row's KW*Cin weights padded to a multiple of 8, K_pad = roundup64(KH * segp)); else K_pad = K = KH*KW*Cin."""
    w = np.asarray(w_hwio, np.float32)
    if w.ndim == 2:
        w = w[None, None]
    KH, KW, Cin, Cout = w.shape
    seg = KW * Cin
    segp = (seg + 7) // 8 * 8
    K_pad = (KH * segp + 63) // 64 * 64 if gather else KH * seg
    w_nk = np.zeros(((Cout + 63) // 64 * 64, K_pad), np.float32)
    if gather:
        wg = w.reshape(KH, seg, Cout)
        for ky in range(KH):
            w_nk[:Cout, ky * segp:ky * segp + seg] = wg[ky].T
    else:
        w_nk[:Cout, :KH * seg] = w.reshape(KH * seg, Cout).T
    return w_nk


def conv1_planes_layout(w_hwio):
    """ResNet conv1 7x7x3x64 -> [64, 256]: K index ky*32 + kx*4 + c over 8 x 8 x 4 taps, zero on the phantom row / pixel / channel."""
    w_nk = np.zeros((64, 8, 8, 4), np.float32)
    w_nk[:, :7, :7, :3] = np.asarray(w_hwio, np.float32).transpose(3, 0, 1, 2)
    return w_nk.reshape(64, 256)


def split(w_nk, kind):
    """kind 'f16' | 'tf32' -> (hi, lo) of w_nk."""
    return f16_split(w_nk) if kind == 'f16' else tf32_split(w_nk)
