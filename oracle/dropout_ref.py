"""ORACLE (test infrastructure, not product): the IEF dropout masks in numpy, bit for bit with csrc/dropout.cuh.

Element (n, j) of site `site` at step `step`, width C, w = n*C + j:
    word = Philox4x32-10(counter = (w >> 2, site, step & 0xffffffff, step >> 32), key = (seed & 0xffffffff, seed >> 32))[w & 3]
    u    = float32((word & 0x7fffff) | 0x3f800000) - 1                        (TF's Uint32ToFloat)
    keep = floor(float32(p + u)) == 1                                          (TF 1.8 nn.dropout, float32)
    y    = float32(float32(x / p) * keep)
p is nn.dropout's float32 keep_prob: slim.dropout(keep_prob) reaches it as 1 - (1 - keep_prob) worked out in Python float64, then
rounded to float32 (`nn_keep_prob`).  site = ((call*8 + head)*4 + stage)*2 + layer (`site`).  All arithmetic is uint64 numpy.
"""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 arrays (broadcastable), key: 2 uint32 values -> 4 uint64 arrays holding the uint32 output words."""
    c = [np.asarray(x, np.uint64) & MASK32 for x in ctr]
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK32, (k1 + W1) & MASK32
        p0, p1 = M0 * c[0], M1 * c[2]                       # < 2^64: exact in uint64
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK32
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return c


def site(call, head, stage, layer):
    """call 0 = the pred strips, 1 = the hal strips; head 0 = main, then the delta heads in ascending dt; stage 0..2; layer 0 = dropout1
    (after fc1), 1 = dropout2 (after fc2)."""
    assert 0 <= call and 0 <= head < 8 and 0 <= stage < 4 and layer in (0, 1)
    return ((call * 8 + head) * 4 + stage) * 2 + layer


def nn_keep_prob(keep_prob):
    """The float32 keep_prob nn.dropout computes with for slim.dropout(keep_prob) (TF 1.8 core_layers.Dropout: rate = 1 - keep_prob,
    then nn.dropout(1 - rate), a Python float64 made a float32 tensor)."""
    return np.float32(1.0 - (1.0 - float(keep_prob)))


def words(seed, step, site_, N, C):
    """The uint32 word of every element, [N, C] uint64."""
    w = np.arange(N * C, dtype=np.uint64)
    g = w >> np.uint64(2)
    step, seed = int(step), int(seed)
    out = philox4x32_10((g, np.uint64(site_), np.uint64(step & 0xFFFFFFFF), np.uint64(step >> 32)), (seed & 0xFFFFFFFF, seed >> 32))
    e = (w & np.uint64(3)).astype(np.int64)
    return np.choose(e, out).reshape(N, C)


def uniform(word):
    """TF's Uint32ToFloat: float32 in [0, 1) from the low 23 bits."""
    bits = ((np.asarray(word, np.uint64) & np.uint64(0x7FFFFF)) | np.uint64(0x3F800000)).astype(np.uint32)
    return bits.view(np.float32) - np.float32(1.0)


def keep_from_uniform(u, p):
    """nn.dropout's binary tensor: floor(keep_prob + u) in float32."""
    p = np.float32(p)
    return np.floor(np.asarray(u, np.float32) + p).astype(np.float32)


def mask(seed, step, site_, N, C, p):
    """[N, C] uint8: 1 where element (n, j) is kept (p = nn.dropout's float32 keep_prob)."""
    return keep_from_uniform(uniform(words(seed, step, site_, N, C)), p).astype(np.uint8)


def apply(x, keep, p):
    """nn.dropout's output in float32: (x / p) * binary."""
    p = np.float32(p)
    return (np.asarray(x, np.float32) / p) * np.asarray(keep, np.float32)


def ief_masks(seed, step, call, N, num_heads, p, num_stage=3, C=1024):
    """{(head, stage, layer): [N, C] uint8} for one IEF call over N rows."""
    return {(h, s, l): mask(seed, step, site(call, h, s, l), N, C, p) for h in range(num_heads) for s in range(num_stage) for l in (0, 1)}
