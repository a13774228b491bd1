"""The TF32 rounding of the 1xTF32 gradient mode (grad_precision='tf32'), emulated on the host: hd::ptx::rn_tf32 keeps the nearest value
with the low 13 mantissa bits clear, ties rounding away from zero in magnitude, by (bits + 0x1000) & 0xFFFFE000 on the fp32 pattern."""
import numpy as np


def rn_tf32(a):
    """float32 array -> float32 array of TF32 heads, rounded as the kernels round them."""
    b = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
