"""Static configuration of the inference path (the subset of src/config.py flags the path reads)."""
from __future__ import annotations

import os

from dataclasses import dataclass, field
from typing import Any, Sequence


@dataclass
class HMMRConfig(object):
    """Duck-type compatible with the absl config object `Tester` reads (tester.py:28-57, omega.py:33).

    Defaults are the reference's: T=20 (config.py:44), num_kps=25 (:45), num_conv_layers=3 (:46),
    delta_t_values=[-5,5] (:47), img_size=224 (:66), num_stage=3 (:69).
    `load_path` may be a .npz of TF-named variables; `weights` / `smpl_model` may hold in-memory dicts.
    """
    batch_size: int = 8
    sequence_length: int = 20
    num_conv_layers: int = 3
    delta_t_values: Sequence[int] = (-5, 5)
    num_kps: int = 25
    num_stage: int = 3
    img_size: int = 224
    pred_mode: str = 'pred'
    load_path: str = ''
    smpl_model_path: str = ''
    weights: Any = None
    smpl_model: Any = None
    # 'auto' (= 'tc3h' where Cin % 64 == 0, else 'tc3', else 'simt') | 'tc3h' | 'tc3' | 'tc1' | 'simt': FP32-class except 'tc1' (1xTF32).
    # 'tc1h': half-precision inference (HD_IMPL_TC_1XF16): the networks' GEMMs on fp16 heads alone, one MMA per product, no remainder
    # buffers; about 1e-3 relative on the phis (DESIGN.md section 2).  SMPL stays FP32-class.  The training entries refuse it.
    impl: str = os.environ.get('HD_IMPL', 'auto')
    frame_chunk: int = 160        # frames per pass of ResNet root + blocks 1-2 (activation working set vs. L2)
    late_chunk: int = 640         # frames per pass of ResNet blocks 3-4 (small maps: batch wide to fill 132 SMs)
    extra: dict = field(default_factory=dict)
