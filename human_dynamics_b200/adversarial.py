"""The adversarial pose prior D_pose of HMMR (reference src/discriminators.py) as a trainable torch module on the GPU.

D_pose scores the 23 non-root joint rotations of a pose: per joint a shared 1x1-conv MLP (9 -> 32 -> 32, ReLU) and a 32 -> 1 head, and
for the whole pose two 1024-wide FC layers over the flattened [23 * 32] trunk and a 1024 -> 1 output; logits (N, 24).  It is trained with
the LSGAN losses of src/ops.py (compute_loss_d_real / compute_loss_d_fake for D, compute_loss_e_fake back into theta for the
encoder), which are ordinary torch code:

    disc = PoseDiscriminator(seed=0)                      # or PoseDiscriminator(weights): anything engine.load_weights accepts
    opt_d = torch.optim.Adam(disc.parameters(), 1e-4)
    d_loss = compute_loss_d_real(disc(real_rots)) + compute_loss_d_fake(disc(fake_rots.detach()))
    d_loss.backward(); opt_d.step()                        # the fc packs are rewritten before the next forward
    disc.requires_grad_(False)                             # E step: the gradient reaches theta only
    e_loss = compute_loss_e_fake(disc(batch_rodrigues(theta)[:, 1:]))

The forward and backward run csrc/dpose.cu and hd_conv_gemm (the FC layers: 3xTF32 for fc1, whose K = 736 is not a multiple of 64, the
fp16-split pack for fc2 (impl 'auto'); the backward's GEMMs are 3xTF32, or 1xTF32 with grad_precision='tf32').  Results are deterministic: a pose's logits and input gradient
depend on that pose only, and the weight gradients are fixed-order sums.  No weight decay: the reference's l2_regularizer terms go into a
collection its trainer never reads.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import _lib
from ._lib import lib, check, fptr, current_stream
from .nets import BackwardDataPack, PackedConv, dgrad_op, grad_one_pass
from .trainable import TrainableModule, _col_sum, _round, _vp, _wgrad, _xt

F32 = torch.float32
J, CH, FLAT, HID = 23, 32, 736, 1024

# module parameters, in the order DPoseFunction takes them; the 23 heads pose_out_j<j> are held stacked ([23, 32] and [23])
PARAM_NAMES = ['D_pose/D_conv1/weights', 'D_pose/D_conv1/biases', 'D_pose/D_conv2/weights', 'D_pose/D_conv2/biases',
               'D_pose/pose_out_j/weights', 'D_pose/pose_out_j/biases',
               'D_pose/D_alljoints_fc1/weights', 'D_pose/D_alljoints_fc1/biases', 'D_pose/D_alljoints_fc2/weights',
               'D_pose/D_alljoints_fc2/biases', 'D_pose/D_alljoints_out/weights', 'D_pose/D_alljoints_out/biases']
# offsets of the small layers' gradients in hd_dpose_grad_reduce's packed output (include/hd_b200.h)
_PACKED = {0: (0, 288), 1: (288, 320), 2: (320, 1344), 3: (1344, 1376), 4: (1376, 2112), 5: (2112, 2135), 10: (2135, 3159), 11: (3159, 3160)}


def tf_names():
    """The TF variable names of D_pose, in the order the reference creates them."""
    from .synthetic import DPOSE_LAYERS
    return ['D_pose/%s/%s' % (n, k) for n, _ in DPOSE_LAYERS for k in ('weights', 'biases')]


def stack_heads(w):
    """{PARAM_NAMES name: float32 ndarray} from TF-named D_pose arrays (tf_names()): the 23 heads pose_out_j<j> stacked."""
    a = {n: np.asarray(w[n], np.float32) for n in tf_names()}
    a['D_pose/pose_out_j/weights'] = np.stack([a['D_pose/pose_out_j%d/weights' % j].reshape(CH) for j in range(J)])
    a['D_pose/pose_out_j/biases'] = np.concatenate([a['D_pose/pose_out_j%d/biases' % j].reshape(1) for j in range(J)])
    return a


def split_heads(a):
    """The reverse of stack_heads: {PARAM_NAMES name: array} -> {TF name: array in the reference's shape}."""
    from .synthetic import DPOSE_LAYERS
    out = {}
    for name, shape in DPOSE_LAYERS:
        if name.startswith('pose_out_j'):
            j = int(name[len('pose_out_j'):])
            out['D_pose/%s/weights' % name] = a['D_pose/pose_out_j/weights'][j].reshape(shape).copy()
            out['D_pose/%s/biases' % name] = a['D_pose/pose_out_j/biases'][j:j + 1].copy()
        else:
            out['D_pose/%s/weights' % name] = a['D_pose/%s/weights' % name].reshape(shape)
            out['D_pose/%s/biases' % name] = a['D_pose/%s/biases' % name]
    return out


def _load(weights):
    """engine.load_weights, except that a checkpoint's D_* variables are read (load_weights leaves them out, as Tester does)."""
    from . import tf_checkpoint
    from .engine import load_weights
    if isinstance(weights, str):
        prefix = weights[:-6] if weights.endswith('.index') else weights
        if tf_checkpoint.is_checkpoint(prefix):
            return tf_checkpoint.load_checkpoint(prefix, names=tf_names())
    return load_weights(weights)


def dpose_forward(d, x):
    """x (N, 23, 9) contiguous -> (logits (N, 24), saved (h1, h2, f1, f2) for the backward)."""
    N = x.shape[0]
    st = current_stream()
    dev = x.device
    P = d._p
    h1, h2 = torch.empty((N, FLAT), dtype=F32, device=dev), torch.empty((N, FLAT), dtype=F32, device=dev)
    f1, f2 = torch.empty((N, HID), dtype=F32, device=dev), torch.empty((N, HID), dtype=F32, device=dev)
    logits = torch.empty((N, J + 1), dtype=F32, device=dev)
    check(lib.hd_dpose_trunk_forward(fptr(x), *[fptr(P[i]) for i in range(6)], fptr(h1), fptr(h2), fptr(logits), N, st),
          'hd_dpose_trunk_forward')
    d.fc1.bind(h2, N, 1, 1, f1, impl='auto').run(st)
    d.fc2.bind(f1, N, 1, 1, f2, impl='auto').run(st)
    check(lib.hd_dpose_out_forward(fptr(f2), fptr(P[10]), fptr(P[11]), fptr(logits), N, st), 'hd_dpose_out_forward')
    return logits, (h1, h2, f1, f2)


def dpose_backward(d, x, saved, g, want_dx, want_dw):
    """Gradients for an upstream g (N, 24) contiguous: (dx (N, 23, 9) or None, [one per PARAM_NAMES] or None)."""
    h1, h2, f1, f2 = saved
    N = g.shape[0]
    st = current_stream()
    dev = g.device
    P = d._p
    df2, df1 = torch.empty((N, HID), dtype=F32, device=dev), torch.empty((N, HID), dtype=F32, device=dev)
    dflat = torch.empty((N, FLAT), dtype=F32, device=dev)
    # df2 = g[:, 23] w_out^T * (f2 > 0);  df1 = (df2 . Wfc2^T) * (f1 > 0);  dflat = df1 . Wfc1^T
    check(lib.hd_fc_small_dgrad(_vp(g, J * 4), J + 1, fptr(P[10]), HID, 1, fptr(f2), fptr(df2), N, st), 'hd_fc_small_dgrad')
    dgrad_op(d.fc2_bwd, df2, N, 1, 1, 1, 1, df1, one_pass=d.one_pass).run(st)
    check(lib.hd_relu_backward(fptr(f1), fptr(df1), fptr(df1), N * HID, st), 'hd_relu_backward')
    dgrad_op(d.fc1_bwd, df1, N, 1, 1, 1, 1, dflat, one_pass=d.one_pass).run(st)
    dx = torch.empty((N, J, 9), dtype=F32, device=dev) if want_dx else None
    ws_bytes = int(lib.hd_dpose_workspace_bytes(N)) if want_dw else 0
    ws = torch.empty(ws_bytes // 4, dtype=F32, device=dev) if want_dw else None
    check(lib.hd_dpose_trunk_backward(fptr(x) if want_dw else None, fptr(h1), fptr(h2), fptr(dflat), fptr(g), fptr(f2),
                                      fptr(P[0]), fptr(P[2]), fptr(P[4]), fptr(dx), fptr(ws), ws_bytes, N, st), 'hd_dpose_trunk_backward')
    if not want_dw:
        return dx, None
    packed = torch.empty(3160, dtype=F32, device=dev)
    check(lib.hd_dpose_grad_reduce(fptr(ws), ws_bytes, N, fptr(packed), st), 'hd_dpose_grad_reduce')
    grads = [None] * len(PARAM_NAMES)
    for i, (a, b) in _PACKED.items():
        grads[i] = packed[a:b].view(P[i].shape)
    kp = _round(N, 32)
    for i, inp, gin, cin in ((6, h2, df1, FLAT), (8, f1, df2, HID)):
        W, bias = torch.empty((cin, HID), dtype=F32, device=dev), torch.empty(HID, dtype=F32, device=dev)
        _wgrad(_xt([(inp, N, cin)], cin, kp, st), cin, kp, [(gin, N, HID)], HID, W, st, d.one_pass)
        _col_sum(gin, N, HID, HID, bias, st)
        grads[i], grads[i + 1] = W, bias
    return dx, grads


class DPoseFunction(torch.autograd.Function):
    """rotmats (N, 23, 9) -> logits (N, 24); differentiable w.r.t. the rotations and every D_pose parameter.  The backward computes the
    input gradient only when the rotations need it, and the weight gradients only when a parameter needs one."""

    @staticmethod
    def forward(ctx, disc, x, *params):
        logits, saved = dpose_forward(disc, x)
        ctx.disc = disc
        ctx.save_for_backward(x, *saved)
        return logits

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        disc = ctx.disc
        need = ctx.needs_input_grad
        want_dw = any(need[2:])
        if want_dw or need[1]:
            disc.sync_bwd_packs()
        x, *saved = ctx.saved_tensors
        dx, grads = dpose_backward(disc, x, saved, g.contiguous(), need[1], want_dw)
        grads = grads or [None] * len(PARAM_NAMES)
        return (None, dx) + tuple(gr if n else None for gr, n in zip(grads, need[2:]))


class PoseDiscriminator(TrainableModule):
    """D_pose as fp32 parameters on one CUDA device.  `weights`: anything engine.load_weights accepts that holds the D_pose/* variables
    (other variables are ignored); without it, slim's default initialisation from `seed` (synthetic.make_dpose_weights).

    Parameters are addressable by PARAM_NAMES (`disc.param('D_pose/D_conv1/weights')`); the 23 heads pose_out_j<j> are stacked into
    'D_pose/pose_out_j/weights' [23, 32] and '.../biases' [23].  A parameter changed in place (optimizer.step()) is repacked before the
    next forward / backward.  Under torch.no_grad(), or when nothing requires grad, the forward builds no graph.  grad_precision: 'fp32'
    (3xTF32 backward GEMMs) or 'tf32' (1xTF32, nets.GRAD_PRECISIONS); the forward is the same in both."""

    def __init__(self, weights=None, seed=0, device=None, grad_precision='fp32'):
        super().__init__()
        from .synthetic import make_dpose_weights
        self.one_pass = grad_one_pass(grad_precision, 'PoseDiscriminator')
        if not torch.cuda.is_available():
            raise _lib.HDError('PoseDiscriminator needs a CUDA device: the hot path has no CPU fallback')
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        w = make_dpose_weights(seed) if weights is None else _load(weights)
        missing = [n for n in tf_names() if n not in w]
        if missing:
            raise _lib.HDError('PoseDiscriminator: the weights lack %d D_pose variables (first: %s)' % (len(missing), missing[0]))
        a = stack_heads(w)
        for n in PARAM_NAMES:
            self._params[n] = nn.Parameter(torch.from_numpy(np.ascontiguousarray(a[n])).to(self.device))
        self._p = [self._params[n] for n in PARAM_NAMES]
        with torch.cuda.device(self.device):
            P = [p.data for p in self._p]
            self.fc1 = PackedConv(P[6], self.device, post_shift=P[7], post_relu=True, tc='auto')     # Cin 736: TF32 pack, 3xTF32
            self.fc2 = PackedConv(P[8], self.device, post_shift=P[9], post_relu=True, tc='auto')     # Cin 1024: fp16-split pack
            self.fc1_bwd = BackwardDataPack(P[6], 1, FLAT, HID)
            self.fc2_bwd = BackwardDataPack(P[8], 1, HID, HID)
        self._fwd_packs += [(PARAM_NAMES[6], self.fc1), (PARAM_NAMES[8], self.fc2)]
        self._bwd_packs += [(PARAM_NAMES[6], self.fc1_bwd), (PARAM_NAMES[8], self.fc2_bwd)]
        self._packs_written(self.device)

    def _input(self, rotmats):
        x = rotmats
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise _lib.HDError('PoseDiscriminator: a CUDA tensor is required (no CPU fallback exists)')
        if x.dtype != F32 or x.dim() not in (3, 4) or tuple(x.shape[1:]) not in ((J, 9), (J, 1, 9)) or x.shape[0] < 1:
            raise _lib.HDError('PoseDiscriminator: expected float32 (N, 23, 9) or (N, 23, 1, 9) with N >= 1, got %s %s'
                               % (x.dtype, tuple(x.shape)))
        if x.device != self.device:
            raise _lib.HDError('PoseDiscriminator: tensor is on %s, the model on %s' % (x.device, self.device))
        return x.reshape(x.shape[0], J, 9).contiguous()

    def forward(self, rotmats):
        """rotmats (N, 23, 9) or (N, 23, 1, 9) -> logits (N, 24): the 23 per-joint scores, then the whole-pose score."""
        x = self._input(rotmats)
        self.sync_packs()
        if self._grad_on(PARAM_NAMES, x):
            return DPoseFunction.apply(self, x, *self._p)
        with torch.no_grad():
            return dpose_forward(self, x.detach())[0]

    def relu_masks(self, rotmats):
        """The ReLU masks (pre-activation > 0) of the GPU forward as CPU bool tensors: 'conv1' / 'conv2' [N, 23, 32], 'fc1' / 'fc2'
        [N, 1024].  An inspection aid for comparing against a float64 reference at near-tie sites."""
        x = self._input(rotmats)
        with torch.no_grad():
            self.sync_packs()
            _, (h1, h2, f1, f2) = dpose_forward(self, x)
        N = x.shape[0]
        return {'conv1': (h1 > 0).reshape(N, J, CH).cpu(), 'conv2': (h2 > 0).reshape(N, J, CH).cpu(), 'fc1': (f1 > 0).cpu(),
                'fc2': (f2 > 0).cpu()}

    def tf_variables(self):
        """The D_pose/* variables under the reference's names and shapes: {name: float32 ndarray}."""
        return split_heads({n: self.param(n).detach().cpu().numpy() for n in PARAM_NAMES})
