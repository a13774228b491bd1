"""The reference trainer's objective (src/trainer_sequence_fc.py) on the GPU, and HMMRTrainer, one reference training iteration.

`build_objective(config, B, T, K)` lists the loss terms that compute_losses_batched, compute_losses_deltas (the delta sets and the
hallucinated sets) and the e_shape part of compute_losses_prior add for a config, as term descriptors of csrc/losses.cu over a fixed
set of inputs (`Objective.INPUTS`).  `LossFunction` evaluates them: two launches forward, one backward, whatever the number of terms.
The named losses are the reference's keys (e_kp, e_joints, e_smpl, e_const, e_kp_dt_future, ..., e_hallucinate, e_*_hal*), each the
sum of its terms, with the weights of trainer_sequence_fc.py:280-310.

    trainer = HMMRTrainer(TrainConfig(do_hallucinate=True, do_hallucinate_preds=True), weights, smpl_model)
    for batch, mocap in loader:                       # batch: the reference loader's dict; mocap: (trainer.n_fake(B, T), 216)
        out = trainer.step(batch, mocap)              # device scalars, no synchronise
    trainer.save_checkpoint('/path/model.ckpt-1000')  # Tester and PoseDiscriminator load it

    trainer = HMMRTrainer(cfg, weights, smpl_model, optimizer=TFAdam)         # TF's Adam: the checkpoint holds the optimizer state
    trainer = HMMRTrainer.resume(cfg, '/path/model.ckpt-1000', smpl_model)    # ... which resume restores (tf.train.Supervisor's restore)

With precomputed_phi=False (the reference's online-augmentation path) a batch carries `images` (B, T, S, S, 3) float32 in [-1, 1], e.g.
augment.TubeAugmentor(...)['images'], instead of `phis`: the frozen ResNet runs over all B*T crops in training mode (batch statistics,
nets.ResNetTrainPlan) without autograd, and each `step` applies the trunk's update ops once (one moving-average step of its 49
batch-norm layers, decay 0.997), which save_checkpoint writes.  With freeze_phi=False as well, the trunk trains: its conv weights, biases
and batch-norm gamma / beta (trunk.TrainableResNet) join E's optimizer, e_loss's gradient reaches them through the phis, and
save_checkpoint writes their trained values.  Like the reference (whose gather_losses never adds slim's regularisation losses), the
trunk trains without weight decay.

IEF dropout: the reference trains every IEF call with is_training=True, so slim.dropout(keep_prob=0.5) follows the ReLU of fc1 and
fc2 at each stage of every head, in both IEF calls of a step.  `TrainConfig(ief_keep_prob=0.5)` does the same on the GPU: the masks
are a documented function of (seed, global_step at the start of the step, call, head, stage, layer, row, column) (csrc/dropout.cuh,
restated by oracle/dropout_ref.py), so a run is reproducible from `seed` and a resumed run continues the mask stream where it
stopped.  The default, ief_keep_prob=1.0, keeps the inference graph (dropout the identity).

Differences from the reference trainer: with dropout, TF's own random stream, whose op seeds come from graph construction, is not
reproduced -- the placement and arithmetic of the masks are the reference's, the bits drawn are not; the default optimizer, torch's Adam, adds eps to sqrt(v_hat) where TF's adds it to sqrt(v) before the bias correction, and
`optimizer=optim.TFAdam` removes that difference (TF's arithmetic, with its slots, beta powers and global_step in the checkpoint, so
that `HMMRTrainer.resume(config, prefix, smpl_model)` continues a run where it stopped); the static `use_hmr_only` branch is not built, and freeze_phi=False needs image input (precomputed phis have no trunk to train).  A frame with no visible keypoint in an optimal-camera term
contributes 0 (the reference's procrustes2d_vis divides 0 / 0 there and the loss is NaN).  The moving statistics start from whatever
`weights` holds, so a resumed run continues them; a fresh reference run restores only the trainable variables from its hmr_noS5
checkpoint (trainer_sequence_fc.py:346-392), so its moving statistics start at 0 / 1 -- pass those values in `weights` to reproduce it.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _lib
from ._lib import lib, check, current_stream
from .config import HMMRConfig
from .nets import grad_one_pass, require_training_impl

F32 = torch.float32


@dataclass
class TrainConfig(HMMRConfig):
    """HMMRConfig plus the training flags of the reference's src/config.py, with its defaults."""
    e_lw_kp: float = 60.
    e_lw_joints: float = 60.
    e_lw_smpl: float = 60.
    e_lw_const: float = 1.
    e_lw_pose: float = 1.
    e_lw_shape: float = 1.
    e_lw_hallucinate: float = 1.
    d_lw_pose: float = 1.
    e_lr: float = 1e-5
    d_lr: float = 1e-4
    use_3d_label: bool = True
    mosh_ignore: bool = False
    predict_delta: bool = True
    do_hallucinate: bool = False
    do_hallucinate_preds: bool = False
    precomputed_phi: bool = True
    freeze_phi: bool = True
    # Precision of every backward GEMM (the trunk's, the temporal model's and D_pose's weight and data gradients): 'fp32' (3xTF32,
    # FP32-class) or 'tf32' (one TF32 MMA per product on round-to-nearest heads).  The forward passes, losses and optimizers are the
    # same in both (DESIGN.md section 2).
    grad_precision: str = 'fp32'
    # keep_prob of the IEF heads' dropout (slim.dropout after the ReLU of fc1 and fc2, src/models.py:101-105): 1.0 = the identity,
    # the reference trains with 0.5.  `seed` (src/config.py:132) keys its masks.
    ief_keep_prob: float = 1.0
    seed: int = 1

    def __post_init__(self):
        grad_one_pass(self.grad_precision, 'TrainConfig')
        if not 0.0 < float(self.ief_keep_prob) <= 1.0:
            raise _lib.HDError('TrainConfig: ief_keep_prob must be in (0, 1], got %r' % (self.ief_keep_prob,))
        if int(self.seed) != self.seed or not 0 <= int(self.seed) < 2 ** 64:
            raise _lib.HDError('TrainConfig: seed must be an integer in [0, 2^64), got %r' % (self.seed,))


def loss_weights(config):
    """trainer_sequence_fc.py:280-310 (the static-branch keys left out)."""
    c = config
    w = {'d_pose': c.d_lw_pose, 'e_const': c.e_lw_const, 'e_joints': c.e_lw_joints, 'e_kp': c.e_lw_kp, 'e_pose': c.e_lw_pose,
         'e_shape': c.e_lw_shape, 'e_smpl': c.e_lw_smpl, 'e_hallucinate': c.e_lw_hallucinate}
    for suf in ('_dt_future', '_dt_past', '_hal', '_hal_future', '_hal_past'):
        w.update({'e_joints' + suf: c.e_lw_joints, 'e_kp' + suf: c.e_lw_kp, 'e_smpl' + suf: c.e_lw_smpl})
    return {k: float(v) for k, v in w.items()}


def loss_keys(config):
    """The keys of the reference's self.losses for a config (trainer_sequence_fc.py:235-274), in its order."""
    keys = ['d_pose', 'e_const', 'e_joints', 'e_kp', 'e_pose', 'e_shape', 'e_smpl']
    if config.predict_delta:
        keys += ['e_joints_dt_future', 'e_kp_dt_future', 'e_smpl_dt_future', 'e_joints_dt_past', 'e_kp_dt_past', 'e_smpl_dt_past']
    if config.do_hallucinate:
        keys += ['e_hallucinate', 'e_joints_hal', 'e_kp_hal', 'e_smpl_hal']
        if config.do_hallucinate_preds:
            keys += ['e_joints_hal_future', 'e_kp_hal_future', 'e_smpl_hal_future', 'e_joints_hal_past', 'e_kp_hal_past',
                     'e_smpl_hal_past']
    return keys


def delta_values(config):
    dts = [int(d) for d in config.delta_t_values]
    if 0 in dts:
        raise _lib.HDError('delta_t_values must not contain 0')
    return dts


def prediction_sets(config):
    """The prediction sets in the order the reference appends them to pred_poses_all: the hallucinated sets (do_hallucinate: the present,
    then each delta_t with do_hallucinate_preds), the present prediction, then the delta heads (predict_delta).  [(group, dt)]."""
    dts = delta_values(config)
    sets = []
    if config.do_hallucinate:
        sets.append(('hal', 0))
        if config.do_hallucinate_preds:
            sets += [('hal', d) for d in dts]
    sets.append(('pred', 0))
    if config.predict_delta:
        sets += [('dt', d) for d in dts]
    return sets


def n_fake(config, B, T):
    """Mocap poses D needs per step: the loader's count (data_loader_sequence.py:185-196), B*T*(1+|dt|) with the present part doubled
    under do_hallucinate and the delta part doubled under do_hallucinate_preds."""
    m = B * T
    d = B * T * len(delta_values(config)) if config.predict_delta else 0
    if config.do_hallucinate:
        m *= 2
        if config.do_hallucinate_preds:
            d *= 2
    return m + d


_SUFFIX = {('pred', 0): '', ('hal', 0): '_hal'}


def _name(group, dt, base):
    if dt == 0:
        return base + _SUFFIX[(group, 0)]
    return base + ('_%s_%s' % ('dt' if group == 'dt' else 'hal', 'future' if dt > 0 else 'past'))


class Objective(object):
    """The term list of one config and shape.  Inputs (INPUTS order; S = len(sets), N = B*T):
      omega [S, B, T, 85]  joints [S, B, T, K, 3]  rots [S, B, T, 216]         the predictions, sets concatenated in `sets` order
      labels [B, T, K, 3]  gt_rots [B, T, 216]  gt_shape [B, 10]  gt3ds [B, T, 14, 3]  w_joints [B]  w_smpl [B]
      strips, pred_strips [B, T, 2048]                                           (do_hallucinate only)"""
    INPUTS = ('omega', 'joints', 'rots', 'labels', 'gt_rots', 'gt_shape', 'gt3ds', 'w_joints', 'w_smpl', 'strips', 'pred_strips')
    # the inputs LossFunction differentiates; the labels and weights take no gradient (apply_loss refuses them with requires_grad)
    DIFFERENTIABLE = ('omega', 'joints', 'rots', 'strips', 'pred_strips')

    def __init__(self, config, B, T, K):
        self.config, self.B, self.T, self.K = config, int(B), int(T), int(K)
        if self.B < 1 or self.T < 1 or self.K < 14:
            raise _lib.HDError('build_objective: need B >= 1, T >= 1 and K >= 14, got %d, %d, %d' % (B, T, K))
        self.sets = prediction_sets(config)
        self.inputs = self.INPUTS if config.do_hallucinate else self.INPUTS[:9]
        self.terms, self.term_names, self.cam_terms = [], [], []
        S = len(self.sets)
        row = {'omega': 85, 'joints': K * 3, 'rots': 216, 'labels': K * 3, 'gt_rots': 216, 'gt3ds': 42, 'strips': 2048, 'pred_strips': 2048}
        for s, (group, dt) in enumerate(self.sets):
            if abs(dt) >= T:
                continue                   # an empty window: the reference's term is 0 (tf.losses with no weight)
            Tw = T - abs(dt)
            p_t0, q_t0 = (abs(dt), 0) if dt < 0 else (0, dt)

            def side(slot, off=0, t0=0, frame=None, clip=None, base_set=s):
                r = row[slot]
                fr = r if frame is None else frame
                set_off = base_set * B * T * r if slot in ('omega', 'joints', 'rots') else 0
                return (slot, set_off + off, T * fr if clip is None else clip, fr, t0)

            kp = dict(kind=_lib.HD_LOSS_KP_L1, B=B, Tw=Tw, K=K, D=3, scale=1., p=side('joints', t0=p_t0), q=side('labels', t0=q_t0))
            if dt == 0:
                kp.update(proj=_lib.HD_LOSS_KP_CAMERA, cam=side('omega', 0, p_t0))
            else:
                kp.update(proj=_lib.HD_LOSS_KP_OPTCAM)
                self.cam_terms.append((len(self.terms), (group, dt)))
            self._add(_name(group, dt, 'e_kp'), kp)
            if config.use_3d_label:
                mse = dict(kind=_lib.HD_LOSS_MSE_ROWS, B=B, Tw=Tw, K=0, scale=0.5)
                self._add(_name(group, dt, 'e_joints'), dict(mse, proj=1, D=42, p=side('joints', t0=p_t0), q=side('gt3ds', t0=q_t0),
                                                             w='w_joints'))
                self._add(_name(group, dt, 'e_smpl'), dict(mse, proj=0, D=216, p=side('rots', t0=p_t0), q=side('gt_rots', t0=q_t0),
                                                           w='w_smpl'))
                self._add(_name(group, dt, 'e_smpl'), dict(mse, proj=0, D=10, p=side('omega', 75, p_t0),
                                                           q=('gt_shape', 0, 10, 0, q_t0), w='w_smpl'))
            if (group, dt) == ('pred', 0) and T > 1:
                self._add('e_const', dict(kind=_lib.HD_LOSS_MSE_ROWS, proj=0, B=B, Tw=T - 1, K=0, D=10, scale=0.5,
                                          p=side('omega', 75, 1), q=side('omega', 75, 0)))
        if config.do_hallucinate:
            self._add('e_hallucinate', dict(kind=_lib.HD_LOSS_MSE_ROWS, proj=0, B=B, Tw=T, K=0, D=2048, scale=1.,
                                            p=('pred_strips', 0, T * 2048, 2048, 0), q=('strips', 0, T * 2048, 2048, 0)))
        self._add('e_shape', dict(kind=_lib.HD_LOSS_MSE_ROWS, proj=0, B=S * B, Tw=T, K=0, D=10, scale=1., p=('omega', 75, T * 85, 85, 0)))
        keys = loss_keys(config)
        self.names = [k for k in keys if k not in ('d_pose', 'e_pose')]
        w = loss_weights(config)
        self.weights = {k: w[k] for k in keys}
        M = np.zeros((len(self.names), len(self.terms)), np.float32)
        for j, n in enumerate(self.term_names):
            M[self.names.index(n), j] = 1.
        self.matrix = M
        self.cam_frames = [self.terms[i]['B'] * self.terms[i]['Tw'] for i, _ in self.cam_terms]
        self._device_matrix = {}

    def _add(self, name, term):
        self.terms.append(term)
        self.term_names.append(name)

    def shapes(self):
        """Expected shape of each input."""
        S, B, T, K = len(self.sets), self.B, self.T, self.K
        sh = {'omega': (S, B, T, 85), 'joints': (S, B, T, K, 3), 'rots': (S, B, T, 216), 'labels': (B, T, K, 3), 'gt_rots': (B, T, 216),
              'gt_shape': (B, 10), 'gt3ds': (B, T, 14, 3), 'w_joints': (B,), 'w_smpl': (B,), 'strips': (B, T, 2048),
              'pred_strips': (B, T, 2048)}
        return [sh[n] for n in self.inputs]

    def descriptors(self, tensors, cams=None):
        """ctypes array of hd_loss_term over the input tensors (dict slot -> contiguous CUDA float32 tensor)."""
        arr = (_lib.LossTerm * len(self.terms))()
        T = self.T
        cam_off = {}
        o = 0
        for (i, _), n in zip(self.cam_terms, self.cam_frames):
            cam_off[i] = o
            o += n * 3
        for i, t in enumerate(self.terms):
            d = arr[i]
            d.kind, d.proj, d.B, d.Tw, d.K, d.D, d.scale = t['kind'], t['proj'], t['B'], t['Tw'], t['K'], t['D'], t['scale']
            slot, off, clip, frame, t0 = t['p']
            d.p, d.p_clip, d.p_frame, d.p_t0, d.p_T = tensors[slot].data_ptr() + 4 * off, clip, frame, t0, T
            if 'q' in t:
                slot, off, clip, frame, t0 = t['q']
                d.q, d.q_clip, d.q_frame, d.q_t0, d.q_T = tensors[slot].data_ptr() + 4 * off, clip, frame, t0, T
            if 'cam' in t:
                slot, off, clip, frame, _ = t['cam']
                d.cam, d.cam_clip, d.cam_frame = tensors[slot].data_ptr() + 4 * off, clip, frame
            if 'w' in t:
                d.w = tensors[t['w']].data_ptr()
            if cams is not None and i in cam_off:
                d.cam_out = cams.data_ptr() + 4 * cam_off[i]
        return arr

    def cameras(self, cams):
        """The optimal cameras LossFunction returned, split per delta set: {(group, dt): (B, Tw, 3)}."""
        out, o = {}, 0
        for (i, key), n in zip(self.cam_terms, self.cam_frames):
            out[key] = cams[o:o + 3 * n].view(self.B, self.terms[i]['Tw'], 3)
            o += 3 * n
        return out

    def named(self, values):
        """Named losses (one device vector, `names` order) from the term values: the reference's per-key sums.  The 0/1 matrix is
        copied to each device once, so that a training step issues no host-device synchronisation."""
        m = self._device_matrix.get(values.device)
        if m is None:
            m = self._device_matrix[values.device] = torch.from_numpy(self.matrix).to(values.device)
        return m @ values


def build_objective(config, B, T, K):
    return Objective(config, B, T, K)


def _checked(obj, inputs):
    out = {}
    for name, x, shape in zip(obj.inputs, inputs, obj.shapes()):
        if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != F32:
            raise _lib.HDError('LossFunction: %s must be a float32 CUDA tensor (no CPU fallback exists)' % name)
        if tuple(x.shape) != shape:
            raise _lib.HDError('LossFunction: %s has shape %s, expected %s' % (name, tuple(x.shape), shape))
        out[name] = x.contiguous()
    return out


def apply_loss(obj, *inputs):
    """LossFunction.apply, refusing a gradient on an input the objective treats as a constant (labels, weights): the check has to run
    here, outside the Function's forward, where grad mode is still on."""
    if torch.is_grad_enabled():
        for name, x in zip(obj.inputs, inputs):
            if isinstance(x, torch.Tensor) and x.requires_grad and name not in obj.DIFFERENTIABLE:
                raise _lib.HDError('LossFunction: %s takes no gradient (labels and weights are constants); pass it detached' % name)
    return LossFunction.apply(obj, *inputs)


class LossFunction(torch.autograd.Function):
    """(objective, *inputs in objective.inputs order) -> (values [n_terms], optimal cameras [sum of B*Tw*3 over the delta sets])."""

    @staticmethod
    def forward(ctx, obj, *inputs):
        t = _checked(obj, inputs)
        dev = inputs[0].device
        cams = torch.empty(sum(obj.cam_frames) * 3, dtype=F32, device=dev)
        arr = obj.descriptors(t, cams)
        ws_bytes = int(lib.hd_loss_workspace_bytes(arr, len(obj.terms)))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        values = torch.empty(len(obj.terms), dtype=F32, device=dev)
        check(lib.hd_loss_forward(arr, len(obj.terms), C.c_void_p(values.data_ptr()), C.c_void_p(ws.data_ptr()), ws_bytes, current_stream()),
              'hd_loss_forward')
        ctx.obj = obj
        ctx.mark_non_differentiable(cams)
        ctx.save_for_backward(ws, *[t[n] for n in obj.inputs])
        return values, cams

    @staticmethod
    @once_differentiable
    def backward(ctx, dvalues, dcams):
        obj = ctx.obj
        ws, *xs = ctx.saved_tensors
        t = dict(zip(obj.inputs, xs))
        need = ctx.needs_input_grad[1:]
        out = [None] * len(xs)
        targets = [(i, n) for i, n in enumerate(obj.inputs) if need[i] and n in obj.DIFFERENTIABLE]
        if not targets or dvalues is None:
            return (None,) + tuple(out)
        gl = (_lib.LossGrad * len(targets))()
        for j, (i, n) in enumerate(targets):
            out[i] = torch.empty_like(t[n])
            gl[j].src, gl[j].grad, gl[j].numel = t[n].data_ptr(), out[i].data_ptr(), t[n].numel()
        arr = obj.descriptors(t)
        dv = dvalues.contiguous()
        check(lib.hd_loss_backward(arr, len(obj.terms), gl, len(targets), C.c_void_p(dv.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                                   current_stream()), 'hd_loss_backward')
        return (None,) + tuple(out)


def evaluate(obj, inputs):
    """Named losses of an objective: ({name: 0-d tensor}, optimal cameras {(group, dt): (B, Tw, 3)}), differentiable."""
    values, cams = apply_loss(obj, *[inputs[n] for n in obj.inputs])
    named = obj.named(values)
    return {n: named[i] for i, n in enumerate(obj.names)}, obj.cameras(cams)


# ------------------------------------------------------------------------------------------------------------------------------------
# the trainer
# ------------------------------------------------------------------------------------------------------------------------------------
class HMMRTrainer(object):
    """One reference training iteration per `step` (trainer_sequence_fc.py build_model + setup_optimizers + one sess.run of e_opt and
    d_opt): f_movie (and fc2_res with do_hallucinate) over precomputed phis, the IEF heads from the tiled mean_param, one SMPL call over
    every prediction set, the objective, D_pose on reals + fakes, and both updates from the same pre-step parameters.

    `optimizer`: optional factory (params, lr) -> torch optimizer, default torch.optim.Adam; optim.TFAdam is TF's Adam, whose slots and
    beta powers save_checkpoint writes.  `global_step` counts the applied updates like the reference's (both minimize calls pass it:
    +2 per step that trains D, +1 with d_lw_pose = 0); it starts at the checkpoint's when `weights` is a checkpoint prefix, else at 0.
    With config.precomputed_phi=False, `weights` must also hold the resnet_v2_50/* variables (see the module docstring)."""

    def __init__(self, config, weights, smpl_model, disc_weights=None, optimizer=None, device=None):
        from .adversarial import PoseDiscriminator
        from .trainable import TemporalModel
        from src.tf_smpl.batch_smpl import SMPL
        self.config = config
        require_training_impl(config.impl, 'HMMRTrainer')
        grad_one_pass(config.grad_precision, 'HMMRTrainer')
        if config.do_hallucinate and not config.predict_delta:
            raise _lib.HDError('do_hallucinate needs predict_delta (the reference asserts it, src/config.py:271)')
        if not config.freeze_phi and config.precomputed_phi:
            raise _lib.HDError('freeze_phi=False trains the ResNet, which needs image input: set precomputed_phi=False (precomputed '
                               'phis have no trunk to train)')
        self.model = TemporalModel(weights, config, device=device)
        gp = config.grad_precision
        self.trunk = None if config.precomputed_phi else _TrainTrunk(self.model._source, self.model.device,
                                                                     trainable=not config.freeze_phi, grad_precision=gp)
        self._pending = None                  # the trunk plan of the last forward: step applies its update ops
        self.disc = PoseDiscriminator(disc_weights, device=self.model.device, grad_precision=gp) if disc_weights is not None else \
            PoseDiscriminator(seed=0, device=self.model.device, grad_precision=gp)
        self.smpl = smpl_model if hasattr(smpl_model, 'consts') else SMPL(smpl_model)
        make = optimizer or (lambda params, lr: torch.optim.Adam(params, lr))
        self.e_params = list(self.model.parameters())
        if self.trunk is not None and self.trunk.net is not None:     # get_unfrozen_E_vars without freeze_phi: the resnet_v2_50/* variables
            self.e_params += list(self.trunk.net.parameters())
        self.d_params = list(self.disc.parameters())
        self.e_opt = make(self.e_params, config.e_lr)
        self.d_opt = make(self.d_params, config.d_lr)
        self._objectives = {}
        self.global_step = _checkpoint_step(weights)

    @classmethod
    def resume(cls, config, prefix, smpl_model, device=None):
        """Continue a run from its checkpoint (tf.train.Supervisor's restore from logdir, trainer_sequence_fc.py:410-418): E, D and
        the moving statistics from `prefix` as in the constructor, optim.TFAdam for both optimizers with every slot, both pairs of beta
        powers (D's only when d_lw_pose > 0) and global_step restored.  A missing entry raises HDError naming it.  To fine-tune from a
        checkpoint without optimizer state, construct with weights=prefix instead: the slots start at zero."""
        from .optim import TFAdam
        from .tf_checkpoint import is_checkpoint, load_checkpoint
        prefix = prefix[:-len('.index')] if isinstance(prefix, str) and prefix.endswith('.index') else prefix
        if not is_checkpoint(prefix):
            raise _lib.HDError('HMMRTrainer.resume: %r is not a TensorFlow checkpoint prefix (no .index file)' % (prefix,))
        tr = cls(config, prefix, smpl_model, disc_weights=prefix, optimizer=TFAdam, device=device)
        want = tr.optimizer_state_names()
        state = load_checkpoint(prefix, names=set(want))
        missing = [n for n in want if n not in state]
        if missing:
            raise _lib.HDError('HMMRTrainer.resume: %s lacks %d optimizer entries, first: %s' % (prefix, len(missing), missing[0]))
        trained = set(tr._e_names())
        tr.e_opt.load_tf_slots(state, [n if n in trained else None for n in tr._e_param_names()])
        d_trained = config.d_lw_pose > 0
        if d_trained:
            from .adversarial import PARAM_NAMES, stack_heads, tf_names
            d = {}
            for s in ('/Adam', '/Adam_1'):
                d.update({k + s: a for k, a in stack_heads({n: state[n + s] for n in tf_names()}).items() if k in PARAM_NAMES})
            d.update({k: state[k] for k in ('beta1_power_1', 'beta2_power_1')})
            tr.d_opt.load_tf_slots(d, PARAM_NAMES, suffix='_1')
        tr.global_step = int(state['global_step'])
        return tr

    def _e_param_names(self):
        """The TF variable of each of e_params, in order."""
        return list(self.model.names) + (list(self.trunk.net.names) if self.trunk is not None and self.trunk.net is not None else [])

    def _e_names(self):
        """The E variables the reference's optimizer holds (get_unfrozen_E_vars): fc2_res exists in its graph only with
        do_hallucinate, so without it those parameters never get a gradient or slots here either."""
        from .trainable import HAL_NAMES
        return [n for n in self._e_param_names() if self.config.do_hallucinate or n not in HAL_NAMES]

    def optimizer_state_names(self):
        """The optimizer entries a TFAdam trainer's checkpoint holds, as TF names them (E's optimizer is created first in
        setup_optimizers, so its beta powers take the plain names and D's the _1 suffix; D's only when D trains)."""
        from .adversarial import tf_names
        names = [n + s for n in self._e_names() for s in ('/Adam', '/Adam_1')] + ['beta1_power', 'beta2_power']
        if self.config.d_lw_pose > 0:
            names += [n + s for n in tf_names() for s in ('/Adam', '/Adam_1')] + ['beta1_power_1', 'beta2_power_1']
        return names + ['global_step']

    def objective(self, B, T, K):
        key = (B, T, K)
        if key not in self._objectives:
            self._objectives[key] = build_objective(self.config, B, T, K)
        return self._objectives[key]

    def n_fake(self, B, T):
        return n_fake(self.config, B, T)

    def forward(self, batch, mocap_poses):
        """The losses of one iteration on the current parameters, on the autograd graph: (named {key: 0-d tensor}, e_loss, d_loss)."""
        from .smpl import batch_rodrigues
        from src.ops import compute_loss_d_fake, compute_loss_d_real, compute_loss_e_fake
        cfg, model = self.config, self.model
        if cfg.precomputed_phi:
            phis = batch['phis']
        else:
            phis, self._pending = self.trunk(batch['images'])
        B, T = int(phis.shape[0]), int(phis.shape[1])
        K = int(batch['labels'].shape[2])
        obj = self.objective(B, T, K)
        S = len(obj.sets)
        if S * B * T != n_fake(cfg, B, T):
            raise _lib.HDError('prediction sets (%d x %d frames) and the mocap count of the loader (%d) disagree for this config'
                               % (S, B * T, n_fake(cfg, B, T)))
        if tuple(mocap_poses.shape) != (n_fake(cfg, B, T), 216):
            raise _lib.HDError('mocap_poses: expected (%d, 216) = one real pose per fake, got %s'
                               % (n_fake(cfg, B, T), tuple(mocap_poses.shape)))
        N = B * T
        omegas = {}
        strips = model.temporal_encode(phis)
        keys = model.delta_keys if cfg.predict_delta else ()
        om, dl = model.regress(strips.reshape(N, 2048), delta_keys=keys, dropout=self._ief_dropout(0))
        omegas[('pred', 0)] = om
        omegas.update({('dt', k): v for k, v in dl.items()})
        inputs = {}
        if cfg.do_hallucinate:
            pstrips = model.hallucinate(phis)
            hk = keys if cfg.do_hallucinate_preds else ()
            om, dl = model.regress(pstrips.reshape(N, 2048), delta_keys=hk, dropout=self._ief_dropout(1))
            omegas[('hal', 0)] = om
            omegas.update({('hal', k): v for k, v in dl.items()})
            inputs['strips'], inputs['pred_strips'] = strips, pstrips
        omega = torch.cat([omegas[s] for s in obj.sets], 0)
        _, joints, Rs = self.smpl(omega[:, 75:85], omega[:, 3:75], get_skin=True)
        has = batch['has_3d'].to(F32)
        w_smpl = torch.zeros_like(has[:, 1]) if cfg.mosh_ignore else has[:, 1]
        inputs.update(omega=omega.reshape(S, B, T, 85), joints=joints.reshape(S, B, T, K, 3), rots=Rs.reshape(S, B, T, 216),
                      labels=batch['labels'], gt_rots=batch_rodrigues(batch['poses'].reshape(-1, 3)).view(B, T, 216),
                      gt_shape=batch['shape'], gt3ds=batch['gt3ds'].reshape(B, T, 14, 3), w_joints=has[:, 0].contiguous(),
                      w_smpl=w_smpl.contiguous())
        named, cams = evaluate(obj, inputs)
        fakes = Rs.reshape(S * N, 24, 9)[:, 1:]
        reals = mocap_poses.reshape(-1, 24, 9)[:, 1:]
        logits = self.disc(torch.cat([reals, fakes], 0))
        out_real, out_fake = logits[:S * N], logits[S * N:]
        named['e_pose'] = compute_loss_e_fake(out_fake)
        named['d_pose'] = compute_loss_d_fake(out_fake) + compute_loss_d_real(out_real)
        w = obj.weights
        e_loss = sum(named[k] * w[k] for k in obj.names) + named['e_pose'] * w['e_pose']
        d_loss = named['d_pose'] * w['d_pose']
        return {k: named[k] for k in loss_keys(cfg)}, e_loss, d_loss

    def _ief_dropout(self, call):
        """The IEF dropout of call 0 (the pred strips) or 1 (the hal strips) at the current global_step; None with ief_keep_prob 1."""
        p = float(self.config.ief_keep_prob)
        return None if p == 1.0 else (int(self.config.seed), self.global_step, call, p)

    def step(self, batch, mocap_poses):
        """One iteration: both updates computed from the same pre-step parameters, then applied.  e_loss moves the temporal model,
        d_loss D_pose (not at all when d_lw_pose = 0).  Returns {key: loss, 'e_loss', 'd_loss'} as detached device scalars."""
        named, e_loss, d_loss = self.forward(batch, mocap_poses)
        if self._pending is not None:         # UPDATE_OPS, grouped with e_loss (trainer_sequence_fc.py:745-750)
            self._pending.apply_moving_update()
            self._pending = None
        ge = torch.autograd.grad(e_loss, self.e_params, retain_graph=True, allow_unused=True)
        use_d = self.config.d_lw_pose > 0
        gd = torch.autograd.grad(d_loss, self.d_params, allow_unused=True) if use_d else None
        for p, g in zip(self.e_params, ge):
            p.grad = g
        self.e_opt.step()
        self.e_opt.zero_grad(set_to_none=True)
        self.global_step += 1
        if use_d:
            for p, g in zip(self.d_params, gd):
                p.grad = g
            self.d_opt.step()
            self.d_opt.zero_grad(set_to_none=True)
            self.global_step += 1
        out = {k: v.detach() for k, v in named.items()}
        out['e_loss'], out['d_loss'] = e_loss.detach(), d_loss.detach()
        return out

    def tf_variables(self):
        """E and D variables; with image input the trunk's moving statistics are the current ones, and with freeze_phi=False its
        trained weights, biases, gamma and beta as well.  With optim.TFAdam optimizers, also their state (optimizer_state_names()):
        the slots in each variable's shape, the beta powers and global_step (int64).  Optimizer entries that came in with `weights`
        are never passed through."""
        from .optim import TFAdam
        v = {k: a for k, a in self.model.tf_variables().items() if not _optimizer_entry(k)}
        if self.trunk is not None:
            v.update(self.trunk.bn.moving() if self.trunk.net is None else self.trunk.net.tf_variables())
        v.update(self.disc.tf_variables())
        if isinstance(self.e_opt, TFAdam):
            s = self.e_opt.tf_slots(self._e_param_names())
            v.update({k: a.reshape(np.shape(v[k.rsplit('/', 1)[0]])) if k.endswith(('/Adam', '/Adam_1')) else a for k, a in s.items()})
            v['global_step'] = np.asarray(self.global_step, np.int64)
        if isinstance(self.d_opt, TFAdam) and self.config.d_lw_pose > 0:
            from .adversarial import PARAM_NAMES, split_heads
            s = self.d_opt.tf_slots(PARAM_NAMES, suffix='_1')
            for sfx in ('/Adam', '/Adam_1'):
                if all(n + sfx in s for n in PARAM_NAMES):
                    v.update({k + sfx: a for k, a in split_heads({n: s[n + sfx] for n in PARAM_NAMES}).items()})
            v.update({k: s[k] for k in ('beta1_power_1', 'beta2_power_1')})
        return v

    def save_checkpoint(self, prefix):
        """E and D variables in one TensorFlow V2 checkpoint: Tester / HMMREngine read E, PoseDiscriminator reads D."""
        from .tf_checkpoint import save_checkpoint
        save_checkpoint(prefix, self.tf_variables())
        return prefix


def _optimizer_entry(name):
    """A TF optimizer entry rather than a model variable: an Adam slot, a beta power or the step counter."""
    return name.rsplit('/', 1)[-1] in ('Adam', 'Adam_1') or name in ('global_step', 'beta1_power', 'beta2_power', 'beta1_power_1',
                                                                       'beta2_power_1')


def _checkpoint_step(weights):
    """global_step of a checkpoint prefix (load_checkpoint's default skip drops it), 0 for anything else or a checkpoint without one."""
    from .tf_checkpoint import is_checkpoint, load_checkpoint
    if not isinstance(weights, str):
        return 0
    prefix = weights[:-len('.index')] if weights.endswith('.index') else weights
    if not is_checkpoint(prefix):
        return 0
    return int(load_checkpoint(prefix, names=['global_step']).get('global_step', 0))


class _TrainTrunk(object):
    """The ResNet of an image-input trainer: packed once, one ResNetTrainPlan per (frames, size), the moving statistics shared by all of
    them.  Called with images (B, T, S, S, 3) -> (phis (B, T, 2048), the plan that made them): frozen, without autograd; trainable
    (freeze_phi=False), on the graph of trunk.TrainableResNet."""

    def __init__(self, w, device, trainable=False, grad_precision='fp32'):
        from .nets import PackedResNet, ResNetBatchNorm
        from .trunk import conv_names
        missing = [k for k in conv_names() if k not in w]
        if missing:
            raise _lib.HDError('precomputed_phi=False runs the ResNet: weights lack %d resnet_v2_50 variables, e.g. %s'
                               % (len(missing), missing[0]))
        self.device = device
        self.grad_precision = grad_precision
        self._plans = {}
        self.net = None
        if trainable:
            from .trunk import TrainableResNet
            self.net = TrainableResNet(w, device, grad_precision=grad_precision)
            self.bn = self.net.bn
            return
        with torch.cuda.device(device):
            self.bn = ResNetBatchNorm(w, device)
            self.packed = PackedResNet(w, device, tc='auto')

    def plan(self, n, size):
        from .nets import ResNetTrainPlan
        key = (n, size)
        if key not in self._plans:
            self._plans.clear()                   # one batch shape at a time: a plan holds gigabytes of activations at 224 x 224
            self._plans[key] = ResNetTrainPlan(self.packed, self.bn, n, size, grad_precision=self.grad_precision)
        return self._plans[key]

    def __call__(self, images):
        if not isinstance(images, torch.Tensor) or not images.is_cuda or images.dtype != F32 or images.dim() != 5 or \
                images.shape[4] != 3 or images.shape[2] != images.shape[3]:
            raise _lib.HDError('batch["images"] must be a float32 CUDA tensor (B, T, S, S, 3), got %s'
                               % ((images.dtype, tuple(images.shape)) if isinstance(images, torch.Tensor) else type(images),))
        if images.device != self.device:
            raise _lib.HDError('batch["images"] is on %s, the trainer on %s' % (images.device, self.device))
        B, T, S = int(images.shape[0]), int(images.shape[1]), int(images.shape[2])
        if self.net is not None:
            phis, plan = self.net(images.reshape(B * T, S, S, 3))
            return phis.view(B, T, -1), plan
        plan = self.plan(B * T, S)
        phis = torch.empty((B * T, self.packed.out_dim), dtype=F32, device=self.device)
        with torch.no_grad():
            plan.run(images.detach().reshape(B * T, S, S, 3).contiguous(), phis)
        return phis.view(B, T, -1), plan


# ------------------------------------------------------------------------------------------------------------------------------------
# single terms (the src/ drop-ins route through these, so the library path is the only one)
# ------------------------------------------------------------------------------------------------------------------------------------
class _TermList(Objective):
    """An explicit term list over named inputs of given shapes, evaluated by LossFunction like an Objective."""

    def __init__(self, inputs, shapes, terms, T, cam_terms=(), differentiable=('p',)):
        self.inputs, self._shapes, self.terms, self.T = tuple(inputs), [tuple(s) for s in shapes], terms, T
        self.DIFFERENTIABLE = tuple(differentiable)
        self._device_matrix = {}
        self.cam_terms = list(cam_terms)
        self.cam_frames = [terms[i]['B'] * terms[i]['Tw'] for i, _ in self.cam_terms]

    def shapes(self):
        return self._shapes


def kp_loss(kp_gt, kp_pred, optcam=False):
    """compute_loss_e_kp (kp_pred already projected) or, with optcam, compute_loss_e_kp_optcam's loss over N frames: kp_gt (N,K,3),
    kp_pred (N,K,D >= 2).  Returns (loss, best cameras (N,3) or None).  The labels kp_gt are constants: only kp_pred takes a gradient."""
    N, K = kp_gt.shape[0], kp_gt.shape[1]
    D = kp_pred.shape[2]
    t = dict(kind=_lib.HD_LOSS_KP_L1, proj=_lib.HD_LOSS_KP_OPTCAM if optcam else _lib.HD_LOSS_KP_RAW, B=1, Tw=N, K=K, D=D, scale=1.,
             p=('p', 0, N * K * D, K * D, 0), q=('q', 0, N * K * 3, K * 3, 0))
    obj = _TermList(('p', 'q'), [(N, K, D), (N, K, 3)], [t], N, [(0, 'cam')] if optcam else ())
    values, cams = apply_loss(obj, kp_pred, kp_gt)
    return values[0], (cams.view(N, 3) if optcam else None)


def mse_loss(pred, gt, weights=None, scale=1., align=False):
    """scale * tf.losses.mean_squared_error(gt, pred, weights) over N rows (pred (N, ...), gt the same shape or None = 0, weights (N,) or
    None), rows aligned by the pelvis first with `align` (rows of 14+ joints x 3)."""
    N = pred.shape[0]
    D = pred[0].numel()
    names, shapes = ['p'], [tuple(pred.shape)]
    t = dict(kind=_lib.HD_LOSS_MSE_ROWS, proj=int(bool(align)), B=N, Tw=1, K=0, D=D, scale=float(scale), p=('p', 0, D, D, 0))
    args = [pred]
    if gt is not None:
        t['q'] = ('q', 0, D, D, 0)
        names.append('q'), shapes.append(tuple(gt.shape)), args.append(gt)
    if weights is not None:
        t['w'] = 'w'
        names.append('w'), shapes.append((N,)), args.append(weights.reshape(N).to(F32))
    values, _ = apply_loss(_TermList(names, shapes, [t], 1, differentiable=('p', 'q')), *args)
    return values[0]
