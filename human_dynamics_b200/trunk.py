"""The ResNet trunk (slim resnet_v2_50 in training mode) as torch parameters, differentiable on the GPU: what the reference trains with
freeze_phi=False (get_unfrozen_E_vars, trainer_sequence_fc.py:681-685, keeps every trainable resnet_v2_50/* variable in E's optimizer).

The trainable variables are the 53 conv `weights`, the 21 `biases` (conv1, the 4 shortcuts, the 16 conv3) and the 49 batch-norm `gamma`
and `beta`; the moving statistics are not trainable and move only through the update ops (ResNetTrainPlan.apply_moving_update).  The
reference builds the trunk with weight_decay=e_wd (trainer_sequence_fc.py:571), but gather_losses (:700-720) never adds the
regularisation losses to e_loss, so the trunk trains without weight decay, and so does this module.

The forward is nets.ResNetTrainPlan with keep=True (its phis are bit-identical to the frozen trunk's); the backward is the plan's
`backward` (csrc/resnet_grad.cu + hd_conv_gemm 3xTF32, or 1xTF32 with grad_precision='tf32').  A parameter changed in place (optimizer.step()) repacks its forward pack (for
conv1, the padded fp16 plane layout as well) and its data-gradient pack on the device before their next use.

    net = TrainableResNet(weights)                     # anything engine.load_weights accepts, with the resnet_v2_50/* variables
    phis, plan = net(images)                           # images (N, S, S, 3) float32 CUDA in [-1, 1] -> phis (N, 2048) on the graph
    loss(phis).backward(); opt.step()
"""
from __future__ import annotations

import contextlib

import numpy as np
import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import _lib
from .nets import BackwardDataPack, PackedResNet, ResNetBatchNorm, ResNetTrainPlan, RESNET_BLOCKS, grad_one_pass
from .trainable import TrainableModule

F32 = torch.float32


def conv_names(blocks=RESNET_BLOCKS):
    """The trunk's conv weights and biases, in forward order."""
    p = 'resnet_v2_50'
    out = [p + '/conv1/weights', p + '/conv1/biases']
    d_in = 64
    for b, (base, units, _) in enumerate(blocks, start=1):
        for u in range(1, units + 1):
            q = '%s/block%d/unit_%d/bottleneck_v2' % (p, b, u)
            if d_in != 4 * base:
                out += [q + '/shortcut/weights', q + '/shortcut/biases']
            out += [q + '/conv1/weights', q + '/conv2/weights', q + '/conv3/weights', q + '/conv3/biases']
            d_in = 4 * base
    return out


class ResNetFunction(torch.autograd.Function):
    """images (N, S, S, 3) -> phis (N, 2048) through a keep=True ResNetTrainPlan; differentiable w.r.t. the trunk's parameters (the
    images get no gradient).  The backward reads state the forward does not own: the plan's kept maps (rewritten by its next run) and
    the parameters in place (gamma / beta, and the weights through their data-gradient packs).  A graph whose plan has run again, or
    whose parameters were changed in place since (optimizer.step() before backward), refuses its backward instead of returning
    gradients of other values -- the check torch's save_for_backward makes for its own saved tensors."""

    @staticmethod
    def forward(ctx, net, plan, images, *params):
        phis = torch.empty((plan.n, plan.p.out_dim), dtype=F32, device=images.device)
        plan.run(images, phis)
        ctx.net, ctx.plan, ctx.generation = net, plan, plan.generation
        ctx.versions = [q._version for q in params]
        ctx.save_for_backward(images)
        return phis

    @staticmethod
    @once_differentiable
    def backward(ctx, dphi):
        net, plan = ctx.net, ctx.plan
        if plan.generation != ctx.generation:
            raise _lib.HDError('ResNet backward: the trunk ran another forward over this batch shape since this graph was recorded, '
                               'and its saved maps are gone')
        changed = [n for n, v, q in zip(net.names, ctx.versions, (net.param(n) for n in net.names)) if q._version != v]
        if changed:
            raise _lib.HDError('ResNet backward: %d trunk parameters (e.g. %s) were modified in place since this graph was recorded'
                               % (len(changed), changed[0]))
        images, = ctx.saved_tensors
        net.sync_bwd_packs()
        g = plan.backward(dphi.contiguous(), images)
        return (None, None, None) + tuple(net.gradient_of(n, g) for n in net.names)


class TrainableResNet(TrainableModule):
    """The trunk's trainable variables as fp32 parameters on one CUDA device, addressable by TF name (`net.param(name)`), and the
    training-mode forward over them.  The batch-norm gamma / beta parameters share storage with `bn.gamma` / `bn.beta`, which the plans
    read in place; conv weights and biases are read in place by their packs and epilogues.  grad_precision: 'fp32' (3xTF32 weight and
    data gradients) or 'tf32' (1xTF32, nets.GRAD_PRECISIONS); the forward is the same in both."""

    def __init__(self, weights, device=None, blocks=RESNET_BLOCKS, grad_precision='fp32'):
        super().__init__()
        from .engine import load_weights
        grad_one_pass(grad_precision, 'TrainableResNet')
        self.grad_precision = grad_precision
        if not torch.cuda.is_available() and (device is None or torch.device(device).type == 'cuda'):
            raise _lib.HDError('TrainableResNet needs a CUDA device: the hot path has no CPU fallback')
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        w = load_weights(weights) if not isinstance(weights, dict) else weights
        self.blocks = blocks
        cn = conv_names(blocks)
        missing = [k for k in cn if k not in w]
        if missing:
            raise _lib.HDError('TrainableResNet: weights lack %d resnet_v2_50 variables, e.g. %s' % (len(missing), missing[0]))
        self._source = w
        for n in cn:
            self._params[n] = nn.Parameter(torch.tensor(np.asarray(w[n], np.float32), device=self.device))      # a copy
        with torch.cuda.device(self.device) if self.device.type == 'cuda' else contextlib.nullcontext():
            self.bn = ResNetBatchNorm(w, self.device, blocks)
            for i, s in enumerate(self.bn.scopes):
                self._params[s + '/gamma'] = nn.Parameter(self.bn.view(self.bn.gamma, i))
                self._params[s + '/beta'] = nn.Parameter(self.bn.view(self.bn.beta, i))
            wd = dict(w)
            wd.update({n: self._params[n].data for n in cn})
            self.packed = PackedResNet(wd, self.device, tc='auto', blocks=blocks)
            self._build_packs()
        self.names = cn + [s + '/' + k for s in self.bn.scopes for k in ('gamma', 'beta')]
        self._plans = {}

    def _build_packs(self):
        p, pk = self.packed, 'resnet_v2_50'
        self._fwd_packs.append((pk + '/conv1/weights', p.conv1))
        if p.conv1_planes is not None:
            self._fwd_packs.append((pk + '/conv1/weights', p.conv1_planes))
        qs = [n[:-len('/conv1/weights')] for n in conv_names(self.blocks) if n.endswith('bottleneck_v2/conv1/weights')]
        for q, unit in zip(qs, p.units):
            for c in ('shortcut', 'conv1', 'conv2', 'conv3'):
                if c not in unit:
                    continue
                conv, name = unit[c], '%s/%s/weights' % (q, c)
                conv.bwd = BackwardDataPack(self._params[name].data, conv.KH * conv.KW, conv.Cin, conv.Cout)
                self._fwd_packs.append((name, conv))
                self._bwd_packs.append((name, conv.bwd))
        self._packs_written(self.device)

    def plan(self, n, size):
        """The keep=True training plan for n frames of size x size (one batch shape at a time: it holds ~32 MB per frame at 224)."""
        key = (n, size)
        if key not in self._plans:
            self._plans.clear()
            with torch.cuda.device(self.device) if self.device.type == 'cuda' else contextlib.nullcontext():
                self._plans[key] = ResNetTrainPlan(self.packed, self.bn, n, size, keep=True, grad_precision=self.grad_precision)
        return self._plans[key]

    def gradient_of(self, name, grads):
        if name in grads:
            return grads[name]
        i = self.bn.scopes.index(name.rsplit('/', 1)[0])
        return self.bn.view(grads[name.rsplit('/', 1)[1]], i)

    def forward(self, images):
        """images (N, S, S, 3) float32 CUDA -> (phis (N, 2048), the plan that made them: its `apply_moving_update` takes this batch's
        update-op step).  On the autograd graph when grad mode is on and a parameter requires grad."""
        if not isinstance(images, torch.Tensor) or not images.is_cuda or images.dtype != F32 or images.dim() != 4 or images.shape[3] != 3 \
                or images.shape[1] != images.shape[2]:
            raise _lib.HDError('TrainableResNet: images must be a float32 CUDA tensor (N, S, S, 3)')
        if images.device != self.device:
            raise _lib.HDError('TrainableResNet: images on %s, the trunk on %s' % (images.device, self.device))
        n, S = int(images.shape[0]), int(images.shape[1])
        self.sync_packs()
        plan = self.plan(n, S)
        images = images.detach().contiguous()
        if self._grad_on(self.names):
            return ResNetFunction.apply(self, plan, images, *[self._params[k] for k in self.names]), plan
        phis = torch.empty((n, self.packed.out_dim), dtype=F32, device=self.device)
        with torch.no_grad():
            plan.run(images, phis)
        return phis, plan

    def tf_variables(self):
        """{TF name: float32 ndarray}: the trainable variables' current values and the moving statistics."""
        out = {n: self._params[n].detach().cpu().numpy().reshape(np.shape(self._source[n])) for n in self.names if n in self._source}
        for s in self.bn.scopes:
            for k in ('gamma', 'beta'):
                out[s + '/' + k] = self._params[s + '/' + k].detach().cpu().numpy().reshape(np.shape(self._source[s + '/' + k]))
        out.update(self.bn.moving())
        return out


