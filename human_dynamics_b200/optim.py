"""TensorFlow's Adam as a torch optimizer: `TFAdam(params, lr, beta1=0.9, beta2=0.999, epsilon=1e-8)`, tf.train.AdamOptimizer's
defaults and arithmetic (TF 1.8's ApplyAdam, use_nesterov=False), one `hd_adam_tf` launch per step (csrc/adam.cu).

It differs from torch.optim.Adam where a fine-tune spends its first steps: TF adds epsilon to sqrt(v) and folds both bias corrections
into the step size, alpha = lr * sqrt(1 - beta2^t) / (1 - beta1^t); torch adds epsilon to sqrt(v_hat).  The beta powers are two device
scalars advanced once per step after every tensor (TF's _finish), so a step neither synchronises nor copies from the host.

    opt = TFAdam(model.parameters(), lr=1e-5)
    loss.backward(); opt.step()
    slots = opt.tf_slots(names)          # {name/Adam: m, name/Adam_1: v, beta1_power: .., beta2_power: ..} for a TF checkpoint
    opt.load_tf_slots(variables, names)  # the reverse: continue a run from such a checkpoint

As in TF's apply_gradients, a parameter whose .grad is None is left alone with its slots, and its slots are created at its first
gradient.  Every tensor is a float32 CUDA tensor, contiguous, with a dense gradient on the parameter's device; anything else raises
HDError before a launch.  One parameter group (TF's optimizer has one learning rate); its 'lr' is read at every step.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from ._lib import check, current_stream, lib

F32 = torch.float32


class TFAdam(torch.optim.Optimizer):

    def __init__(self, params, lr, beta1=0.9, beta2=0.999, epsilon=1e-8):
        hyper = {}
        for k, x in (('lr', lr), ('beta1', beta1), ('beta2', beta2), ('epsilon', epsilon)):
            try:
                hyper[k] = float(x)
            except (TypeError, ValueError):
                raise _lib.HDError('TFAdam: %s must be a number, got %r' % (k, x)) from None
            if not math.isfinite(hyper[k]):
                raise _lib.HDError('TFAdam: %s must be finite, got %r' % (k, x))
        super().__init__(params, hyper)
        self._powers = None               # device float32 [beta1_power, beta2_power], created with the first slots
        self._plan = None                 # (param ids, param pointers, launch table, device) of the last step's parameter set

    def add_param_group(self, group):
        if self.param_groups:
            raise _lib.HDError('TFAdam takes one parameter group (tf.train.AdamOptimizer has one learning rate and one pair of beta '
                               'powers)')
        super().add_param_group(group)

    @property
    def group(self):
        return self.param_groups[0]

    def _new_powers(self, device, b1, b2):
        p = torch.empty(2, dtype=F32, device=device)       # two fills, not a host copy: a step never waits on the host
        p[0].fill_(b1)
        p[1].fill_(b2)
        return p

    @torch.no_grad()
    def step(self, closure=None):
        """One hd_adam_tf call over every non-empty parameter that has a gradient (none: nothing happens, the powers included)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        g = self.group
        for k in ('lr', 'beta1', 'beta2', 'epsilon'):
            if not math.isfinite(float(g[k])):
                raise _lib.HDError('TFAdam: %s must be finite, got %r' % (k, g[k]))
        items = [p for p in g['params'] if p.grad is not None and p.numel() > 0]
        if not items:
            return loss
        grads = [p.grad for p in items]
        # torch's .grad setter already holds a gradient to its parameter's dtype, device and shape; the layout is left to check
        for i, d in enumerate(grads):
            if d.layout is not torch.strided or not d.is_contiguous():
                raise _lib.HDError('TFAdam: parameter %d (shape %s): the gradient must be dense and contiguous (sparse: %s)'
                                   % (i, tuple(items[i].shape), d.is_sparse))
        pptr = [p.data_ptr() for p in items]
        plan = self._plan
        if plan is None or plan[0] != [id(p) for p in items] or plan[1] != pptr:
            plan = self._plan = self._make_plan(items, pptr)
        table = plan[2]
        table[:, 1] = [d.data_ptr() for d in grads]
        with torch.cuda.device(plan[3]):
            check(lib.hd_adam_tf(table.ctypes.data_as(C.POINTER(_lib.AdamTensor)), len(table), g['lr'], g['beta1'], g['beta2'],
                                 g['epsilon'], C.c_void_p(self._powers.data_ptr()), current_stream()), 'hd_adam_tf')
        # a raw-pointer write does not move the version counter that trainable.TrainableModule's repacking and the stale-graph check in
        # trunk.py read
        torch.autograd.graph.increment_version(items)
        return loss

    def _make_plan(self, items, pptr):
        """Validate a parameter set, create the slots it lacks and the powers, and lay out its hd_adam_tensor table (grad column
        filled per step).  Raises HDError before anything is created."""
        dev = self._powers.device if self._powers is not None else items[0].device
        for i, p in enumerate(items):
            what = 'TFAdam: parameter %d (shape %s)' % (i, tuple(p.shape))
            if not p.is_cuda or p.dtype != F32 or not p.is_contiguous():
                raise _lib.HDError('%s must be a contiguous float32 CUDA tensor (no CPU fallback exists), got %s %s%s'
                                   % (what, p.device, p.dtype, '' if p.is_contiguous() else ', non-contiguous'))
            if p.device != dev:
                raise _lib.HDError('%s is on %s, the optimizer on %s' % (what, p.device, dev))
            st = self.state.get(p)
            if st and any(st[k].shape != p.shape or st[k].device != dev or st[k].dtype != F32 or not st[k].is_contiguous()
                          for k in ('m', 'v')):
                raise _lib.HDError('%s: its slots do not match it' % what)
        with torch.cuda.device(dev):
            for p in items:
                st = self.state[p]
                if not st:
                    st['m'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st['v'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            if self._powers is None:
                self._powers = self._new_powers(dev, self.group['beta1'], self.group['beta2'])
        rows = [(pp, 0, self.state[p]['m'].data_ptr(), self.state[p]['v'].data_ptr(), p.numel()) for p, pp in zip(items, pptr)]
        table = np.array(rows, np.int64).reshape(len(items), 5)        # hd_adam_tensor: four pointers and a long long, 40 bytes
        return [id(p) for p in items], pptr, table, dev

    # ---------------------------------------------------------------- state
    def state_dict(self):
        sd = super().state_dict()
        sd['tf_powers'] = None if self._powers is None else self._powers.detach().clone()
        return sd

    def load_state_dict(self, state_dict):
        sd = dict(state_dict)
        powers = sd.pop('tf_powers', None)
        super().load_state_dict(sd)
        self._plan = None
        for st in self.state.values():            # own copies: torch's loader may hand back the very tensors of a live optimizer
            for k in ('m', 'v'):
                if k in st:
                    st[k] = st[k].clone(memory_format=torch.contiguous_format)
        if powers is None:
            self._powers = None
            return
        params = self.group['params']
        dev = params[0].device if params else torch.device('cuda')
        self._powers = torch.as_tensor(powers, dtype=F32).reshape(2).to(dev).clone()

    def powers(self):
        """(beta1_power, beta2_power) as float32 numbers: beta1 and beta2 before the first step."""
        if self._powers is None:
            return np.float32(self.group['beta1']), np.float32(self.group['beta2'])
        a = self._powers.cpu().numpy()
        return a[0], a[1]

    def tf_slots(self, names, suffix=''):
        """{name/Adam: m, name/Adam_1: v (float32 ndarrays in the parameter's shape), beta1_power<suffix>, beta2_power<suffix> (float32
        scalars)}: names[i] is the TF variable of the group's i-th parameter.  A parameter that has had no gradient has no slots, as in
        TF.  The suffix names the powers of a second optimizer in one graph (TF uniquifies them: beta1_power_1, ...)."""
        params = self.group['params']
        if len(names) != len(params):
            raise _lib.HDError('TFAdam.tf_slots: %d names for %d parameters' % (len(names), len(params)))
        out = {}
        for n, p in zip(names, params):
            st = self.state.get(p)
            if st:
                out[n + '/Adam'] = st['m'].detach().cpu().numpy()
                out[n + '/Adam_1'] = st['v'].detach().cpu().numpy()
        b1, b2 = self.powers()
        out['beta1_power' + suffix] = np.asarray(b1, np.float32)
        out['beta2_power' + suffix] = np.asarray(b2, np.float32)
        return out

    def load_tf_slots(self, variables, names, suffix=''):
        """Set every parameter's slots and the powers from TF-named arrays (tf_slots' names; a slot may have the TF variable's shape,
        it is read in the parameter's).  A parameter named None keeps no slots (TF holds none for a variable without a gradient).  A
        missing entry or a size mismatch raises HDError naming it, before anything changes."""
        params = self.group['params']
        if len(names) != len(params):
            raise _lib.HDError('TFAdam.load_tf_slots: %d names for %d parameters' % (len(names), len(params)))
        params = [p for n, p in zip(names, params) if n is not None]
        names = [n for n in names if n is not None]
        want = [n + s for n in names for s in ('/Adam', '/Adam_1')] + ['beta1_power' + suffix, 'beta2_power' + suffix]
        missing = [k for k in want if k not in variables]
        if missing:
            raise _lib.HDError('TFAdam.load_tf_slots: %d entries missing, first: %s' % (len(missing), missing[0]))
        for n, p in zip(names, params):
            for s in ('/Adam', '/Adam_1'):
                if np.size(variables[n + s]) != p.numel():
                    raise _lib.HDError('TFAdam.load_tf_slots: %s has %d elements, the parameter %d'
                                       % (n + s, np.size(variables[n + s]), p.numel()))
        for k in want[-2:]:
            if np.size(variables[k]) != 1:
                raise _lib.HDError('TFAdam.load_tf_slots: %s must be a scalar' % k)
        self._plan = None
        self.state.clear()
        for n, p in zip(names, params):
            self.state[p] = {k: torch.from_numpy(np.ascontiguousarray(np.asarray(variables[n + s], np.float32)).reshape(tuple(p.shape)))
                             .to(p.device) for k, s in (('m', '/Adam'), ('v', '/Adam_1'))}
        dev = params[0].device if params else torch.device('cuda')
        pw = np.array([np.asarray(variables[k], np.float32).reshape(()) for k in want[-2:]], np.float32)
        self._powers = torch.from_numpy(pw).to(dev)
