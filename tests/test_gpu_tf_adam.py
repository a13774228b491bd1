"""GPU: TF's Adam (hd_adam_tf, optim.TFAdam, HMMRTrainer(optimizer=TFAdam), HMMRTrainer.resume).  The kernel against the float32
restatement of oracle/adam_ref.py bit for bit over 50 steps (ragged sizes, a view one float into its buffer, more tensors than one
launch holds, gradients at 1e+-30, zeros and denormals, powers restored as 0 and as denormals) and the beta powers against numpy's
products; the launch count; a step without host synchronisation; None gradients untouched; the repack after a step; the trainer's
step against the restatement applied to its own gradients (phi input with do_train.sh's flags, and the trunk training from images);
the checkpoint's names, global_step and its readers; and a resumed run bit-identical to an uninterrupted one."""
import math

import numpy as np
import pytest
import torch

from oracle import adam_ref as A
from test_gpu_resnet_grad import _batch, _mocap

pytestmark = pytest.mark.gpu

F = np.float32
B1, B2, EPS = 0.9, 0.999, 1e-8


@pytest.fixture(scope='module')
def train_weights():
    from human_dynamics_b200 import synthetic
    return synthetic.make_synthetic_weights(seed=1, with_hal=True)


@pytest.fixture(scope='module')
def smpl(smpl_model):
    from src.tf_smpl.batch_smpl import SMPL
    return SMPL(smpl_model)


def _np(t):
    return t.detach().cpu().numpy()


def _same(a, b):
    """Bit for bit (NaN matching NaN: a gradient of 1e30 squares to inf, and inf - inf in v is NaN in TF's arithmetic too)."""
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _grad(rng, n, step):
    g = (rng.normal(0, 1, n) * rng.lognormal(0, 2, n)).astype(F)
    k = step % 5                                  # special values on a few elements, a different mix each step
    if n >= 8:
        g[0], g[1] = F(1e30) if k == 0 else F(-1e-30), F(1e-40) if k < 3 else F(-3e-42)      # huge / tiny, denormals
        g[2:4] = 0
    return g


class _Ref(object):
    """The float32 restatement over a list of tensors, and the powers."""

    def __init__(self, params, lr, b1p=F(B1), b2p=F(B2)):
        self.p = [a.copy() for a in params]
        self.m = [np.zeros_like(a) for a in params]
        self.v = [np.zeros_like(a) for a in params]
        self.lr, self.b = lr, (F(b1p), F(b2p))

    def step(self, grads, which=None):
        for i, g in enumerate(grads):
            if g is None:
                continue
            self.p[i], self.m[i], self.v[i] = A.apply_adam_f32(self.p[i], g, self.m[i], self.v[i], self.lr, B1, B2, EPS, *self.b)
        self.b = A.finish(*self.b, B1, B2)


def _check(opt, params, ref):
    for i, p in enumerate(params):
        assert _same(_np(p), ref.p[i]), ('param', i)
        st = opt.state.get(p)
        if st:
            assert _same(_np(st['m']), ref.m[i]) and _same(_np(st['v']), ref.v[i]), ('slots', i)
    b1, b2 = opt.powers()
    assert b1.view(np.uint32) == ref.b[0].view(np.uint32) and b2.view(np.uint32) == ref.b[1].view(np.uint32)


SIZES = [1, 3, 4, 5, 1023, (1 << 20) + 3]


@pytest.mark.parametrize('powers', ['fresh', 'zero', 'denormal'])
def test_kernel_bit_exact_over_50_steps(powers):
    from human_dynamics_b200.optim import TFAdam
    rng = np.random.RandomState(7)
    init = [rng.normal(0, 1, n).astype(F) for n in SIZES]
    params = [torch.nn.Parameter(torch.from_numpy(a).cuda()) for a in init]
    buf = torch.from_numpy(rng.normal(0, 1, 4099).astype(F)).cuda()
    view = torch.nn.Parameter(buf[1:4098])          # one float into its buffer: not 16-byte aligned, the element-wise path
    assert view.data_ptr() % 16 == 4
    params.append(view)
    init.append(_np(view).copy())
    lr = 1e-3
    opt = TFAdam(params, lr)
    b0 = {'fresh': (F(B1), F(B2)), 'zero': (F(0), F(0)), 'denormal': (F(3e-41), F(2 ** -149))}[powers]
    ref = _Ref(init, F(lr), *b0)
    if powers != 'fresh':
        names = ['t%d' % i for i in range(len(params))]
        slots = {'t%d/Adam' % i: np.zeros(a.shape, F) for i, a in enumerate(init)}
        slots.update({'t%d/Adam_1' % i: np.zeros(a.shape, F) for i, a in enumerate(init)})
        slots.update(beta1_power=b0[0], beta2_power=b0[1])
        opt.load_tf_slots(slots, names)
    for step in range(50):
        grads = [_grad(rng, a.size, step) for a in init]
        for p, g in zip(params, grads):
            p.grad = torch.from_numpy(g).cuda()
        opt.step()
        ref.step(grads)
        if step in (0, 1, 9, 49):
            _check(opt, params, ref)


def test_buffer_neighbours_of_a_view_untouched():
    from human_dynamics_b200.optim import TFAdam
    buf = torch.arange(64, dtype=torch.float32, device='cuda')
    before = buf.clone()
    view = torch.nn.Parameter(buf[1:62])
    view.grad = torch.ones(61, device='cuda')
    TFAdam([view], 1e-2).step()
    assert torch.equal(buf[0], before[0]) and torch.equal(buf[62:], before[62:])
    assert not torch.equal(buf[1:62], before[1:62])


def test_many_tensors_and_launch_count():
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.optim import TFAdam
    rng = np.random.RandomState(3)
    n = _lib.HD_ADAM_MAX_TENSORS + 44
    sizes = rng.randint(1, 70, n)
    init = [rng.normal(0, 1, int(s)).astype(F) for s in sizes]
    params = [torch.nn.Parameter(torch.from_numpy(a).cuda()) for a in init]
    opt = TFAdam(params, 1e-3)
    ref = _Ref(init, F(1e-3))
    for step in range(3):
        grads = [_grad(rng, a.size, step) for a in init]
        for p, g in zip(params, grads):
            p.grad = torch.from_numpy(g).cuda()
        torch.cuda.synchronize()
        _lib.lib.hd_launch_count_reset()
        opt.step()
        assert _lib.lib.hd_launch_count() == math.ceil(n / _lib.HD_ADAM_MAX_TENSORS) + 1
        ref.step(grads)
    _check(opt, params, ref)


def test_step_without_host_sync_and_none_gradients():
    from human_dynamics_b200.optim import TFAdam
    rng = np.random.RandomState(4)
    init = [rng.normal(0, 1, (33, 7)).astype(F), rng.normal(0, 1, 100).astype(F), rng.normal(0, 1, 5).astype(F)]
    params = [torch.nn.Parameter(torch.from_numpy(a).cuda()) for a in init]
    opt = TFAdam(params, 1e-3)
    ref = _Ref(init, F(1e-3))
    plan = [(True, False, True), (True, True, False), (False, True, True)]
    for step, has in enumerate(plan):
        grads = [rng.normal(0, 1, a.shape).astype(F) if h else None for a, h in zip(init, has)]
        for p, g in zip(params, grads):
            p.grad = None if g is None else torch.from_numpy(g).cuda()
        versions = [p._version for p in params]
        slots = {i: (opt.state[p]['m'].clone(), opt.state[p]['v'].clone()) for i, p in enumerate(params) if opt.state.get(p)}
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            opt.step()
        finally:
            torch.cuda.set_sync_debug_mode('default')
        ref.step(grads)
        for i, (p, g) in enumerate(zip(params, grads)):
            if g is None:                              # no gradient: parameter, version and slots untouched (no slots before its first)
                assert p._version == versions[i]
                assert (i in slots) == bool(opt.state.get(p))
                if i in slots:
                    assert torch.equal(opt.state[p]['m'], slots[i][0]) and torch.equal(opt.state[p]['v'], slots[i][1])
            else:
                assert p._version > versions[i]
        _check(opt, params, ref)


def test_rejected_inputs_launch_nothing():
    from human_dynamics_b200 import _lib
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200.optim import TFAdam
    p = torch.nn.Parameter(torch.zeros(8, device='cuda'))
    q = torch.nn.Parameter(torch.zeros(8, 2, device='cuda'))
    d = torch.nn.Parameter(torch.zeros(8, device='cuda', dtype=torch.float64))
    # (torch itself refuses a .grad of another dtype, device or shape than its parameter)
    cases = [
        (d, torch.ones(8, device='cuda', dtype=torch.float64), 'float32'),
        (p, torch.ones(16, device='cuda')[::2], 'contiguous'),
        (p, torch.ones(8, device='cuda').to_sparse(), 'sparse'),
        (q, torch.ones(2, 8, device='cuda').t(), 'contiguous'),
    ]
    for param, g, what in cases:
        opt = TFAdam([param], 1e-3)
        param.grad = g
        _lib.lib.hd_launch_count_reset()
        with pytest.raises(HDError, match=what):
            opt.step()
        assert _lib.lib.hd_launch_count() == 0 and not opt.state
        param.grad = None
    nc = torch.nn.Parameter(torch.zeros(4, 4, device='cuda').t())
    nc.grad = torch.zeros(4, 4, device='cuda').t()
    with pytest.raises(HDError, match='contiguous'):
        TFAdam([nc], 1e-3).step()


def test_state_dict_round_trip():
    from human_dynamics_b200.optim import TFAdam
    rng = np.random.RandomState(5)
    init = [rng.normal(0, 1, 300).astype(F), rng.normal(0, 1, (4, 9)).astype(F)]
    mk = lambda: [torch.nn.Parameter(torch.from_numpy(a).cuda()) for a in init]    # noqa: E731
    pa, pb = mk(), mk()
    oa = TFAdam(pa, 1e-3)
    grads = [[torch.from_numpy(rng.normal(0, 1, a.shape).astype(F)).cuda() for a in init] for _ in range(4)]
    for g in grads[:2]:
        for p, x in zip(pa, g):
            p.grad = x
        oa.step()
    for p, q in zip(pa, pb):
        q.data.copy_(p.data)
    ob = TFAdam(pb, 1e-3)
    ob.load_state_dict(oa.state_dict())
    assert ob.powers() == oa.powers()
    for g in grads[2:]:
        for opt, ps in ((oa, pa), (ob, pb)):
            for p, x in zip(ps, g):
                p.grad = x
            opt.step()
    assert all(torch.equal(p, q) for p, q in zip(pa, pb))
    assert all(torch.equal(oa.state[p][k], ob.state[q][k]) for p, q in zip(pa, pb) for k in ('m', 'v'))
    assert ob.powers() == oa.powers()
    s = oa.tf_slots(['a', 'b'])
    assert s['b/Adam'].shape == (4, 9) and s['beta1_power'] == oa.powers()[0]


def test_temporal_model_repacks_after_a_step(train_weights):
    from human_dynamics_b200.optim import TFAdam
    from human_dynamics_b200.trainable import TemporalModel
    model = TemporalModel(train_weights)
    rng = np.random.RandomState(6)
    phi = torch.from_numpy(rng.normal(0, 1, (2, 8, 2048)).astype(F)).cuda()
    with torch.no_grad():
        model.regress(model.temporal_encode(phi).reshape(16, 2048))          # packs built and used once
    opt = TFAdam(model.parameters(), 1e-2)
    for p in model.parameters():
        p.grad = torch.from_numpy(rng.normal(0, 1, tuple(p.shape)).astype(F)).cuda()
    opt.step()
    fresh = TemporalModel(model.tf_variables())
    with torch.no_grad():
        a = model.temporal_encode(phi)
        b = fresh.temporal_encode(phi)
        assert torch.equal(a, b)
        oa, da = model.regress(a.reshape(16, 2048))
        ob, db = fresh.regress(b.reshape(16, 2048))
        assert torch.equal(oa, ob) and all(torch.equal(da[k], db[k]) for k in da)
        assert torch.equal(model.hallucinate(phi), fresh.hallucinate(phi))


# ------------------------------------------------------------------------------------------------------------------------------------
# the trainer
# ------------------------------------------------------------------------------------------------------------------------------------
def _phi_batch(B, T, seed):
    b = _batch(B, T, 16, seed)
    del b['images']
    b['phis'] = torch.from_numpy(np.random.RandomState(seed + 1).normal(0, 1, (B, T, 2048)).astype(F)).cuda()
    return b


def _setup(kind):
    """(config kwargs, B, T, batch maker): do_train.sh's flags over phis, or the trunk training from 64 x 64 images."""
    from human_dynamics_b200.objective import TrainConfig
    if kind == 'phi':
        cfg = TrainConfig(num_conv_layers=3, do_hallucinate=True, do_hallucinate_preds=True, e_lr=1e-4)
        return cfg, 2, 6, lambda s: _phi_batch(2, 6, s)
    cfg = TrainConfig(precomputed_phi=False, freeze_phi=False, e_lr=1e-4)
    return cfg, 2, 4, lambda s: _batch(2, 4, 64, s)


@pytest.mark.parametrize('kind', ['phi', 'image'])
def test_trainer_step_is_the_restatement(train_weights, smpl, smpl_model, kind, tmp_path):
    from human_dynamics_b200.adversarial import PoseDiscriminator, tf_names
    from human_dynamics_b200.engine import HMMREngine, load_weights
    from human_dynamics_b200.objective import HMMRTrainer
    from human_dynamics_b200.optim import TFAdam
    cfg, B, T, mk = _setup(kind)
    twin = HMMRTrainer(cfg, train_weights, smpl, optimizer=TFAdam)
    tr = HMMRTrainer(cfg, train_weights, smpl, optimizer=TFAdam)
    assert tr.global_step == 0 and isinstance(tr.e_opt, TFAdam) and isinstance(tr.d_opt, TFAdam)
    batch, mocap = mk(5), _mocap(tr.n_fake(B, T), 6)
    # the gradients of that step's backward, from an identical trainer (the forward and backward are deterministic)
    _, e_loss, d_loss = twin.forward(batch, mocap)
    ge = torch.autograd.grad(e_loss, twin.e_params, retain_graph=True, allow_unused=True)
    gd = torch.autograd.grad(d_loss, twin.d_params, allow_unused=True)
    before = [_np(p).copy() for p in tr.e_params + tr.d_params]
    tr.step(batch, mocap)
    ne = len(tr.e_params)
    for lr, sl, gs in ((cfg.e_lr, slice(0, ne), ge), (cfg.d_lr, slice(ne, None), gd)):
        ref = _Ref(before[sl], F(lr))
        ref.step([None if g is None else _np(g) for g in gs])
        ps = (tr.e_params + tr.d_params)[sl]
        opt = tr.e_opt if sl.start == 0 else tr.d_opt
        _check(opt, ps, ref)
    assert tr.global_step == 2
    tr.step(mk(7), _mocap(tr.n_fake(B, T), 8))
    assert tr.global_step == 4
    # the checkpoint: the variables plus exactly the oracle's optimizer entries, each slot in its variable's shape
    prefix = tr.save_checkpoint(str(tmp_path / 'model.ckpt-4'))
    from human_dynamics_b200.tf_checkpoint import load_checkpoint
    allv = load_checkpoint(prefix, skip=lambda n: False)
    plain = HMMRTrainer(cfg, train_weights, smpl)                         # torch Adam: the variables alone, as before
    var_names = set(plain.tf_variables())
    assert 'global_step' not in var_names
    want = A.state_names(tr._e_names(), tf_names(), True)
    assert sorted(set(allv) - var_names) == sorted(want) and var_names <= set(allv)
    assert allv['global_step'].dtype == np.int64 and int(allv['global_step']) == 4
    for n in want:
        if n.endswith(('/Adam', '/Adam_1')):
            assert allv[n].shape == allv[n.rsplit('/', 1)[0]].shape, n
    b = A.finish(*A.finish(F(B1), F(B2), B1, B2), B1, B2)
    assert allv['beta1_power'] == b[0] and allv['beta1_power_1'] == b[0] and allv['beta2_power_1'] == b[1]
    # its readers
    w = load_weights(prefix)
    assert not any(n in w for n in want)
    d = PoseDiscriminator(prefix)
    x = _mocap(5, 1).reshape(5, 24, 9)[:, 1:].contiguous()
    with torch.no_grad():
        assert torch.equal(d(x), tr.disc(x))
    if kind == 'image':
        phi = HMMREngine(prefix, smpl_model).encode_images(batch['images'].reshape(B * T, 64, 64, 3))
        assert bool(torch.isfinite(phi).all())
        return
    from human_dynamics_b200.config import HMMRConfig
    from human_dynamics_b200 import synthetic
    from src.evaluation.tester import Tester
    hc = HMMRConfig(load_path=prefix, batch_size=1, sequence_length=20)
    hc.smpl_model = smpl_model
    res = Tester(hc).predict(synthetic.make_images(20, seed=4).reshape(1, 20, 224, 224, 3), copy=True)
    assert np.isfinite(np.asarray(res['omegas'])).all()


def test_trainer_without_d_counts_one_per_step(train_weights, smpl, tmp_path):
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from human_dynamics_b200.adversarial import tf_names
    from human_dynamics_b200.optim import TFAdam
    from human_dynamics_b200.tf_checkpoint import load_checkpoint
    cfg = TrainConfig(d_lw_pose=0.)
    tr = HMMRTrainer(cfg, train_weights, smpl, optimizer=TFAdam)
    for s in range(3):
        tr.step(_phi_batch(2, 5, s), _mocap(tr.n_fake(2, 5), s))
    assert tr.global_step == 3 and not tr.d_opt.state
    prefix = tr.save_checkpoint(str(tmp_path / 'model.ckpt-3'))
    allv = load_checkpoint(prefix, skip=lambda n: False)
    assert 'beta1_power_1' not in allv and not any(k.startswith('D_pose') and k.endswith('Adam') for k in allv)
    assert sorted(k for k in allv if k not in HMMRTrainer(cfg, train_weights, smpl).tf_variables()) == \
        sorted(A.state_names(tr._e_names(), tf_names(), False))
    # a new trainer from that checkpoint starts its count there; resume restores it too
    assert HMMRTrainer(cfg, prefix, smpl).global_step == 3
    assert HMMRTrainer.resume(cfg, prefix, smpl).global_step == 3


@pytest.mark.parametrize('kind', ['phi', 'image'])
def test_resume_is_bit_identical(train_weights, smpl, kind, tmp_path):
    from human_dynamics_b200.objective import HMMRTrainer, n_fake
    from human_dynamics_b200.optim import TFAdam
    cfg, B, T, mk = _setup(kind)
    k = 2
    data = [(mk(20 + s), _mocap(n_fake(cfg, B, T), 40 + s)) for s in range(2 * k)]
    straight = HMMRTrainer(cfg, train_weights, smpl, optimizer=TFAdam)
    losses_a = [straight.step(*d) for d in data]
    first = HMMRTrainer(cfg, train_weights, smpl, optimizer=TFAdam)
    for d in data[:k]:
        first.step(*d)
    prefix = first.save_checkpoint(str(tmp_path / ('model.ckpt-%d' % first.global_step)))
    del first
    resumed = HMMRTrainer.resume(cfg, prefix, smpl)
    assert resumed.global_step == 2 * k
    losses_b = [resumed.step(*d) for d in data[k:]]
    for la, lb in zip(losses_a[k:], losses_b):
        for key in la:
            assert torch.equal(la[key], lb[key]), key
    va, vb = straight.tf_variables(), resumed.tf_variables()
    assert sorted(va) == sorted(vb)
    for n in va:
        assert np.array_equal(va[n], vb[n]) and np.asarray(va[n]).dtype == np.asarray(vb[n]).dtype, n
    assert int(vb['global_step']) == 4 * k


def test_resume_names_a_missing_entry(train_weights, smpl, tmp_path):
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from human_dynamics_b200.optim import TFAdam
    from human_dynamics_b200.tf_checkpoint import save_checkpoint
    cfg = TrainConfig()
    tr = HMMRTrainer(cfg, train_weights, smpl, optimizer=TFAdam)
    tr.step(_phi_batch(2, 5, 1), _mocap(tr.n_fake(2, 5), 1))
    v = tr.tf_variables()
    for drop in ('mean_param/Adam_1', 'D_pose/pose_out_j7/biases/Adam'):
        w = {n: a for n, a in v.items() if n != drop}
        prefix = save_checkpoint(str(tmp_path / ('m-' + drop.replace('/', '_'))), w)
        with pytest.raises(HDError, match=drop):
            HMMRTrainer.resume(cfg, prefix, smpl)
    # a checkpoint without optimizer state fine-tunes with fresh slots
    plain = save_checkpoint(str(tmp_path / 'plain'), HMMRTrainer(cfg, train_weights, smpl).tf_variables())
    ft = HMMRTrainer(cfg, plain, smpl, optimizer=TFAdam)
    assert ft.global_step == 0 and not ft.e_opt.state
