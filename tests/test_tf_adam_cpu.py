"""TF's Adam checked WITHOUT a GPU: the float32 operation-order restatement (oracle/adam_ref.py) against float64 over 1 000 steps, known
answers of the first step, zero gradients and underflowing beta powers, the checkpoint's optimizer names for do_train.sh's flags, and
every argument error of hd_adam_tf and TFAdam raised before a launch."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import adam_ref as A

F = np.float32
B1, B2, EPS = 0.9, 0.999, 1e-8


def _f64(x):
    """A hyper-parameter as TF holds it (a float32 constant), in float64: the float64 run then differs from the float32 one only by
    the float32 run's roundings."""
    return float(F(x))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.mark.parametrize('lr,scale', [(1e-3, 1.0), (1e-5, 0.05)])
def test_float32_tracks_float64_over_1000_steps(lr, scale):
    rng = np.random.RandomState(0)
    n = 4096
    p0 = rng.normal(0, scale, n).astype(F)
    s32 = [p0.copy(), np.zeros(n, F), np.zeros(n, F)]
    s64 = [p0.astype(np.float64), np.zeros(n), np.zeros(n)]
    w32, w64 = (F(B1), F(B2)), (_f64(B1), _f64(B2))
    worst = 0.0
    for _ in range(1000):
        g = (rng.normal(0, 1, n) * rng.lognormal(0, 2, n)).astype(F)           # magnitudes over several decades
        s32 = list(A.apply_adam_f32(*s32[:1], g, *s32[1:], lr, B1, B2, EPS, *w32))
        s64 = list(A.apply_adam_f64(*s64[:1], g, *s64[1:], _f64(lr), _f64(B1), _f64(B2), _f64(EPS), *w64))
        w32 = A.finish(*w32, B1, B2)
        w64 = A.finish(*w64, _f64(B1), _f64(B2), np.float64)
        assert all(a.dtype == F for a in s32)
        worst = max(worst, *(_rel(a, b) for a, b in zip(s32, s64)))
    # per-tensor relative L2 of p, m and v at every step; the worst measured is 7.9e-7 (p: its roundings add up as a random walk)
    assert worst < 1e-6, worst
    assert abs(float(w32[1]) - w64[1]) / w64[1] < 1e-6


@pytest.mark.parametrize('g', [0.1, -0.37, 1.0, -3.0, 100.0])
def test_first_step_known_answer(g):
    lr = F(1e-3)
    n = 7
    gv = np.full(n, g, F)
    p, m, v = A.apply_adam_f32(np.zeros(n, F), gv, np.zeros(n, F), np.zeros(n, F), lr, B1, B2, EPS, F(B1), F(B2))
    # m = (1 - beta1) g, v = (1 - beta2) g^2 in fp32: 0.1 g and 0.001 g^2 up to the float32 constants 1 - 0.9f, 1 - 0.999f
    assert np.array_equal(m, (F(1) - F(B1)) * gv) and np.array_equal(v, (F(1) - F(B2)) * (gv * gv))
    assert np.allclose(m, 0.1 * g, rtol=3e-7, atol=0) and np.allclose(v, 1e-3 * g * g, rtol=2e-5, atol=0)
    # for |g| >> epsilon the first update is lr * sign(g), whatever |g|
    assert np.allclose(-p, float(lr) * np.sign(g), rtol=1e-5, atol=0)


def test_zero_gradient_from_zero_slots_moves_nothing():
    rng = np.random.RandomState(1)
    p0 = rng.normal(0, 1, 1000).astype(F)
    p, m, v = A.apply_adam_f32(p0, np.zeros_like(p0), np.zeros_like(p0), np.zeros_like(p0), 1e-3, B1, B2, EPS, F(B1), F(B2))
    assert np.array_equal(p, p0) and not m.any() and not v.any()


def test_powers_underflow_without_nan():
    """0.9^t leaves the normal float32 range after about 830 steps.  With gradual underflow (IEEE, as the kernel runs: no flush to
    zero) it then stops at 4 * 2^-149, where 4 * 0.9 = 3.6 rounds back to 4, instead of reaching 0; a flush-to-zero build would give
    0.  Either way 1 - beta1_power is exactly 1 long before, so the update is the same, and finite."""
    b = (F(B1), F(B2))
    for _ in range(1100):
        b = A.finish(*b, B1, B2)
        assert np.isfinite(b[0]) and np.isfinite(b[1])
    tiny = F(2.0 ** -149)
    assert b[0] == 4 * tiny and A.finish(*b, B1, B2)[0] == b[0] and 0 < b[1] < 1
    assert F(1) - b[0] == F(1) and F(1) - F(0) == F(1)
    rng = np.random.RandomState(2)
    p0, g = rng.normal(0, 1, 64).astype(F), rng.normal(0, 1, 64).astype(F)
    z = np.zeros_like(g)
    p, m, v = A.apply_adam_f32(p0, g, z, z, 1e-3, B1, B2, EPS, b[0], b[1])
    p_zero, _, _ = A.apply_adam_f32(p0, g, z, z, 1e-3, B1, B2, EPS, F(0), b[1])
    assert np.isfinite(p).all() and not np.array_equal(p, p0) and np.array_equal(p, p_zero)


# ------------------------------------------------------------------------------------------------------------------------------------
# the checkpoint's optimizer names
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('with_d', [True, False])
def test_optimizer_names_for_do_train_flags(with_d):
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.adversarial import tf_names
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    from human_dynamics_b200.trainable import trainable_names
    # do_train.sh: --batch_size=8 --num_conv_layers 3 --T 20 --do_hallucinate --do_hallucinate_preds (precomputed phis)
    cfg = TrainConfig(batch_size=8, sequence_length=20, num_conv_layers=3, do_hallucinate=True, do_hallucinate_preds=True,
                      d_lw_pose=1. if with_d else 0.)
    w = synthetic.make_synthetic_weights(seed=1, with_hal=True)
    e = trainable_names(w, 3, cfg.delta_t_values)
    stub = types.SimpleNamespace(config=cfg, model=types.SimpleNamespace(names=e), trunk=None)
    stub._e_param_names = lambda: HMMRTrainer._e_param_names(stub)
    stub._e_names = lambda: HMMRTrainer._e_names(stub)
    got = HMMRTrainer.optimizer_state_names(stub)
    want = A.state_names(e, tf_names(), with_d)
    assert got == want
    assert len(set(got)) == len(got)
    assert len(e) == 3 * 8 + 3 * 6 + 1 + 6
    assert len(tf_names()) == 2 * (2 + 23 + 3)                   # D_conv1, D_conv2, the 23 heads, fc1, fc2 and the output layer
    assert len(got) == 2 * len(e) + 2 + (2 * len(tf_names()) + 2 if with_d else 0) + 1
    assert ('beta1_power_1' in got) == with_d and 'beta1_power' in got and got[-1] == 'global_step'
    assert ('D_pose/pose_out_j22/weights/Adam_1' in got) == with_d
    assert 'fc2_res/fc3/biases/Adam' in got and 'mean_param/Adam_1' in got


def test_optimizer_entries_are_not_model_variables(tmp_path):
    from human_dynamics_b200 import tf_checkpoint
    from human_dynamics_b200.objective import _checkpoint_step, _optimizer_entry
    names = A.state_names(['a/weights', 'mean_param'], ['D_pose/D_conv1/weights'], True)
    for n in names:
        assert _optimizer_entry(n), n
    for n in ('a/weights', 'mean_param', 'resnet_v2_50/conv1/biases', 'D_pose/D_conv1/weights', 'x/Adamish'):
        assert not _optimizer_entry(n), n
    # weights read from a checkpoint leave every optimizer entry out (D's beta powers included); global_step is read on its own
    v = {n: np.zeros((), np.int64) if n == 'global_step' else np.ones(3, F) for n in names}
    v['global_step'] = np.asarray(41, np.int64)
    v['a/weights'] = np.ones(3, F)
    prefix = tf_checkpoint.save_checkpoint(str(tmp_path / 'model.ckpt-41'), v)
    assert sorted(tf_checkpoint.load_checkpoint(prefix)) == ['a/weights']
    assert _checkpoint_step(prefix) == 41 and _checkpoint_step(prefix + '.index') == 41 and _checkpoint_step({}) == 0


# ------------------------------------------------------------------------------------------------------------------------------------
# argument errors, before any launch and without a device
# ------------------------------------------------------------------------------------------------------------------------------------
def _table(n, **over):
    from human_dynamics_b200 import _lib
    t = (_lib.AdamTensor * max(1, n))()
    for e in t:
        e.param, e.grad, e.m, e.v, e.numel = 0x1000, 0x2000, 0x3000, 0x4000, 16
    for k, v in over.items():
        setattr(t[0], k, v)
    return t


@pytest.mark.parametrize('case', ['n<0', 'table', 'param', 'grad', 'm', 'v', 'numel', 'powers', 'lr', 'beta1', 'beta2', 'epsilon'])
def test_hd_adam_tf_argument_errors(case):
    from human_dynamics_b200 import _lib
    lib = _lib.lib
    args = dict(t=_table(2), n=2, lr=1e-3, beta1=B1, beta2=B2, epsilon=EPS, powers=C.c_void_p(0x5000))
    if case == 'n<0':
        args['n'] = -1
    elif case == 'table':
        args['t'] = None
    elif case in ('param', 'grad', 'm', 'v'):
        args['t'] = _table(2, **{case: None})
    elif case == 'numel':
        args['t'] = _table(2, numel=-1)
    elif case == 'powers':
        args['powers'] = None
    else:
        args[case] = float('nan') if case in ('lr', 'beta2') else float('inf')
    before = lib.hd_launch_count()
    rc = lib.hd_adam_tf(args['t'], args['n'], args['lr'], args['beta1'], args['beta2'], args['epsilon'], args['powers'], None)
    assert rc == 1                                   # HD_ERR_INVALID
    assert lib.hd_launch_count() == before
    assert b'hd_adam_tf' in lib.hd_last_error()


def test_tfadam_argument_errors():
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200.optim import TFAdam
    p = torch.nn.Parameter(torch.zeros(4))
    for bad in (dict(lr=float('nan')), dict(lr=1e-3, beta1=float('inf')), dict(lr=1e-3, epsilon='x'), dict(lr=1e-3, beta2=None)):
        with pytest.raises(HDError):
            TFAdam([p], **bad)
    opt = TFAdam([p], 1e-3)
    assert opt.defaults == dict(lr=1e-3, beta1=0.9, beta2=0.999, epsilon=1e-8)
    with pytest.raises(HDError, match='one parameter group'):
        opt.add_param_group({'params': [torch.nn.Parameter(torch.zeros(2))]})
    opt.step()                                       # no gradient: nothing to do
    p.grad = torch.ones(4)
    with pytest.raises(HDError, match='CUDA'):       # a CPU parameter
        opt.step()
    q = torch.nn.Parameter(torch.zeros(4, dtype=torch.float64))
    q.grad = torch.ones(4, dtype=torch.float64)
    with pytest.raises(HDError, match='float32'):
        TFAdam([q], 1e-3).step()
    opt.group['lr'] = float('inf')                   # e.g. from a scheduler: checked at every step
    with pytest.raises(HDError, match='finite'):
        opt.step()
    opt.group['lr'] = 1e-3
    opt.zero_grad(set_to_none=True)
    assert not opt.state
    with pytest.raises(HDError, match='2 names for 1 parameters'):
        opt.tf_slots(['a', 'b'])
    b1, b2 = opt.tf_slots(['a'])['beta1_power'], opt.tf_slots(['a'])['beta2_power']
    assert b1 == F(B1) and b2 == F(B2) and b1.dtype == F and b1.shape == ()
    with pytest.raises(HDError, match='a/Adam_1'):
        opt.load_tf_slots({'a/Adam': np.zeros(4, F), 'beta1_power': F(.9), 'beta2_power': F(.999)}, ['a'])
    with pytest.raises(HDError, match='a/Adam has 3 elements'):
        opt.load_tf_slots({'a/Adam': np.zeros(3, F), 'a/Adam_1': np.zeros(4, F), 'beta1_power': F(.9), 'beta2_power': F(.999)}, ['a'])
    assert not opt.state


def test_resume_refuses_a_missing_checkpoint(tmp_path):
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200.objective import HMMRTrainer, TrainConfig
    with pytest.raises(HDError, match='not a TensorFlow checkpoint'):
        HMMRTrainer.resume(TrainConfig(), str(tmp_path / 'model.ckpt-7'), None)
