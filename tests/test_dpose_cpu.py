"""CPU: the D_pose fixture (tests/golden/dpose_v1.npz, made by tests/golden/make_dpose_golden.py from the reference's own
discriminators.py and ops.py), the numpy oracle (oracle/dpose_ref.py) against it and against finite differences, the variable names
PoseDiscriminator exports, and the C-ABI's argument checks (no device needed)."""
import ctypes
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GEN = os.path.join(HERE, 'golden', 'make_dpose_golden.py')


def _gen():
    spec = importlib.util.spec_from_file_location('_make_dpose_golden', GEN)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def gold():
    with np.load(os.path.join(HERE, 'golden', 'dpose_v1.npz')) as z:
        return {k: z[k] for k in z.files}


def test_golden_inputs_regenerate(gold):
    w, xr, xf, beta = _gen().inputs()
    assert np.array_equal(xr, gold['x_real']) and np.array_equal(xf, gold['x_fake']) and np.array_equal(beta, gold['beta'])
    for n, s in zip(gold['var_names'], gold['var_shapes']):
        assert tuple(np.shape(w[str(n)])) == tuple(int(d) for d in s if d), n


@pytest.mark.skipif(not os.path.isdir(os.path.join(os.environ.get('HD_REFERENCE_ROOT', '/nonexistent'), 'src')),
                    reason='HD_REFERENCE_ROOT does not name a reference checkout')
def test_golden_generator_reproduces_the_fixture():
    r = subprocess.run([sys.executable, GEN, '--check'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout


def test_variable_names_match_tf_variables(gold):
    """The names and shapes the reference's graph creates are what PoseDiscriminator.tf_variables() writes (checked on the host side of
    the export: adversarial.tf_names and synthetic.DPOSE_LAYERS)."""
    from human_dynamics_b200 import adversarial, synthetic
    names = [str(n) for n in gold['var_names']]
    assert names == adversarial.tf_names()
    shapes = {str(n): tuple(int(d) for d in s if d) for n, s in zip(gold['var_names'], gold['var_shapes'])}
    for layer, shape in synthetic.DPOSE_LAYERS:
        assert shapes['D_pose/%s/weights' % layer] == shape
        assert shapes['D_pose/%s/biases' % layer] == (shape[-1],)


def test_oracle_matches_golden(gold):
    from oracle import dpose_ref as R
    w = _gen().inputs()[0]
    x = np.concatenate([gold['x_real'], gold['x_fake']]).reshape(-1, 23, 9)
    out32, _ = R.forward(x.astype(np.float32), R.params_from_tf(w, np.float32))
    out64, _ = R.forward(x.astype(np.float64), R.params_from_tf(w, np.float64))
    ref = gold['logits']
    assert np.abs(out32 - ref).max() <= 1e-5 * np.abs(ref).max()
    assert np.abs(out64 - ref).max() <= 1e-5 * np.abs(ref).max()
    nr = len(gold['x_real'])
    for got, key in ((R.loss_e_fake(out32[nr:]), 'e_pose'), (R.loss_d_fake(out32[nr:]), 'd_fake'), (R.loss_d_real(out32[:nr]), 'd_real'),
                     (R.loss_shape(gold['beta']), 'e_shape')):
        assert abs(got - gold[key]) <= 1e-5 * abs(gold[key]), key


def test_dropin_losses_match_golden(gold):
    from src import ops
    nr = len(gold['x_real'])
    out = torch.from_numpy(gold['logits'])
    assert abs(ops.compute_loss_e_fake(out[nr:]).item() - gold['e_pose']) <= 1e-6 * abs(gold['e_pose'])
    assert abs(ops.compute_loss_d_fake(out[nr:]).item() - gold['d_fake']) <= 1e-6 * abs(gold['d_fake'])
    assert abs(ops.compute_loss_d_real(out[:nr]).item() - gold['d_real']) <= 1e-6 * abs(gold['d_real'])
    assert abs(ops.compute_loss_shape(torch.from_numpy(gold['beta'])).item() - gold['e_shape']) <= 1e-6 * abs(gold['e_shape'])


def _small_params(seed):
    """Float64 parameters with the real shapes but random biases, so every site is exercised."""
    from human_dynamics_b200 import synthetic
    from oracle import dpose_ref as R
    return R.params_from_tf(synthetic.make_dpose_weights(seed, bias_scale=0.2), np.float64)


@pytest.mark.parametrize('N', [1, 3])
def test_oracle_backward_gradcheck(N):
    """torch.autograd.gradcheck (fast mode: random directional derivatives) of the oracle's hand-written backward, w.r.t. x and every
    parameter at the real sizes, against finite differences."""
    from oracle import dpose_ref as R
    p = _small_params(5)
    H = 1024
    rng = np.random.RandomState(N)
    x = torch.from_numpy(rng.normal(0, 0.7, size=(N, 23, 9))).requires_grad_()
    leaves = {k: torch.from_numpy(np.ascontiguousarray(v)).requires_grad_() for k, v in p.items()}
    assert leaves['Wf2'].shape == (H, H)
    assert torch.autograd.gradcheck(lambda x, *ps: R.torch_apply(x, dict(zip(R.KEYS, ps))), (x,) + tuple(leaves[k] for k in R.KEYS),
                                    eps=1e-6, atol=1e-5, rtol=1e-4, fast_mode=True)


def test_oracle_float64_self_consistent():
    """float64 forward = float64 forward of the float32-rounded parameters to float32 precision, and the loss gradient's linearity."""
    from oracle import dpose_ref as R
    p = _small_params(6)
    x = np.random.RandomState(1).normal(0, 0.7, size=(4, 23, 9))
    a, cache = R.forward(x, p)
    b, _ = R.forward(x.astype(np.float32), {k: np.asarray(v, np.float32) for k, v in p.items()})
    assert np.abs(a - b).max() <= 1e-5 * np.abs(a).max()
    g = np.random.RandomState(2).normal(size=a.shape)
    dx1, g1 = R.backward(p, cache, g)
    dx2, g2 = R.backward(p, cache, 2 * g)
    assert np.allclose(2 * dx1, dx2, rtol=1e-12, atol=0) and all(np.allclose(2 * g1[k], g2[k], rtol=1e-12, atol=0) for k in R.KEYS)


def test_abi_argument_checks_without_device():
    from human_dynamics_b200 import _lib
    L = _lib.lib
    p = ctypes.c_void_p(16)            # never dereferenced: every call below fails its argument check first
    assert L.hd_dpose_workspace_bytes(0) == 0 and L.hd_dpose_workspace_bytes(-3) == 0
    ws = L.hd_dpose_workspace_bytes(65)
    assert ws == 2 * (23 * 1376 + 759 + 1025) * 4
    assert L.hd_dpose_trunk_forward(None, p, p, p, p, p, p, p, p, p, 4, None) == 1
    assert L.hd_dpose_trunk_forward(p, p, p, p, p, p, p, p, p, p, 0, None) == 1
    assert L.hd_dpose_out_forward(p, p, p, None, 4, None) == 1
    assert L.hd_dpose_out_forward(ctypes.c_void_p(20), p, p, p, 4, None) == 1          # unaligned h
    assert L.hd_dpose_trunk_backward(p, p, p, p, p, p, p, p, p, None, None, 0, 4, None) == 1        # neither dx nor ws
    assert L.hd_dpose_trunk_backward(p, p, p, p, p, p, p, p, p, None, p, ws - 4, 65, None) == 1     # workspace too small
    assert L.hd_dpose_trunk_backward(None, p, p, p, p, p, p, p, p, None, p, ws, 65, None) == 1      # ws without x
    assert L.hd_dpose_grad_reduce(p, ws - 4, 65, p, None) == 1
    assert L.hd_dpose_grad_reduce(p, ws, 65, None, None) == 1
    assert b'hd_dpose_grad_reduce' in L.hd_last_error()


def test_cpu_tensors_raise():
    from human_dynamics_b200._lib import HDError
    from human_dynamics_b200 import adversarial
    if torch.cuda.is_available():
        pytest.skip('the CPU-tensor refusal on a CUDA machine is covered by tests/test_gpu_dpose.py')
    with pytest.raises(HDError):
        adversarial.PoseDiscriminator(seed=0)
