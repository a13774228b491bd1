"""CPU: the IEF dropout masks' host restatement (oracle/dropout_ref.py) -- Philox4x32-10's known-answer vectors, the keep decision over
every uniform TF can draw -- and the masked float64 oracles against tests/golden/ief_dropout_v1.npz, made by running the reference's
own batch_pred_omega(is_training=True) over the TensorFlow stand-in with these masks (tests/golden/make_ief_dropout_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import dropout_ref as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'ief_dropout_v1.npz')

KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize('ctr,key,want', KAT)
def test_philox_known_answers(ctr, key, want):
    got = D.philox4x32_10([np.uint64(c) for c in ctr], key)
    assert [int(x) for x in got] == list(want)


def test_words_follow_the_counter_layout():
    """Element w of a site is word w & 3 of the call at counter (w >> 2, site, step lo, step hi), key (seed lo, seed hi)."""
    seed, step, site, N, C = 0x123456789abcdef0, (5 << 32) + 17, 37, 3, 7
    w = D.words(seed, step, site, N, C).reshape(-1)
    for e in (0, 5, 11, 20):
        ref = D.philox4x32_10([np.uint64(e >> 2), np.uint64(site), np.uint64(17), np.uint64(5)], (0x9abcdef0, 0x12345678))
        assert int(w[e]) == int(ref[e & 3])


@pytest.mark.parametrize('p', [0.5, 0.7, 0.9])
def test_keep_decision_over_every_uniform(p):
    """All 2^23 uniforms: the device's predicate fp32(p + u) >= 1 is nn.dropout's floor(p + u) in float32; at p = 0.5 it is bit 22."""
    low = np.arange(1 << 23, dtype=np.uint64)
    u = D.uniform(low)
    assert u.dtype == np.float32 and u.min() == 0 and u.max() < 1
    assert np.array_equal(np.unique(u), u)                                 # one uniform per 23-bit value
    p32 = D.nn_keep_prob(p)
    floor = D.keep_from_uniform(u, p32)
    device = ((u + p32) >= np.float32(1)).astype(np.float32)
    assert np.array_equal(floor, device)
    assert abs(floor.mean() - p) < 1e-6
    if p == 0.5:
        assert np.array_equal(floor, ((low >> np.uint64(22)) & np.uint64(1)).astype(np.float32))
        x = np.random.RandomState(0).normal(0, 1, 1000).astype(np.float32)
        assert np.array_equal(D.apply(x, np.ones(1000), p32), 2 * x)     # x / 0.5 is exact


def test_nn_keep_prob_rounding():
    """slim.dropout(keep_prob) reaches nn.dropout as float32(1 - (1 - keep_prob)) worked out in float64."""
    for p in (0.5, 0.7, 0.9, 0.3, 0.1, 1.0):
        assert D.nn_keep_prob(p) == np.float32(1.0 - (1.0 - p))
    assert D.nn_keep_prob(0.5) == np.float32(0.5)
    assert D.nn_keep_prob(3e-10) != np.float32(3e-10)        # where float64's 1 - (1 - p) loses bits of p, float32 sees them


def test_sites_are_distinct():
    sites = {D.site(c, h, s, l) for c in (0, 1) for h in range(8) for s in range(4) for l in (0, 1)}
    assert len(sites) == 2 * 8 * 4 * 2 and min(sites) == 0


@pytest.fixture(scope='module')
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope='module')
def gweights():
    from human_dynamics_b200 import synthetic
    return synthetic.make_synthetic_weights(seed=1)


def case_masks(golden, name):
    """The masks the golden case was made with: {dt: [(dropout1, dropout2) per stage]}, head 0 = main, then ascending dt."""
    keys = [int(k) for k in golden['keys']]
    N = int(golden['B']) * int(golden['T'])
    m = D.ief_masks(int(golden['seed']), int(golden['%s_step' % name]), int(golden['%s_call' % name]), N, 1 + len(keys),
                    D.nn_keep_prob(float(golden['keep_prob'])))
    return {dt: [(m[(h, s, 0)], m[(h, s, 1)]) for s in range(3)] for h, dt in enumerate([0] + sorted(keys))}, m


@pytest.mark.parametrize('name', ['pred', 'hal'])
def test_standin_saw_every_dropout(golden, name):
    """2 layers x 3 stages x (1 + |dt|) heads per IEF call, in the reference's order: main, then the delta heads as listed."""
    ops = [str(o) for o in golden['%s_dropout_ops' % name]]
    keys = [int(k) for k in golden['keys']]
    assert len(ops) == 2 * 3 * (1 + len(keys))
    scopes = ['single_view_ief'] + ['single_view_ief' + ('_future%d' % k if k > 0 else '_past%d' % -k) for k in keys]
    assert ops == ['%s/3D_module/dropout%d' % (sc, l) for sc in scopes for _ in range(3) for l in (1, 2)]


@pytest.mark.parametrize('name', ['pred', 'hal'])
def test_masked_oracle_equals_reference(golden, gweights, name):
    from oracle import ief_dropout_ref, nets_ref
    masks, _ = case_masks(golden, name)
    B, T = int(golden['B']), int(golden['T'])
    keys = [int(k) for k in golden['keys']]
    p = float(D.nn_keep_prob(float(golden['keep_prob'])))
    start = np.tile(np.asarray(gweights['mean_param'], np.float32).reshape(1, 85), (B * T, 1))
    om, dl = ief_dropout_ref.batch_pred_omega(golden['%s_feats' % name], B, gweights, start, T, keys, masks, p)
    ref = golden['%s_omega' % name]
    assert np.abs(om.numpy() - ref).max() / np.abs(ref).max() <= 1e-5
    for k in keys:
        ref = golden['%s_delta_%d' % (name, k)]
        assert np.abs(dl[k].numpy() - ref).max() / np.abs(ref).max() <= 1e-5, k
    # the inference graph is far from it: the golden is not the identity
    om0, _ = nets_ref.batch_pred_omega(golden['%s_feats' % name], B, gweights, 85, start, T, 'single_view_ief', keys, True, True,
                                       torch.float64)
    assert np.abs(om0.numpy() - golden['%s_omega' % name]).max() > 1e-2


def test_grad_oracle_with_masks_and_its_gradcheck():
    """oracle/ief_dropout_ref's differentiable hmr_ief with explicit dropout masks: its gradients pass gradcheck (small widths: it is
    shape-generic), and an all-kept mask at keep_prob 1 is nets_grad_ref's inference graph."""
    from oracle import ief_dropout_ref as R, nets_grad_ref as g
    rng = np.random.RandomState(3)
    N, F, H, d = 3, 6, 5, 4
    t = lambda *s: torch.tensor(rng.normal(0, 0.7, s), dtype=torch.float64, requires_grad=True)   # noqa: E731
    phi, start = t(N, F), t(N, d)
    p = (t(F + d, H), t(H), t(H, H), t(H), t(H, d), t(d))
    keep = {'x.s%d.fc%d' % (s, l): torch.tensor(rng.rand(N, H) < 0.6) for s in range(3) for l in (1, 2)}
    drop = (keep, 0.7)
    assert torch.autograd.gradcheck(lambda *a: R.grad_hmr_ief(a[0], a[1], a[2:], 'x', drop), (phi, start) + p)
    ones = ({k: torch.ones_like(v) for k, v in keep.items()}, 1.0)
    assert torch.equal(R.grad_hmr_ief(phi, start, p, 'x', ones), g.hmr_ief(phi, start, p, 'x'))


def test_standin_dropout_raises_without_a_provider():
    """The stand-in's nn / contrib.layers / slim dropout: training mode raises until oracle/ref_exec/training_dropout installs a
    provider, and again after uninstall; is_training=False stays the identity."""
    import subprocess
    import sys
    code = ('import sys; sys.path.insert(0, %r); sys.path.insert(1, %r)\n'
            'import numpy as np, tensorflow as tf\n'
            'from tensorflow.contrib import layers, slim\n'
            'from oracle.ref_exec import training_dropout\n'
            'x = tf.constant(np.ones((2, 8), np.float32))\n'
            'def raises():\n'
            '    for f in (layers.dropout, slim.dropout):\n'
            '        assert f(x, 0.5, is_training=False) is x\n'
            '        try:\n            f(x, 0.5, is_training=True)\n            raise SystemExit(1)\n        except NotImplementedError:\n            pass\n'
            'raises()\n'
            'paths = []\n'
            'training_dropout.install(lambda path: paths.append(path) or (lambda shape: np.full(shape, 0.5, np.float32)))\n'
            'with tf.variable_scope("a"):\n    y = slim.dropout(x, 0.7, is_training=True, scope="dropout1")\n'
            'assert layers.dropout(x, 0.5, is_training=False) is x\n'
            'assert paths == ["a/dropout1"]\n'
            'assert np.array_equal(tf.Session().run(y), np.full((2, 8), np.float32(1) / np.float32(0.7), np.float32))\n'
            'training_dropout.uninstall()\n'
            'raises()\n'
            % (os.path.join(ROOT, 'oracle', 'ref_exec', 'stubs'), ROOT))
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
