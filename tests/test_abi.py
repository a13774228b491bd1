"""CPU: the C-ABI library loads and exports every symbol include/hd_b200.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, 'include', 'hd_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(hd_[a-z0-9_]+)\s*\(', src)))


def test_header_symbols_exported_and_bound():
    from human_dynamics_b200 import _lib
    names = _declared()
    assert len(names) >= 15
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), 'libhd_b200.so does not export %s' % n
        assert n in _lib.SIGNATURES, 'ctypes binding missing for %s' % n
    assert sorted(_lib.SIGNATURES) == names, 'binding table and header disagree'
    assert _lib.lib.hd_version() >= 100
    assert _lib.lib.hd_status_string(0) == b'ok' and _lib.lib.hd_status_string(4).startswith(b'unsupported')


def test_struct_layouts_match_header_sizes():
    """hd_conv_desc / hd_smpl_consts mirrors: field counts and natural-alignment sizes."""
    from human_dynamics_b200 import _lib
    assert ctypes.sizeof(_lib.ConvDesc) == 344
    assert ctypes.sizeof(_lib.SmplConsts) == 16 + 9 * 8 + 24 * 4
    assert _lib.ConvDesc.in_ld.offset == 8 and _lib.ConvDesc.w_kn.offset == 64 and _lib.ConvDesc.out.offset == 176


def test_no_cpu_fallback_paths():
    """Product code must not import the oracle, and ops must refuse CPU tensors."""
    import torch
    import pytest
    for sub in ('human_dynamics_b200', 'src'):
        for dp, _, files in os.walk(os.path.join(ROOT, sub)):
            for f in files:
                if f.endswith('.py'):
                    txt = open(os.path.join(dp, f)).read()
                    assert not re.search(r'^\s*(from|import)\s+oracle', txt, flags=re.M), '%s imports the oracle' % f
    from src.tf_smpl.batch_lbs import batch_rodrigues
    from src.tf_smpl.projection import batch_orth_proj_idrot
    from human_dynamics_b200._lib import HDError
    with pytest.raises(HDError):
        batch_rodrigues(torch.zeros(4, 3))
    with pytest.raises(HDError):
        batch_orth_proj_idrot(torch.zeros(2, 5, 3), torch.zeros(2, 3))
    if not torch.cuda.is_available():
        from human_dynamics_b200.engine import HMMREngine
        with pytest.raises(HDError):
            HMMREngine({}, {})


def test_invalid_arguments_return_status_not_crash():
    from human_dynamics_b200 import _lib
    d = _lib.ConvDesc()
    assert _lib.lib.hd_conv_gemm(ctypes.byref(d), None) == 1           # HD_ERR_INVALID: null in/out
    assert b'null' in _lib.lib.hd_last_error()
    assert _lib.lib.hd_rodrigues(None, None, 4, None) == 1
    assert _lib.lib.hd_smpl_workspace_bytes(10) >= 10 * 24 * 21 * 4


def test_conv_desc_matches_compiled_struct():
    """Compile a one-liner against include/hd_b200.h with gcc and compare sizeof/offsetof with the ctypes mirror."""
    import subprocess, tempfile, shutil
    from human_dynamics_b200 import _lib
    if shutil.which('gcc') is None:
        import pytest
        pytest.skip('gcc not available')
    fields = ['in_ld', 'w_kn', 'Cout', 'pre_scale', 'post_relu', 'res', 'out', 'impl', 'tmap_hi', 'in_hi', 'out_hi', 'out2_ld',
              'post2_relu', 'tmap_res', 'tmap_out_lo', 'flags', 'tmap_lo_n64', 'out_subsample']
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "hd_b200.h"\nint main(){printf("%zu %zu", sizeof(hd_conv_desc), sizeof(hd_smpl_consts));\n'
    src += ''.join('printf(" %%zu", offsetof(hd_conv_desc, %s));\n' % f for f in fields) + 'return 0;}\n'
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, 't.c'); exe = os.path.join(td, 't')
        open(c, 'w').write(src)
        subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe])
        out = [int(x) for x in subprocess.check_output([exe]).split()]
    assert out[0] == ctypes.sizeof(_lib.ConvDesc) and out[1] == ctypes.sizeof(_lib.SmplConsts)
    for f, off in zip(fields, out[2:]):
        assert getattr(_lib.ConvDesc, f).offset == off, f


def test_host_logic_without_gpu():
    """Pure host logic of the plan / driver layer (no device needed)."""
    import types
    import pytest
    from human_dynamics_b200.engine import HMMREngine
    from human_dynamics_b200 import HMMRConfig
    fake = types.SimpleNamespace(config=HMMRConfig(frame_chunk=160), H2D_PIECE=HMMREngine.H2D_PIECE)
    sched = HMMREngine.stage_a_schedule(fake, 640, True)            # streaming from the host: small first pass
    assert sched[0] == (0, 32) and sum(n for _, n in sched) == 640 and all(n <= 160 for _, n in sched)
    assert [s for s, _ in sched] == [0] + [32 + 160 * i for i in range(4)]
    assert HMMREngine.stage_a_schedule(fake, 640, False) == [(0, 160), (160, 160), (320, 160), (480, 160)]
    assert HMMREngine.stage_a_schedule(fake, 20, True) == [(0, 20)]
    # Tester refuses to start without weights, like the reference (tester.py:31-38), but without ipdb
    from src.evaluation.tester import Tester
    with pytest.raises(Exception):
        Tester(HMMRConfig(load_path=''))
    with pytest.raises(Exception):
        Tester(HMMRConfig(load_path='/nonexistent/model.npz'))
    # TF-style SAME / conv2d_same output sizes used by the plans
    from oracle.pack_ref import f16_split, tf32_split
    import numpy as np
    w = np.random.RandomState(0).normal(0, 0.05, size=(7, 5)).astype(np.float32)
    hi, lo = f16_split(w)
    assert np.abs(hi.astype(np.float64) + lo.astype(np.float64) / 2048.0 - w).max() < 2.0 ** -22 * np.abs(w).max() * 2
    th, tl = tf32_split(w)
    assert np.all((th.view(np.uint32) & 0x1FFF) == 0) and np.all((tl.view(np.uint32) & 0x1FFF) == 0)
    assert np.abs(th.astype(np.float64) + tl.astype(np.float64) - w).max() < 2.0 ** -21 * np.abs(w).max()

def test_plain_c_consumer(tmp_path):
    """tests/c/consumer.c: gcc -std=c99 against include/hd_b200.h, dlopen of the shipped library, a network-level create call whose
    weight callback has nothing to offer -> HD_ERR_INVALID naming the first variable it asked for (no device touched)."""
    import shutil
    import subprocess
    from human_dynamics_b200 import _lib
    if shutil.which('gcc') is None:
        pytest.skip('gcc not available')
    exe = str(tmp_path / 'consumer')
    subprocess.check_call(['gcc', '-std=c99', '-Wall', '-Werror', '-D_DEFAULT_SOURCE', '-I', os.path.join(ROOT, 'include'),
                           os.path.join(ROOT, 'tests', 'c', 'consumer.c'), '-o', exe, '-ldl'])
    r = subprocess.run([exe, _lib.LIB_PATH], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    assert r.returncode == 0, r.stdout
    assert 'rc=1' in r.stdout and 'resnet_v2_50/conv1/weights' in r.stdout and 'asked=1' in r.stdout
    from human_dynamics_b200.preprocess import crop_geometry
    g = crop_geometry((240, 320), [40.3, 200.7, 0.62])
    want = 'geom rc=0 %d %d %d %d center=%d,%d start=%d,%d' % (g['new_size'][0], g['new_size'][1], g['origin'][0], g['origin'][1],
                                                             g['center'][0], g['center'][1], g['start_pt'][0], g['start_pt'][1])
    assert want in r.stdout, (want, r.stdout)
