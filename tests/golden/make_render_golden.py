"""Generates tests/golden/render_v1.npz by EXECUTING THE REFERENCE'S OWN src/util/render/nmr_renderer.py and torch_utils.py, unmodified,
from a checkout of the reference project, with `neural_renderer` (NMR, a torch-0.4 CUDA extension) replaced by a recording stub:

  * the stub's Renderer records what NMR is handed -- image_size, the vertices after projection and the y flip (VERT_IDS only),
    the faces, the texture colour and the light / background settings -- and returns seeded rgb in [-0.2, 1.2] and seeded alpha in
    {0, 1/4, 1/2, 3/4, 1}, so the recorded uint8 results pin the composite arithmetic (R8) exactly;
  * torch.Tensor.cuda is the identity (the generator needs no GPU) and numpy's removed `np.int` alias is set, as
    make_ref_exec_golden.py sets it.

That pins everything the reference authored around NMR: projection, flip, camera chain of visualize_img_orig (both above and below
max_img_size), make_square / remove_pads, the rotated() view, the rend_mask / alpha / img variants.  What NMR itself does with
those inputs (R3-R6 of oracle/render_ref.py) stays unpinned.

    HD_REFERENCE_ROOT=<reference checkout> python tests/golden/make_render_golden.py
"""
import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = os.environ.get('HD_REFERENCE_ROOT', '')
STUBS = os.path.join(ROOT, 'oracle', 'ref_exec', 'stubs')
VERT_IDS = np.arange(0, 6890, 53)
CAMS = np.array([[0.9, 0.0, 0.0], [1.1, 0.12, -0.08], [0.7, -0.2, 0.15]], np.float32)
# visualize_img_orig cases: (H, W, max_img_size, start_pt x, y, scale)
ORIG_CASES = [(90, 120, 100, 150, 140, 1.3), (60, 80, 100, 120, 110, 0.9)]


def stub_seed(call_index):
    return 1000 + call_index


def stub_outputs(call_index, kind, B, S):
    """What the stub returns for its call_index-th call: rgb [B,3,S,S] in [-0.2, 1.2] or alpha [B,S,S] in quarters (float32)."""
    rng = np.random.RandomState(stub_seed(call_index))
    if kind == 'rgb':
        return rng.uniform(-0.2, 1.2, size=(B, 3, S, S)).astype(np.float32)
    return (rng.randint(0, 5, size=(B, S, S)) / 4.0).astype(np.float32)


def _by_path(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class Recorder(object):
    def __init__(self):
        self.calls = []


REC = Recorder()


def make_nr_stub():
    import torch
    nr = types.ModuleType('neural_renderer')

    class Renderer(object):
        def __init__(self, image_size, camera_mode='look_at', perspective=True):
            self.image_size = image_size
            self.camera_mode, self.perspective = camera_mode, perspective

        def _record(self, kind, vertices, faces, textures=None):
            i = len(REC.calls)
            B = vertices.shape[0]
            rec = {'kind': kind, 'image_size': int(self.image_size), 'verts': vertices.detach().numpy()[:, VERT_IDS].copy(),
                   'faces_sum': int(faces.long().sum()), 'faces_shape': tuple(faces.shape),
                   'camera_mode': self.camera_mode, 'perspective': self.perspective,
                   'light': np.array(list(self.light_direction) + [self.light_intensity_directional, self.light_intensity_ambient]),
                   'bg': np.array(self.background_color, np.float64)}
            if textures is not None:
                t = textures.detach().numpy()
                assert np.all(t == t[:, :1, :1, :1, :1, :]), 'single-colour texture expected'
                rec['texture'] = t[:, 0, 0, 0, 0, :].copy()
            REC.calls.append(rec)
            return torch.from_numpy(stub_outputs(i, kind, B, int(self.image_size)))

        def render(self, vertices, faces, textures):
            return self._record('rgb', vertices, faces, textures)

        def render_silhouettes(self, vertices, faces):
            return self._record('alpha', vertices, faces)

    nr.Renderer = Renderer
    return nr


def setup_paths():
    if not os.path.isdir(os.path.join(REF, 'src', 'util', 'render')):
        raise SystemExit('reference tree not found at %s' % REF)
    for p in (ROOT, os.path.join(ROOT, 'tests'), ''):
        while p in sys.path:
            sys.path.remove(p)
    sys.path[:0] = [STUBS, REF]
    for m in [m for m in sys.modules if m == 'src' or m.startswith('src.')]:
        del sys.modules[m]
    if not hasattr(np, 'int'):
        np.int = int                                 # nmr_renderer.py:63 uses the alias numpy removed in 1.24; same type
    import torch
    torch.Tensor.cuda = lambda self, *a, **k: self
    sys.modules['neural_renderer'] = make_nr_stub()
    return _by_path('_hd_synthetic', os.path.join(ROOT, 'human_dynamics_b200', 'synthetic.py'))


def main():
    syn = setup_paths()
    from src.util.render import nmr_renderer as M
    out = {'vert_ids': VERT_IDS, 'cams': CAMS}
    smpl = syn.make_synthetic_smpl(seed=2)
    beta, theta = syn.make_smpl_inputs(3, seed=5)
    verts = (smpl['v_template'][None] + np.einsum('vkb,nb->nvk', smpl['shapedirs'], beta)).astype(np.float32)   # 3 meshes [3,V,3]
    out['verts'] = verts
    face_path = os.path.join(REF, 'src', 'tf_smpl', 'smpl_faces.npy')
    rng = np.random.RandomState(9)
    S = 32
    r = M.VisRenderer(img_size=S, face_path=face_path)
    cases = []

    def run(name, fn):
        n0 = len(REC.calls)
        res = fn()
        cases.append(name)
        if isinstance(res, tuple):
            for k, v in enumerate(res):
                out['%s_out%d' % (name, k)] = np.asarray(v)
        else:
            out[name + '_out'] = np.asarray(res)
        out[name + '_calls'] = np.arange(n0, len(REC.calls))

    img255 = rng.uniform(0, 255, size=(S, S, 3)).astype(np.float32)
    out['img255'] = img255
    for i, cam in enumerate(CAMS):
        run('cam%d' % i, lambda cam=cam: r(verts[0], cam=cam))
    run('default_cam', lambda: r(verts[0]))
    run('img', lambda: r(verts[1], cam=CAMS[1], img=img255))
    run('alpha', lambda: r(verts[1], cam=CAMS[1], alpha=True))
    run('mask', lambda: r(verts[1], cam=CAMS[1], rend_mask=True))
    run('batch_img', lambda: r(verts, cam=CAMS, img=np.stack([img255] * 3)))
    run('batch_mask', lambda: r(verts, cam=CAMS, rend_mask=True))
    run('rotated90', lambda: r.rotated(verts[2], 90, cam=CAMS[2]))
    run('rotated_x30', lambda: r.rotated(verts[2], 30, axis='x', cam=CAMS[0], color_name='pink'))
    kps = rng.uniform(-0.8, 0.8, size=(25, 2)).astype(np.float32)
    out['kps'] = kps
    for j, (H, W, mx, sx, sy, sc) in enumerate(ORIG_CASES):
        img = rng.uniform(-1, 1, size=(H, W, 3)).astype(np.float32)
        out['orig%d_img' % j] = img
        run('orig%d' % j, lambda img=img, mx=mx, sx=sx, sy=sy, sc=sc: M.visualize_img_orig(
            cam=CAMS[1], kp_pred=kps, vert=verts[1], renderer=r, start_pt=np.array([sx, sy]), scale=sc, proc_img_shape=[224, 224],
            img=img, rotated_view=True, max_img_size=mx, no_text=True))
        out['orig%d_case' % j] = np.array([H, W, mx, sx, sy, sc], np.float64)
    r.renderer.image_size = S
    out['cases'] = np.array(cases)
    for i, c in enumerate(REC.calls):
        for k, v in c.items():
            if isinstance(v, (str, bool)):
                v = np.array(str(v))
            out['call%d_%s' % (i, k)] = np.asarray(v)
    out['num_calls'] = np.array(len(REC.calls))
    path = os.path.join(ROOT, 'tests', 'golden', 'render_v1.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes,', len(out), 'arrays,', len(REC.calls), 'stub calls')


if __name__ == '__main__':
    main()
