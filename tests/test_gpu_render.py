"""GPU: hd_render_mesh (csrc/render.cu) against the float64 restatement of R1-R8 (oracle/render_ref.py), its determinism, and the
Python surfaces on top of it (MeshRenderer, the VisRenderer drop-in, run_video.render_overlays).

Two meshes: the real SMPL face table over the synthetic capsule vertices (faces join random points: huge, overlapping triangles)
and a seeded smooth closed surface with SMPL's V = 6890 and F = 13776 (synthetic.make_smooth_mesh: realistic coverage, small
triangles, one layer per side).
Agreement is judged per sample: the same face id for >= 99.9 % of samples, and every disagreement explained by float32 vs
float64 at a face edge (barycentric margin < 1e-5) or a depth near-tie."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import render_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FACES = np.load(os.path.join(ROOT, 'src', 'tf_smpl', 'smpl_faces.npy')).astype(np.int64)
EDGE, TIE = 1e-5, 1e-5


def meshes(name, N, seed=0):
    """N frames of one mesh: per-frame seeded rotation about y and a small jitter; cams around the demo's [0.9, 0, 0]."""
    rng = np.random.RandomState(seed)
    if name == 'capsule':
        from human_dynamics_b200 import synthetic
        base = synthetic.make_synthetic_smpl(seed=2)['v_template'].astype(np.float32)
        faces = FACES
    else:
        from human_dynamics_b200 import synthetic
        base, faces = synthetic.make_smooth_mesh(seed=11)
    V = []
    for i in range(N):
        a = rng.uniform(-0.6, 0.6)
        Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        V.append(base @ Ry.T + rng.normal(0, 0.002, size=base.shape))
    cams = np.stack([rng.uniform(0.8, 1.1, N), rng.uniform(-0.1, 0.1, N), rng.uniform(-0.1, 0.1, N)], 1)
    return np.stack(V).astype(np.float32), cams.astype(np.float32), faces


def gpu_render(verts, cams, faces, S, background=None, rot=None, color='blue'):
    """hd_render_mesh through the C-ABI with a caller-owned workspace -> (rgb uint8, alpha, face id per sample (-1 empty))."""
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.render import make_params
    v = verts if isinstance(verts, torch.Tensor) else torch.from_numpy(verts).cuda()
    c = cams if isinstance(cams, torch.Tensor) else torch.from_numpy(cams).cuda()
    f = torch.from_numpy(np.ascontiguousarray(faces, np.int32)).cuda()
    N, Vn = v.shape[0], v.shape[1]
    ws = torch.empty(int(_lib.lib.hd_render_workspace_bytes(N, S, f.shape[0])), dtype=torch.uint8, device='cuda')
    out = torch.empty((N, S, S, 3), dtype=torch.uint8, device='cuda')
    alpha = torch.empty((N, S, S), dtype=torch.float32, device='cuda')
    bg = None if background is None else (background if isinstance(background, torch.Tensor) else torch.from_numpy(background).cuda())
    p = make_params(color, rot=rot)
    _lib.check(_lib.lib.hd_render_mesh(C.c_void_p(v.data_ptr()), v.stride(0), N, Vn, C.c_void_p(f.data_ptr()), f.shape[0],
                                       C.c_void_p(c.data_ptr()), c.stride(0), C.byref(p), None if bg is None else C.c_void_p(bg.data_ptr()),
                                       S, C.c_void_p(out.data_ptr()), C.c_void_p(alpha.data_ptr()), C.c_void_p(ws.data_ptr()),
                                       ws.numel(), _lib.current_stream()), 'hd_render_mesh')
    keys = ws[:N * 4 * S * S * 8].view(torch.int64).view(N, 2 * S, 2 * S).cpu().numpy()
    fid = np.where(keys == -1, -1, keys & 0xffffffff)
    return out.cpu().numpy(), alpha.cpu().numpy(), fid


def check_frame(g_rgb, g_alpha, g_fid, verts, cam, faces, S, background=None, rot=None):
    """One frame against the oracle: face-id agreement with every disagreement explained; alpha / RGB where ids agree."""
    ref = R.rasterize(verts, cam, faces, S, rot=rot)
    o_fid = ref['face']
    same = g_fid == o_fid
    assert same.mean() >= 0.999, same.mean()
    vv = R.rotate_about_mean(verts, rot) if rot is not None else verts
    for r, c in np.argwhere(~same):
        g, o = int(g_fid[r, c]), int(o_fid[r, c])
        mg, dg = R.face_at(vv, cam, faces, g, r, c, S) if g >= 0 else (None, None)
        mo, do = R.face_at(vv, cam, faces, o, r, c, S) if o >= 0 else (None, None)
        at_edge = (mg is not None and abs(mg) < EDGE) or (mo is not None and abs(mo) < EDGE)
        near_tie = mg is not None and mo is not None and mg > -EDGE and abs(dg - do) <= TIE * abs(do)
        assert at_edge or near_tie, ('unexplained disagreement', r, c, g, o, mg, mo, dg, do)
    pix_same = same.reshape(S, 2, S, 2).all(axis=(1, 3))
    assert np.array_equal(g_alpha[pix_same], ref['alpha'][pix_same])
    want = R.composite(ref['rgb'], ref['alpha'], background)
    d = np.abs(g_rgb.astype(np.int32) - want.astype(np.int32))
    assert d[pix_same].max() <= 1, d[pix_same].max()
    return same.mean()


@pytest.mark.parametrize('mesh', ['capsule', 'smooth'])
def test_s224_matches_oracle_with_and_without_background(mesh):
    verts, cams, faces = meshes(mesh, 3, seed=1)
    bg = np.random.RandomState(4).uniform(-1, 1, size=(3, 224, 224, 3)).astype(np.float32)
    rgb, alpha, fid = gpu_render(verts, cams, faces, 224)
    rgb_b, alpha_b, fid_b = gpu_render(verts, cams, faces, 224, background=bg)
    assert np.array_equal(fid, fid_b) and np.array_equal(alpha, alpha_b)
    assert set(np.unique(alpha).tolist()) <= {0.0, 0.25, 0.5, 0.75, 1.0}
    for i in (0, 2):
        check_frame(rgb[i], alpha[i], fid[i], verts[i], cams[i], faces, 224)
        check_frame(rgb_b[i], alpha_b[i], fid_b[i], verts[i], cams[i], faces, 224, background=bg[i])


@pytest.mark.parametrize('mesh', ['capsule', 'smooth'])
def test_rotated_view_matches_oracle(mesh):
    from human_dynamics_b200.render import rotation
    verts, cams, faces = meshes(mesh, 2, seed=2)
    rot = rotation(90, 'y')
    rgb, alpha, fid = gpu_render(verts, cams, faces, 224, rot=rot)
    check_frame(rgb[1], alpha[1], fid[1], verts[1], cams[1], faces, 224, rot=rot)


@pytest.mark.parametrize('mesh', ['capsule', 'smooth'])
def test_s720_matches_oracle(mesh):
    verts, cams, faces = meshes(mesh, 1, seed=3)
    bg = np.random.RandomState(5).uniform(-1, 1, size=(1, 720, 720, 3)).astype(np.float32)
    rgb, alpha, fid = gpu_render(verts, cams, faces, 720, background=bg)
    check_frame(rgb[0], alpha[0], fid[0], verts[0], cams[0], faces, 720, background=bg[0])


def test_bit_identity_launches_batches_and_strided_views():
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.render import MeshRenderer
    verts, cams, faces = meshes('smooth', 640, seed=6)
    mr = MeshRenderer(faces)
    v, c = torch.from_numpy(verts).cuda(), torch.from_numpy(cams).cuda()
    a = mr.render(v, c, 224).cpu().numpy()
    b = mr.render(v, c, 224).cpu().numpy()
    assert np.array_equal(a, b)
    for i in (0, 317, 639):
        assert np.array_equal(mr.render(v[i:i + 1], c[i:i + 1], 224).cpu().numpy()[0], a[i]), i
    mr.max_workspace_bytes = 100 * int(_lib.lib.hd_render_workspace_bytes(1, 224, len(faces)))
    assert np.array_equal(mr.render(v, c, 224).cpu().numpy(), a)                         # 100-frame chunks
    # a verts_delta-like [B, T, D, V, 3] buffer read in place through a strided view, cams from omegas_delta[..., :3]
    B, T, D = 32, 20, 2
    vd = torch.zeros((B, T, D, v.shape[1], 3), device='cuda')
    od = torch.zeros((B, T, D, 85), device='cuda')
    vd[:, :, 1] = v.view(B, T, -1, 3)
    od[:, :, 1, :3] = c.view(B, T, 3)
    vs = vd[:, :, 1].reshape(B * T, -1, 3)
    cs = od[:, :, 1, :3].reshape(B * T, 3)
    assert vs.stride(0) == D * v.shape[1] * 3 and cs.stride(0) == D * 85
    assert np.array_equal(mr.render(vs, cs, 224).cpu().numpy(), a)


def test_out_of_range_faces_are_skipped():
    verts, cams, faces = meshes('smooth', 1, seed=7)
    bad = faces.copy()
    bad[5] = [0, 1, len(verts[0]) + 5]
    bad[900] = [-1, 2, 3]
    bad[13775] = [7, 2 ** 31 - 1, 8]
    rgb, alpha, fid = gpu_render(verts, cams, bad, 224)
    assert not np.isin(fid, [5, 900, 13775]).any()
    check_frame(rgb[0], alpha[0], fid[0], verts[0], cams[0], bad, 224)
    keep = np.setdiff1d(np.arange(len(faces)), [5, 900, 13775])
    rgb2, alpha2, _ = gpu_render(verts, cams, faces[keep], 224)
    assert np.array_equal(alpha, alpha2) and np.abs(rgb.astype(int) - rgb2.astype(int)).max() <= 1


def test_bad_arguments_and_cpu_tensors():
    from human_dynamics_b200 import _lib
    from human_dynamics_b200.render import MeshRenderer, make_params
    verts, cams, faces = meshes('smooth', 2, seed=8)
    v, c = torch.from_numpy(verts).cuda(), torch.from_numpy(cams).cuda()
    f = torch.from_numpy(faces.astype(np.int32)).cuda()
    out = torch.empty((2, 64, 64, 3), dtype=torch.uint8, device='cuda')
    need = int(_lib.lib.hd_render_workspace_bytes(2, 64, len(faces)))
    ws = torch.empty(need, dtype=torch.uint8, device='cuda')
    p = make_params()
    call = lambda S=64, n=2, wsb=need, cam_ld=3: _lib.lib.hd_render_mesh(
        C.c_void_p(v.data_ptr()), v.stride(0), n, v.shape[1], C.c_void_p(f.data_ptr()), len(faces), C.c_void_p(c.data_ptr()), cam_ld,
        C.byref(p), None, S, C.c_void_p(out.data_ptr()), None, C.c_void_p(ws.data_ptr()), wsb, _lib.current_stream())
    assert call(wsb=need - 1) == 2
    assert call(S=0) == 1 and call(S=4096) == 1 and call(cam_ld=2) == 1
    assert call() == 0
    torch.cuda.synchronize()
    mr = MeshRenderer(faces)
    with pytest.raises(_lib.HDError):
        mr.render(torch.from_numpy(verts), torch.from_numpy(cams), 64)
    with pytest.raises(_lib.HDError):
        MeshRenderer(np.zeros((0, 3), np.int64))


def test_visrenderer_shapes_and_dtypes():
    """The drop-in returns what the reference's VisRenderer returns (nmr_renderer.py:81-225)."""
    from src.util.render.nmr_renderer import VisRenderer
    from human_dynamics_b200 import synthetic
    smpl = synthetic.make_synthetic_smpl(seed=2)
    v1 = smpl['v_template'].astype(np.float32)
    vb = np.stack([v1, v1 * 0.9, v1 * 1.1])
    cam = np.array([0.9, 0.05, -0.05], np.float32)
    r = VisRenderer(img_size=96)
    single = r(v1, cam=cam)
    assert single.shape == (96, 96, 3) and single.dtype == np.uint8
    batch = r(vb, cam=np.tile(cam, (3, 1)))
    assert batch.shape == (3, 96, 96, 3) and batch.dtype == np.uint8
    assert np.array_equal(batch[0], single)
    assert r(v1, cam=cam, rend_mask=True).shape == (96, 96, 3)
    assert r(vb, cam=np.tile(cam, (3, 1)), rend_mask=True).shape == (1, 96, 96, 9)
    rgba = r(v1, cam=cam, alpha=True)
    assert rgba.shape == (96, 96, 4) and rgba.dtype == np.uint8 and set(np.unique(rgba[..., 3])) <= {0, 63, 127, 191, 255}
    img = np.random.RandomState(0).uniform(0, 255, size=(96, 96, 3))
    comp = r(v1, cam=cam, img=img)
    assert comp.shape == (96, 96, 3) and comp.dtype == np.uint8
    empty = rgba[..., 3] == 0
    assert np.array_equal(comp[empty], img[empty].astype(np.uint8))
    assert r(vb, cam=np.tile(cam, (3, 1)), img=np.stack([img] * 3)).shape == (3, 96, 96, 3)
    rot = r.rotated(v1, 90, cam=cam)
    assert rot.shape == (96, 96, 3) and rot.dtype == np.uint8 and not np.array_equal(rot, single)
    r.renderer.image_size = 64                                                        # visualize_img_orig assigns it
    assert r(v1, cam=cam).shape == (64, 64, 3)
    with pytest.raises(NotImplementedError):
        r(v1, cam=cam, texture=np.ones((1, 13776, 1, 1, 1, 3)))


def test_render_overlays_on_a_tester_run(weights, smpl_model):
    """render_overlays on a synthetic Tester run: the crop and frame overlays against the oracle on the first and last frame; the
    frame background against the host resize_img path, both with a resize (frame larger than max_img_size) and at scale 1."""
    pytest.importorskip('cv2')
    from human_dynamics_b200 import HMMRConfig, _lib
    from src.evaluation.run_video import process_video_frames, render_overlays
    from src.evaluation.tester import Tester
    from src.util.render.nmr_renderer import orig_frame_cam, orig_frame_size
    from human_dynamics_b200.render import rotation
    from oracle import preproc_ref
    N, H, W = 6, 150, 200
    rng = np.random.RandomState(3)
    yy, xx = np.mgrid[0:H, 0:W]
    frames = np.stack([np.clip((120 + 90 * np.sin(xx / (5.0 + i) + i) * np.cos(yy / 6.0))[..., None] + rng.randint(-30, 30, size=(H, W, 3)),
                               0, 255) for i in range(N)]).astype(np.uint8)
    boxes = np.stack([rng.uniform(80, 120, N), rng.uniform(60, 90, N), rng.uniform(0.9, 1.3, N)], axis=1)
    crops, infos = process_video_frames(frames, boxes)
    tester = Tester(HMMRConfig(batch_size=1, sequence_length=20, weights=weights, smpl_model=smpl_model))
    preds = tester.predict_all_images(crops.cpu().numpy())
    faces = FACES
    for max_img_size in (160, 720):                     # 160: resized by 0.8; 720: scale 1
        out = render_overlays(preds, crops, infos, frames=frames, max_img_size=max_img_size)
        scale_orig, Hs, Ws, S = orig_frame_size(H, W, max_img_size)
        assert out['crop'].shape == (N, 224, 224, 3) and out['frame'].shape == (N, Hs, Ws, 3) == out['frame_rotated'].shape
        geom = torch.tensor([[Hs, Ws, 0, 0]] * N, dtype=torch.int32, device='cuda')
        bg = torch.empty((N, S, S, 3), dtype=torch.float32, device='cuda')
        fr = torch.from_numpy(frames).cuda()
        _lib.check(_lib.lib.hd_process_image(C.c_void_p(fr.data_ptr()), N, H, W, C.c_void_p(geom.data_ptr()), C.c_void_p(bg.data_ptr()),
                                             S, None, None, 0, _lib.current_stream()), 'hd_process_image')
        bg = bg.cpu().numpy()
        for i in (0, N - 1):
            host = ((frames[i] / 255.) - 0.5) * 2
            if scale_orig is not None:
                host, _ = preproc_ref.resize_img(host, scale_orig)
            assert host.shape[:2] == (Hs, Ws)
            assert np.abs(bg[i, :Hs, :Ws] - host).max() < 2e-6
            cam_o = orig_frame_cam(preds['cams'][i], np.asarray(infos[i]['start_pt']), infos[i]['scale'], infos[i]['im_shape'], S, scale_orig)
            for key, cam, size, back, rot in (('crop', preds['cams'][i], 224, crops[i].cpu().numpy(), None),
                                              ('frame', cam_o, S, bg[i], None),
                                              ('frame_rotated', cam_o, S, None, rotation(90))):
                ref = R.rasterize(preds['verts'][i], cam, faces, size, rot=rot)
                want = R.composite(ref['rgb'], ref['alpha'], back)
                got = out[key][i].cpu().numpy()
                if key != 'crop':
                    want = want[:Hs, :Ws]
                close = np.abs(got.astype(int) - want.astype(int)).max(axis=-1) <= 1
                assert close.mean() >= 0.995, (key, max_img_size, i, close.mean())
