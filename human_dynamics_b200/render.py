"""GPU mesh rendering: the visualiser of the reference's demo (src/util/render/nmr_renderer.py, NMR with an orthographic look_at
camera) as one C-ABI call, hd_render_mesh (csrc/render.cu; model R1-R8 in oracle/render_ref.py).

`MeshRenderer(faces).render(verts, cams, S)` draws a batch of meshes, one colour each, and returns uint8 [N,S,S,3] on the GPU,
optionally over a [-1, 1] background image (the crops `process_image` produces) and optionally rotated about each frame's vertex
mean (the 90-degree side view).  Frames are processed in chunks whose workspace stays under `max_workspace_bytes`; every frame is
rendered independently, so the result does not depend on the chunking.  There is no CPU path: CPU tensors raise HDError.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import lib, check, current_stream

COLORS = {
    # nmr_renderer.py:25-36
    'blue': [0.65098039, 0.74117647, 0.85882353],
    'pink': [.9, .7, .7],
    'mint': [166 / 255., 229 / 255., 204 / 255.],
    'mint2': [202 / 255., 229 / 255., 223 / 255.],
    'green': [153 / 255., 216 / 255., 201 / 255.],
    'green2': [171 / 255., 221 / 255., 164 / 255.],
    'red': [251 / 255., 128 / 255., 114 / 255.],
    'orange': [253 / 255., 174 / 255., 97 / 255.],
    'yellow': [250 / 255., 230 / 255., 154 / 255.],
}
# VisRenderer.__init__ (nmr_renderer.py:59): set_light_dir([1, .5, -1], int_dir=0.3, int_amb=0.7)
DEFAULT_LIGHT = ((1.0, 0.5, -1.0), 0.3, 0.7)
# NMR defaults: eye at [0, 0, -(1/tan 30deg + 1)], near 0.1, far 100
EYE_Z = -(1.0 / np.tan(np.radians(30.0)) + 1.0)
NEAR, FAR = 0.1, 100.0


def make_params(color='blue', light=DEFAULT_LIGHT, bg_color=(1.0, 1.0, 1.0), rot=None):
    """hd_render_params from a colour (name in COLORS or an RGB triple), light = (direction, int_dir, int_amb), background colour
    and an optional 3x3 rotation about the vertex mean."""
    p = _lib.RenderParams()
    rgb = COLORS[color] if isinstance(color, str) else color
    direction, int_dir, int_amb = light
    p.color[:] = [float(c) for c in rgb]
    p.light_dir[:] = [float(c) for c in direction]
    p.directional, p.ambient = float(int_dir), float(int_amb)
    p.bg[:] = [float(c) for c in bg_color]
    p.near_z, p.far_z, p.eye_z = NEAR, FAR, EYE_Z
    if rot is not None:
        p.rot[:] = [float(x) for x in np.asarray(rot, np.float32).reshape(9)]
        p.use_rot = 1
    return p


class MeshRenderer:
    """Renders batches of one mesh topology.  faces: [F,3] integer array or tensor (uploaded once as int32)."""

    max_workspace_bytes = 2 << 30

    def __init__(self, faces, device=None):
        f = faces.detach().cpu().numpy() if isinstance(faces, torch.Tensor) else np.asarray(faces)
        f = np.squeeze(f, 0) if f.ndim == 3 and f.shape[0] == 1 else f
        if f.ndim != 2 or f.shape[1] != 3 or f.shape[0] == 0 or not np.issubdtype(f.dtype, np.integer):
            raise _lib.HDError('MeshRenderer: faces must be a non-empty integer [F,3] array, got %s %s' % (f.shape, f.dtype))
        if f.min() < np.iinfo(np.int32).min or f.max() > np.iinfo(np.int32).max:
            raise _lib.HDError('MeshRenderer: face indices do not fit in int32')
        if not torch.cuda.is_available():
            raise _lib.HDError('MeshRenderer needs a CUDA device: there is no CPU fallback')
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self.faces = torch.from_numpy(np.ascontiguousarray(f, np.int32)).to(self.device)
        self.num_faces = int(f.shape[0])
        self._ws = None

    def workspace(self, N, S):
        need = int(lib.hd_render_workspace_bytes(N, S, self.num_faces))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    def chunk_frames(self, S):
        """Frames per hd_render_mesh call so that the workspace stays under max_workspace_bytes (at least 1)."""
        per = int(lib.hd_render_workspace_bytes(1, S, self.num_faces))
        return max(1, int(self.max_workspace_bytes // per))

    def render(self, verts, cams, img_size, background=None, rot=None, color='blue', light=DEFAULT_LIGHT,
               bg_color=(1.0, 1.0, 1.0), alpha_out=None, out=None):
        """verts [N,V,3] float32 CUDA (any frame stride; a vertex's xyz must be contiguous, else a dense copy is made);
        cams [N,3] float32 CUDA (any row stride); background [N,S,S,3] float32 CUDA in [-1, 1] or None; rot 3x3 or None.
        -> uint8 [N,S,S,3] CUDA.  alpha_out: optional float32 [N,S,S] CUDA tensor that receives the coverage."""
        S = int(img_size)
        if verts.dim() != 3 or verts.shape[2] != 3:
            raise _lib.HDError('MeshRenderer.render: verts must be [N,V,3], got %s' % (tuple(verts.shape),))
        _lib.fptr(verts)
        _lib.fptr(cams)
        N, V = int(verts.shape[0]), int(verts.shape[1])
        if verts.stride(2) != 1 or verts.stride(1) != 3:
            verts = verts.contiguous()
        if cams.dim() == 1:
            cams = cams.unsqueeze(0)
        if tuple(cams.shape) != (N, 3) or cams.stride(1) != 1:
            raise _lib.HDError('MeshRenderer.render: cams must be [N,3] with unit column stride')
        if background is not None:
            _lib.fptr(background)
            if tuple(background.shape) != (N, S, S, 3) or not background.is_contiguous():
                raise _lib.HDError('MeshRenderer.render: background must be a contiguous float32 [N,%d,%d,3] tensor' % (S, S))
        if alpha_out is not None:
            _lib.fptr(alpha_out)
            if tuple(alpha_out.shape) != (N, S, S) or not alpha_out.is_contiguous():
                raise _lib.HDError('MeshRenderer.render: alpha_out must be a contiguous float32 [N,%d,%d] tensor' % (S, S))
        if out is None:
            out = torch.empty((N, S, S, 3), dtype=torch.uint8, device=verts.device)
        elif tuple(out.shape) != (N, S, S, 3) or out.dtype != torch.uint8 or not out.is_contiguous():
            raise _lib.HDError('MeshRenderer.render: out must be a contiguous uint8 [N,%d,%d,3] tensor' % (S, S))
        if N == 0:
            return out
        p = make_params(color, light, bg_color, rot)
        chunk = self.chunk_frames(S)
        ws = self.workspace(min(N, chunk), S)
        stream = current_stream()
        vb, cb = verts.element_size(), cams.element_size()
        for n0 in range(0, N, chunk):
            n = min(chunk, N - n0)
            check(lib.hd_render_mesh(
                C.c_void_p(verts.data_ptr() + n0 * verts.stride(0) * vb), verts.stride(0), n, V,
                C.c_void_p(self.faces.data_ptr()), self.num_faces,
                C.c_void_p(cams.data_ptr() + n0 * cams.stride(0) * cb), cams.stride(0), C.byref(p),
                None if background is None else C.c_void_p(background[n0].data_ptr()), S,
                C.c_void_p(out[n0].data_ptr()), None if alpha_out is None else C.c_void_p(alpha_out[n0].data_ptr()),
                C.c_void_p(ws.data_ptr()), ws.numel(), stream), 'hd_render_mesh')
        return out


def rotation(deg, axis='y'):
    """The rotation VisRenderer.rotated builds (nmr_renderer.py:189-197): Rodrigues of deg about x, y or z, as float32."""
    import cv2
    ax = {'y': [0, 1., 0], 'x': [1., 0, 0]}.get(axis, [0, 0, 1.])
    return cv2.Rodrigues(np.deg2rad(deg) * np.array(ax))[0].astype(np.float32)
