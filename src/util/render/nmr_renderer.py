"""Drop-in for the reference's src/util/render/nmr_renderer.py: `VisRenderer` with the same constructor and call surface, rendering
on the GPU with hd_render_mesh (human_dynamics_b200.render) instead of the Neural Mesh Renderer.  numpy (or torch) in, numpy out,
like the reference.  The camera chain of `visualize_img_orig` / `visualize_mesh_og` (crop camera -> original-frame camera),
`make_square` and `remove_pads` are here too; skeleton and text drawing (render_utils.py) are not.
"""
from __future__ import absolute_import, division, print_function

import os

import numpy as np
import torch

from human_dynamics_b200.render import COLORS, DEFAULT_LIGHT, MeshRenderer, rotation

colors = COLORS
_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))


def get_dims(x):
    return x.dim() if isinstance(x, torch.Tensor) else x.ndim


class RendererSettings(object):
    """The attributes of NMR's Renderer that the reference reads and writes (image_size is assigned by visualize_img_orig)."""

    def __init__(self, image_size):
        self.image_size = image_size
        self.light_direction, self.light_intensity_directional, self.light_intensity_ambient = DEFAULT_LIGHT
        self.background_color = [1, 1, 1.]


class VisRenderer(object):
    """Renders SMPL meshes with the HMR orthographic camera.  faces are F x 3 or 1 x F x 3; visualisation only (no gradients)."""

    def __init__(self, img_size=256, face_path='src/tf_smpl/smpl_faces.npy', t_size=1):
        self.renderer = RendererSettings(img_size)
        self.set_light_dir([1, .5, -1], int_dir=0.3, int_amb=0.7)
        self.set_bgcolor([1, 1, 1.])
        self.img_size = img_size
        if not os.path.exists(face_path) and not os.path.isabs(face_path):
            face_path = os.path.join(_ROOT, face_path)
        self.faces_np = np.load(face_path).astype(np.int64)
        self.mesh = MeshRenderer(self.faces_np)
        self.default_cam = np.array([[0.9, 0, 0]], np.float32)

    def _render(self, verts, cam, texture, rend_mask, alpha, img, color_name, rot):
        if texture is not None:
            raise NotImplementedError('VisRenderer: only one colour per mesh is supported (texture must be None)')
        num_batch = 1
        if get_dims(verts) == 3 and verts.shape[0] != 1:
            num_batch = verts.shape[0]
            if cam is not None:
                assert get_dims(cam) == 2 and cam.shape[0] == num_batch
            if img is not None:
                assert img.ndim == 4 and img.shape[0] == num_batch
        dev = self.mesh.device
        v = torch.as_tensor(verts, dtype=torch.float32).to(dev)
        if v.dim() == 2:
            v = v.unsqueeze(0)
        if cam is None:
            c = torch.from_numpy(np.repeat(self.default_cam, num_batch, axis=0)).to(dev)
        else:
            c = torch.as_tensor(cam, dtype=torch.float32).to(dev)
            if c.dim() == 1:
                c = c.unsqueeze(0)
        S = int(self.renderer.image_size)
        r = self.renderer
        light = (r.light_direction, r.light_intensity_directional, r.light_intensity_ambient)
        a = torch.empty((v.shape[0], S, S), dtype=torch.float32, device=dev)
        rend = self.mesh.render(v, c, S, rot=rot, color=colors[color_name], light=light, bg_color=r.background_color, alpha_out=a)
        rend = rend.cpu().numpy()
        mask = a.cpu().numpy()
        if rend_mask:
            # render_silhouettes -> unsqueeze(0) -> repeat(1, 3, 1, 1) -> NHWC, as the reference does (nmr_renderer.py:147-155)
            sil = np.tile(mask[None], (1, 3, 1, 1)).transpose((0, 2, 3, 1))
            sil = np.clip(sil, 0, 1) * 255.0
            return (sil[0] if num_batch == 1 else sil).astype(np.uint8)
        if num_batch == 1:
            rend, mask = rend[0], mask[0]
        if alpha or img is not None:
            if img is not None:
                # img is in [0, 255] here (visualize_img scales it); the mesh colour enters as the rendered uint8 value
                m = np.repeat(np.expand_dims(mask, -1), 3, axis=-1)
                return (img * (1 - m) + rend.astype(np.float32) * m).astype(np.uint8)
            mask = mask.reshape((rend.shape[:2]) + (1,))
            return self.make_alpha(rend, mask)
        return rend

    def __call__(self, verts, cam=None, texture=None, rend_mask=False, alpha=False, img=None, color_name='blue'):
        """verts: V x 3 or B x V x 3; cam: [s, tx, ty] or B x 3 (HMR's camera).  -> S x S x 3 uint8 (B x S x S x 3 batched)."""
        return self._render(verts, cam, texture, rend_mask, alpha, img, color_name, None)

    def rotated(self, verts, deg, axis='y', cam=None, texture=None, rend_mask=False, alpha=False, color_name='blue'):
        """The mesh rotated by deg about `axis` through each frame's vertex mean."""
        v = torch.as_tensor(verts, dtype=torch.float32)
        if v.dim() == 2:
            v = v.unsqueeze(0)
        return self._render(v, cam, texture, rend_mask, alpha, None, color_name, rotation(deg, axis))

    def make_alpha(self, rend, mask):
        rend = rend.astype(np.uint8)
        alpha = (mask * 255).astype(np.uint8)
        return np.dstack((rend, alpha))

    def set_light_dir(self, direction, int_dir=0.8, int_amb=0.8):
        self.renderer.light_direction = direction
        self.renderer.light_intensity_directional = int_dir
        self.renderer.light_intensity_ambient = int_amb

    def set_bgcolor(self, color):
        self.renderer.background_color = color


def orig_frame_cam(cam, start_pt, scale, proc_img_shape, img_size, scale_orig=None):
    """Crop camera -> camera in normalised coordinates of the (resized, squared) original frame: the chain of
    visualize_img_orig / visualize_mesh_og (nmr_renderer.py:361-363,388-404).  scale_orig: the max_img_size resize, or None."""
    undo_scale = 1. / np.array(scale) if scale_orig is None else (1. / np.array(scale)) * scale_orig
    cam_crop = np.hstack([proc_img_shape[0] * cam[0] * 0.5, cam[1:] + (2. / cam[0]) * 0.5])
    cam_orig = np.hstack([cam_crop[0] * undo_scale, cam_crop[1:] + (start_pt - proc_img_shape[0]) / cam_crop[0]])
    new_cam = np.hstack([cam_orig[0] * (2. / img_size), cam_orig[1:] - (1 / ((2. / img_size) * cam_orig[0]))])
    return new_cam.astype(np.float32)


def orig_frame_size(H, W, max_img_size):
    """(scale_orig or None, resized height, width, square size) of visualize_img_orig for an H x W frame (common.resize_img)."""
    if max(H, W) > max_img_size:
        scale_orig = max_img_size / float(max(H, W))
        h, w = (np.floor(np.array([H, W]) * scale_orig)).astype(int)
        return scale_orig, int(h), int(w), int(max(h, w))
    return None, H, W, max(H, W)


def make_square(img):
    """Bc nmr only deals with square image, adds pad to the shorter side."""
    img_size = np.max(img.shape[:2])
    pad_vals = img_size - img.shape[:2]
    img = np.pad(array=img, pad_width=((0, pad_vals[0]), (0, pad_vals[1]), (0, 0)), mode='constant')
    return img, pad_vals


def remove_pads(img, pad_vals):
    """Undos padding done by make_square."""
    if pad_vals[0] != 0:
        img = img[:-pad_vals[0], :]
    if pad_vals[1] != 0:
        img = img[:, :-pad_vals[1]]
    return img
