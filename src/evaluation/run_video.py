"""Crop pre-processing in front of the Tester -- drop-in for `process_image` of the reference's
src/evaluation/run_video.py:56-107.  The arithmetic (scale to [-1,1], cv2-convention bilinear resize, edge pad, crop) runs
in one CUDA kernel on the uint8 frame (human_dynamics_b200.preprocess / hd_process_image).  `render_overlays` is the GPU,
batched form of the mesh overlays `render_preds` (run_video.py:110-202) draws (human_dynamics_b200.render / hd_render_mesh)."""
import ctypes as C
import os

import numpy as np
import torch

from human_dynamics_b200 import _lib
from human_dynamics_b200.preprocess import IMG_SIZE, crop_geometry, process_images
from human_dynamics_b200.render import MeshRenderer, rotation
from src.util.render.nmr_renderer import orig_frame_cam, orig_frame_size

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _read_rgb(im_path):
    import cv2                                  # decoding only (the reference uses skimage.io.imread, RGB order)
    bgr = cv2.imread(im_path, cv2.IMREAD_COLOR)
    if bgr is None:
        raise IOError('cannot read image %s' % im_path)
    return np.ascontiguousarray(bgr[:, :, ::-1])


def process_image(im_path, bbox_param):
    """Processes an image, producing 224x224 crop.

    Args:
        im_path (str | HxWx3 uint8 array).
        bbox_param (3,): [cx, cy, scale].

    Returns:
        dict: image, im_path, im_shape, center, scale, start_pt   (run_video.py:99-107).
    """
    image = im_path if isinstance(im_path, np.ndarray) else _read_rgb(im_path)
    crops, geoms = process_images(image[None], np.asarray(bbox_param, np.float64).reshape(1, 3))
    torch.cuda.current_stream().synchronize()
    g = geoms[0]
    return {'image': crops[0].cpu().numpy(), 'im_path': im_path if isinstance(im_path, str) else None, 'im_shape': g['im_shape'],
            'center': g['center'], 'scale': g['scale'], 'start_pt': g['start_pt']}


def process_video_frames(frames, bbox_params):
    """Batched form for a whole track: frames (N,H,W,3) uint8 (host or CUDA), bbox_params (N,3) ->
    (crops (N,224,224,3) float32 CUDA -- feed `Tester.predict_all_images` / `HMMREngine.encode_images` directly --, infos)."""
    return process_images(frames, bbox_params, IMG_SIZE)


def _as_cuda_f32(x, dev):
    return torch.as_tensor(np.asarray(x, np.float32) if not isinstance(x, torch.Tensor) else x, dtype=torch.float32).to(dev)


def render_overlays(preds, crops, infos, frames=None, max_img_size=720, renderer=None, color='blue'):
    """The mesh overlays of `render_preds` for a whole track, on the GPU, without the skeleton panel, PNGs or ffmpeg.

    preds: `Tester.predict_all_images` output ('verts' [N,V,3], 'cams' [N,3]; numpy or CUDA); crops: the [N,224,224,3] [-1, 1]
    crops and infos: the per-frame dicts of `process_video_frames`; frames: the original uint8 [N,H,W,3] frames (host or CUDA).
    -> dict of CUDA uint8 tensors:
        'crop'          [N,224,224,3]  the mesh over each crop (visualize_img);
        'frame'         [N,Hs,Ws,3]    the mesh over the original frame resized to at most max_img_size (visualize_img_orig);
        'frame_rotated' [N,Hs,Ws,3]    the same mesh turned 90 degrees about y through its vertex mean, on white.
    The frame background is hd_process_image with geometry {Hs, Ws, 0, 0} and S = max(Hs, Ws) (the resize of the reference's
    resize_img); cropping the square render to Hs x Ws stands in for make_square / remove_pads."""
    if renderer is None:
        renderer = MeshRenderer(np.load(os.path.join(_ROOT, 'src', 'tf_smpl', 'smpl_faces.npy')))
    dev = renderer.device
    verts = _as_cuda_f32(preds['verts'], dev)
    cams_np = (preds['cams'].detach().cpu().numpy() if isinstance(preds['cams'], torch.Tensor) else np.asarray(preds['cams']))
    N = verts.shape[0]
    crops = _as_cuda_f32(crops, dev).contiguous()
    S_crop = int(crops.shape[1])
    out = {'crop': renderer.render(verts, _as_cuda_f32(cams_np, dev), S_crop, background=crops, color=color)}
    if frames is None:
        return out
    if isinstance(frames, np.ndarray):
        frames = torch.from_numpy(np.ascontiguousarray(frames))
    H, W = int(frames.shape[1]), int(frames.shape[2])
    scale_orig, Hs, Ws, S = orig_frame_size(H, W, max_img_size)
    cams_orig = np.stack([orig_frame_cam(cams_np[i], np.asarray(infos[i]['start_pt']), infos[i]['scale'], infos[i]['im_shape'], S,
                                         scale_orig) for i in range(N)])
    cams_orig = _as_cuda_f32(cams_orig, dev)
    geom = torch.tensor([[Hs, Ws, 0, 0]], dtype=torch.int32, device=dev).repeat(N, 1).contiguous()
    out['frame'] = torch.empty((N, Hs, Ws, 3), dtype=torch.uint8, device=dev)
    out['frame_rotated'] = torch.empty((N, Hs, Ws, 3), dtype=torch.uint8, device=dev)
    rot = rotation(90, 'y')
    chunk = min(N, renderer.chunk_frames(S), 64)
    bg = torch.empty((chunk, S, S, 3), dtype=torch.float32, device=dev)
    sq = torch.empty((chunk, S, S, 3), dtype=torch.uint8, device=dev)
    for n0 in range(0, N, chunk):
        n = min(chunk, N - n0)
        fr = frames[n0:n0 + n].to(dev, non_blocking=True).contiguous()
        _lib.check(_lib.lib.hd_process_image(C.c_void_p(fr.data_ptr()), n, H, W, C.c_void_p(geom.data_ptr()), C.c_void_p(bg.data_ptr()),
                                             S, None, None, 0, _lib.current_stream()), 'hd_process_image')
        renderer.render(verts[n0:n0 + n], cams_orig[n0:n0 + n], S, background=bg[:n], color=color, out=sq[:n])
        out['frame'][n0:n0 + n] = sq[:n, :Hs, :Ws]
        renderer.render(verts[n0:n0 + n], cams_orig[n0:n0 + n], S, rot=rot, color=color, out=sq[:n])
        out['frame_rotated'][n0:n0 + n] = sq[:n, :Hs, :Ws]
    return out


__all__ = ['process_image', 'process_video_frames', 'crop_geometry', 'render_overlays', 'IMG_SIZE']
