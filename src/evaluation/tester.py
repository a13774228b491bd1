"""Tester -- drop-in for the reference's src/evaluation/tester.py (inference graph + predict).

`Tester(config).predict(images)` returns the same 14-key dict of numpy arrays as the reference's
`sess.run(fetch_dict)` (tester.py:217-258); `predict_all_images` is the sliding-window driver
(tester.py:260-312).  The graph is replaced by an HMMREngine plan on the current CUDA device.
"""
import os

import numpy as np
import torch

from human_dynamics_b200 import runtime as _rt
from human_dynamics_b200.engine import HMMREngine, load_weights


class Tester(object):

    def __init__(self, config, pretrained_resnet_path='', sequence_length=None, engine=None):
        self.config = config
        self.load_path = getattr(config, 'load_path', '')
        weights = getattr(config, 'weights', None)
        if engine is None and weights is None:
            if not self.load_path:
                raise Exception('[!] You need to specify `load_path` to load a pretrained model')     # tester.py:31-34
            if not os.path.exists(self.load_path) and not os.path.exists(self.load_path + '.index'):
                raise Exception('{} doesnt exist..'.format(self.load_path))                           # tester.py:35-38 (no ipdb)
            weights = load_weights(self.load_path)
        if pretrained_resnet_path:                                                                    # tester.py:99-109
            if weights is None:
                raise ValueError('pretrained_resnet_path needs the weights to merge into: pass config.load_path / '
                                 'config.weights instead of a pre-built engine')
            rw = load_weights(pretrained_resnet_path)
            weights = dict(weights)
            weights.update({k: v for k, v in rw.items() if k.startswith('resnet_v2_50')})
        if weights is not None and 'mean_param' not in weights:                                       # tester.py:118-141
            mean_path = os.path.join(os.path.dirname(getattr(config, 'smpl_model_path', '') or ''), 'neutral_smpl_meanwjoints.h5')
            alt = mean_path[:-3] + '.npz'
            from human_dynamics_b200.engine import load_mean_params
            weights = dict(weights)
            weights['mean_param'] = load_mean_params(alt if os.path.exists(alt) else mean_path)

        self.batch_size = config.batch_size
        self.sequence_length = sequence_length if sequence_length else config.sequence_length
        self.pred_mode = config.pred_mode
        self.num_conv_layers = config.num_conv_layers
        self.fov = self.num_conv_layers * 4 + 1                                                       # tester.py:48
        self.delta_t_values = [int(dt) for dt in config.delta_t_values]
        self.img_size = getattr(config, 'img_size', 224)
        self.num_output = 85
        smpl_model = getattr(config, 'smpl_model', None) or getattr(config, 'smpl_model_path', '')
        self.engine = engine if engine is not None else HMMREngine(weights, smpl_model, config)
        self.smpl = self.engine.smpl
        _rt.set_default_engine(self.engine)
        self._pinned = {}
        self._registered = {}

    MAX_REGISTERED = 2

    def _as_pinned(self, arr):
        """A CPU tensor over the caller's numpy buffer that the copy engine can read asynchronously.

        The reference's `sess.run(feed_dict=...)` copies the array into TF's own staging memory first; here the caller's
        buffer itself is page-locked in place (cudaHostRegister, once per buffer -- a video loop that refills the same
        array pays it once).  Falls back to a staged copy through an engine-owned pinned buffer if registration fails."""
        t = torch.from_numpy(arr)
        if t.is_pinned():
            return t
        key = (arr.ctypes.data, arr.nbytes)
        if key not in self._registered:
            while len(self._registered) >= self.MAX_REGISTERED:
                old_key, _ = next(iter(self._registered.items()))
                torch.cuda.cudart().cudaHostUnregister(old_key[0])
                del self._registered[old_key]
            rc = torch.cuda.cudart().cudaHostRegister(arr.ctypes.data, arr.nbytes, 0)
            if int(rc) != 0:
                skey = (tuple(arr.shape), arr.dtype.str)
                if skey not in self._pinned:
                    self._pinned[skey] = torch.empty(tuple(arr.shape), dtype=t.dtype, pin_memory=True)
                self._pinned[skey].copy_(t)
                return self._pinned[skey]
            self._registered[key] = arr                      # keeps the buffer alive while it is page-locked
        return t

    def __del__(self):
        try:
            for key in list(getattr(self, '_registered', {})):
                torch.cuda.cudart().cudaHostUnregister(key[0])
        except Exception:
            pass

    def predict(self, images, as_numpy=True, copy=False):
        """Runs forward pass of model.  images (BxTxHxWx3) numpy / torch (host or device) -> dict (tester.py:229-258).

        Host input = ONE overlapped host->device->host crossing, like sess.run(fetch_dict, feed_dict): the frames stream
        up in pieces while the ResNet runs, all 14 fetch tensors come back into pinned host memory.  The returned numpy
        arrays are views of engine-owned result buffers that are recycled every `HMMREngine.HOST_RING` calls; pass
        copy=True for arrays you own (what sess.run returns) at the price of a 160 MB host memcpy per call."""
        B, T = self.batch_size, self.sequence_length
        exp = (B, T, self.img_size, self.img_size, 3)
        if tuple(images.shape) != exp:
            raise ValueError('images must have the static shape %s baked at construction (tester.py:64-66), got %s'
                             % (exp, tuple(images.shape)))
        if isinstance(images, np.ndarray):
            images = self._as_pinned(np.ascontiguousarray(images, dtype=np.float32))
        if images.is_cuda:
            out = self.engine.predict(images.float())
            out = {k: v for k, v in out.items() if not k.startswith('_')}
            if not as_numpy:
                return out
            torch.cuda.current_stream().synchronize()
            return {k: v.cpu().numpy() for k, v in out.items()}
        host, _, _ = self.engine.predict_host(images if images.dtype == torch.float32 else images.float())
        torch.cuda.current_stream().synchronize()
        if not as_numpy:
            return host
        return {k: (v.numpy().copy() if copy else v.numpy()) for k, v in host.items()}

    def predict_frames(self, frames, bbox_params, as_numpy=True, copy=False):
        """process_image + predict in one crossing: frames (BxTxHxWx3) uint8 video frames, bbox_params (BxTx3) [cx, cy, scale]
        (run_video.py:56-107 then tester.py:229).  The crop runs on the GPU from the uint8 frames (1 byte per sample over
        PCIe instead of 4) and writes the ResNet's first-layer input format directly.  Same result dict as `predict`."""
        B, T = self.batch_size, self.sequence_length
        if tuple(frames.shape[:2]) != (B, T) or frames.shape[-1] != 3 or len(frames.shape) != 5:
            raise ValueError('frames must be (%d,%d,H,W,3) uint8' % (B, T))
        if isinstance(frames, np.ndarray):
            if frames.dtype != np.uint8:
                raise ValueError('frames must be uint8')
            frames = self._as_pinned(np.ascontiguousarray(frames))
        host, _, _ = self.engine.predict_host(frames, bbox_params=np.asarray(bbox_params, np.float64).reshape(B, T, 3))
        torch.cuda.current_stream().synchronize()
        if not as_numpy:
            return host
        return {k: (v.numpy().copy() if copy else v.numpy()) for k, v in host.items()}

    def predict_stream(self, windows, bbox_params=None, copy=False):
        """Streaming form of `predict` for a sequence of windows (what a video does): yields one result dict per window, in order.

        windows: iterable of (B,T,S,S,3) float32 arrays -- or, with `bbox_params` (an iterable of (B,T,3) arrays alongside), of
        (B,T,H,W,3) uint8 frame arrays.  Window i+1 is uploaded and computed while window i's 160 MB of results still travel
        to the host (two device input buffers, two result slots), so the per-window cost is the GPU time, not GPU + PCIe tail.
        A yielded dict is valid until the generator is advanced twice more (or pass copy=True)."""
        boxes = iter(bbox_params) if bbox_params is not None else None
        prev = None
        for w in windows:
            arr = self._as_pinned(np.ascontiguousarray(w)) if isinstance(w, np.ndarray) else w
            bb = None
            if boxes is not None:
                bb = np.asarray(next(boxes), np.float64).reshape(self.batch_size, self.sequence_length, 3)
            cur = self.engine.predict_host(arr, bbox_params=bb, defer=True)
            if prev is not None:
                prev[3].synchronize()
                yield {k: (v.numpy().copy() if copy else v.numpy()) for k, v in prev[0].items()}
            prev = cur
        if prev is not None:
            prev[3].synchronize()
            yield {k: (v.numpy().copy() if copy else v.numpy()) for k, v in prev[0].items()}

    def predict_all_images(self, all_images, cache_features=True):
        """Sliding-window prediction over a whole sequence (tester.py:260-312).  all_images: N x H x W x 3, a numpy array or a float32
        CUDA tensor (read in place on the device, no host round trip with the default cache_features).

        Windows are formed exactly as the reference does (margin zero-images in front, zero-image fill at the back, stride
        g = T - 2*margin, keep [margin:-margin]) because GroupNorm couples all T frames of a window.  With
        `cache_features` (default) the per-frame ResNet runs ONCE per real frame (+ once for the zero image) and the
        windows are assembled from cached features on the device -- the reference pushes every frame through the ResNet
        T/g = 2.5 times; the encoder is per-frame, so the results are identical.  cache_features=False replays the
        reference literally (whole image windows through `predict`).
        """
        B, T = self.batch_size, self.sequence_length
        N = len(all_images)
        H, W = self.img_size, self.img_size
        margin = (self.fov - 1) // 2
        g = self.sequence_length - 2 * margin
        if g <= 0:
            raise ValueError('sequence_length %d leaves no frame with full field of view %d' % (T, self.fov))
        count = int(np.ceil(N / (g * B)))
        num_fill = count * B * g + T - N
        on_device = isinstance(all_images, torch.Tensor) and all_images.is_cuda
        if on_device:
            if all_images.dtype != torch.float32:
                raise ValueError('all_images on the device must be float32, got %s' % all_images.dtype)
            all_images = all_images.contiguous()
        else:
            all_images = np.asarray(all_images, dtype=np.float32)
        if tuple(all_images.shape[1:]) != (H, W, 3):
            raise ValueError('all_images must be N x %d x %d x 3' % (H, W))
        if on_device and not cache_features:
            all_images = all_images.cpu().numpy()
        results = {}
        if cache_features:
            dev = self.engine.device
            phi_parts = []
            for i in range(0, N, 640):                       # bounded device residency of raw frames
                if on_device:
                    x = all_images[i:i + 640].to(dev)
                else:
                    x = torch.from_numpy(all_images[i:i + 640]).to(dev, non_blocking=True)
                phi_parts.append(self.engine.encode_images(x).clone())
            phi_zero = self.engine.encode_images(torch.zeros((1, H, W, 3), dtype=torch.float32, device=dev)).clone()
            phi_padded = torch.cat([phi_zero.expand(margin, -1)] + phi_parts + [phi_zero.expand(num_fill, -1)], dim=0)
            idx = (torch.arange(B, device=dev) * g)[:, None] + torch.arange(T, device=dev)[None, :]       # (B, T) frame ids
            for c in range(count):
                windows = phi_padded[idx + c * B * g]                                                     # (B, T, 2048)
                out = self.engine.predict_from_features(windows.contiguous())
                torch.cuda.current_stream().synchronize()
                for k, v in out.items():
                    if not k.startswith('_'):
                        results.setdefault(k, []).append(v.cpu().numpy())
        else:
            images_padded = np.concatenate((np.zeros((margin, H, W, 3), np.float32), all_images,
                                            np.zeros((num_fill, H, W, 3), np.float32)), axis=0)
            for c in range(count):
                batch = np.stack([images_padded[(c * B + i) * g:(c * B + i) * g + T] for i in range(B)])
                pred = self.predict(batch, copy=True)            # results are kept across calls here
                for k, v in pred.items():
                    results.setdefault(k, []).append(v)
        new_results = {}
        for k, v in results.items():
            v = np.array(v)[:, :, margin:-margin]
            new_results[k] = v.reshape((-1,) + v.shape[3:])[:N]
        return new_results
