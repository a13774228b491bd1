"""HMMR inference engine: the wiring of Tester.build_test_model (src/evaluation/tester.py:169-215) over the
H100 kernels -- images -> ResNet-v2-50 -> f_movie -> IEF (main + delta heads) -> SMPL -> projection.

All compute goes through libhd_b200.so on the current CUDA stream; torch is used for device buffers,
streams and host<->device copies only.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from .config import HMMRConfig
from .nets import FMoviePlan, IEFPlan, PackedConv, PackedFMovie, PackedIEF, PackedResNet, ResNetPlan, sync_packing
from .smpl import SMPLConstants
from ._lib import current_stream


def load_weights(path_or_dict):
    """TF-named variable dict from an in-memory dict, an .npz, or a TensorFlow V2 checkpoint prefix
    (`model.ckpt-NNNN`, recognised like the reference does by its `.index` file, tester.py:35; parsed without TensorFlow
    by human_dynamics_b200.tf_checkpoint)."""
    from . import tf_checkpoint
    if isinstance(path_or_dict, dict):
        return path_or_dict
    if isinstance(path_or_dict, str) and path_or_dict.endswith('.npz'):
        with np.load(path_or_dict) as z:
            return {k: z[k] for k in z.files}
    if isinstance(path_or_dict, str) and path_or_dict.endswith('.index') and tf_checkpoint.is_checkpoint(path_or_dict[:-6]):
        path_or_dict = path_or_dict[:-6]
    if tf_checkpoint.is_checkpoint(path_or_dict):
        return tf_checkpoint.load_checkpoint(path_or_dict)
    raise ValueError('weights must be a dict of TF-named arrays, a .npz path or a TensorFlow checkpoint prefix '
                     '(got %r; `python tools/ckpt_to_npz.py <prefix> out.npz` converts offline)' % (path_or_dict,))


def load_mean_params(path):
    """`neutral_smpl_meanwjoints.h5` of the reference (tester.py:118-141) -> mean_param (1,85) = [0.9,0,0 | pose with root
    (pi,0,0) | shape].  Only the INITIAL value of the trainable `mean_param` variable: a restored checkpoint carries the
    learned one, which wins.  .npz / .npy with 'pose' (72) and 'shape' (10) are read directly; .h5 needs h5py or deepdish
    (not dependencies of this package)."""
    if path.endswith('.npz'):
        with np.load(path) as z:
            pose, shape = np.array(z['pose'], np.float64), np.array(z['shape'], np.float64)
    else:
        try:
            import h5py
        except ImportError as e:
            raise ImportError('reading %s needs h5py (or convert it once: python -c "import deepdish as dd, numpy as np; '
                              'v = dd.io.load(PATH); np.savez(OUT, pose=v[\'pose\'], shape=v[\'shape\'])")' % path) from e
        with h5py.File(path, 'r') as f:
            pose, shape = np.array(f['pose'], np.float64), np.array(f['shape'], np.float64)
    pose = pose.reshape(72).copy()
    pose[:3] = 0.0
    pose[0] = np.pi                                                            # tester.py:126-127
    return np.hstack(([0.9, 0.0, 0.0], pose, shape.reshape(10))).astype(np.float32).reshape(1, 85)


NVTX = os.environ.get('HD_NVTX', '0') != '0'      # NVTX ranges per stage (for nsys / ncu --nvtx timelines); off by default


class _nvtx(object):
    """`with _nvtx('stage'):` -- a torch.cuda.nvtx range when HD_NVTX=1, nothing otherwise."""
    __slots__ = ('name',)

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if NVTX:
            torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *a):
        if NVTX:
            torch.cuda.nvtx.range_pop()
        return False


class _Bounded(dict):
    """dict that forgets its oldest entries beyond `maxlen` (plan / buffer caches keyed by batch shape: a service that sees
    many different shapes must not grow device memory without bound; evicted plans are simply rebuilt on next use)."""

    def __init__(self, maxlen):
        super().__init__()
        self.maxlen = maxlen

    def __setitem__(self, key, value):
        if key not in self:
            while len(self) >= self.maxlen:
                self.pop(next(iter(self)))
        super().__setitem__(key, value)


class PackedHal(object):
    """fc2_res hallucinator (models.py:270-296)."""

    def __init__(self, w, device, tc=False, name='fc2_res'):
        self.fc1 = PackedConv(w[name + '/fc1/weights'], device, post_shift=w[name + '/fc1/biases'], post_relu=True, tc=tc)
        self.fc2 = PackedConv(w[name + '/fc2/weights'], device, post_shift=w[name + '/fc2/biases'], post_relu=True, tc=tc)
        self.fc3 = PackedConv(w[name + '/fc3/weights'], device, post_shift=w[name + '/fc3/biases'], tc=tc)
        sync_packing(device)


class HMMREngine(object):
    def __init__(self, weights, smpl_model, config: HMMRConfig | None = None, device=None, impl=None):
        if not torch.cuda.is_available():
            raise _lib.HDError('HMMREngine needs a CUDA device: the hot path has no CPU fallback')
        self.config = config or HMMRConfig()
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self.impl = impl or self.config.impl
        tc = self.impl if self.impl != 'simt' else False      # which tensor-core packing the layers carry
        w = load_weights(weights)
        self.delta_t_values = [int(d) for d in self.config.delta_t_values]
        with torch.cuda.device(self.device):
            self.resnet = PackedResNet(w, self.device, tc=tc)
            self.fmovie = PackedFMovie(w, self.device, self.config.num_conv_layers, tc=tc) \
                if any(k.startswith('AZ_FC_block2_conv1') for k in w) else None
            self.ief = PackedIEF(w, self.device, delta_t_values=self.delta_t_values, tc=tc)
            self.hal = PackedHal(w, self.device, tc=tc) if 'fc2_res/fc1/weights' in w else None
            self.smpl = smpl_model if isinstance(smpl_model, SMPLConstants) else SMPLConstants(smpl_model, device=self.device)
        self._resnet_plans = _Bounded(8)
        self._weights = w                       # the training-mode trunk reads gamma / beta / moving statistics on first use
        self._train_trunk = None
        self._fmovie_plans = _Bounded(4)
        self._ief_plans = _Bounded(4)
        self._hal_plans = _Bounded(4)
        self._theta0 = _Bounded(8)
        self._phi = _Bounded(96)
        self._outs = _Bounded(4)
        self._graphs = {}

    # ---------------------------------------------------------------- stage API
    EARLY_UNITS = 7          # bottleneck units of blocks 1-2 (3 + 4): stage A; blocks 3-4 are stage B

    def _resnet_plan(self, n, size, stage='A'):
        key = (n, size, stage)
        if key not in self._resnet_plans:
            nu = len(self.resnet.units)
            cut = min(self.EARLY_UNITS, nu)
            if stage == 'A':
                nxt = self.resnet.units[cut]['pre'] if cut < nu else None
                self._resnet_plans[key] = ResNetPlan(self.resnet, n, size, self.impl, units=(0, cut), root=True, tail=False,
                                                     next_pre=nxt, next_has_shortcut=cut < nu and 'shortcut' in self.resnet.units[cut])
            else:
                self._resnet_plans[key] = ResNetPlan(self.resnet, n, size, self.impl, units=(cut, nu), root=False, tail=True)
        return self._resnet_plans[key]

    H2D_PIECE = 32           # frames per host->device copy piece (one event each)

    def stage_a_schedule(self, N, streaming):
        """[(start, n)] of the stage-A passes.  When frames are still arriving from the host the first pass is kept small
        (one copy piece) so compute starts after 19 MB instead of a full chunk; all other passes use `frame_chunk`."""
        cA = max(1, min(int(self.config.frame_chunk), N))
        out, i = [], 0
        if streaming and N > cA and cA > self.H2D_PIECE:
            out.append((0, self.H2D_PIECE))
            i = self.H2D_PIECE
        while i < N:
            n = min(cA, N - i)
            out.append((i, n))
            i += n
        return out

    def _trunk(self, images, phi, events=None, frames=None):
        """ResNet over N frames in two stages: root + blocks 1-2 per `frame_chunk` frames (working set near L2),
        then blocks 3-4 + postnorm/mean per `late_chunk` frames (small maps need many frames to fill the SMs).
        `events[i]` (optional) is waited on before chunk i of stage A (host->device copy of that chunk).
        `frames` = (uint8 [N,H,W,3] CUDA tensor, int32 [N,4] geometry table): stage A then starts from raw video frames --
        process_image (run_video.py:56-107) writes conv1's input planes directly and `images` is unused (None)."""
        if frames is not None:
            N, size = frames[0].shape[0], int(self.config.img_size)
        else:
            N, size = images.shape[0], images.shape[1]
        st = current_stream()
        cA = max(1, min(int(self.config.frame_chunk), N))
        cB = max(1, min(int(self.config.late_chunk), N))
        pa = self._resnet_plan(cA, size, 'A')
        key = ('mid', N, size)
        if key not in self._phi:
            self._phi[key] = torch.empty((N, pa.out_hw, pa.out_hw, pa.out_depth), dtype=torch.float32, device=self.device)
        mid = self._phi[key]
        mid_split = None
        if pa.split and pa.out_split is not None:
            skey = ('mid16', N, size)
            if skey not in self._phi:
                self._phi[skey] = (torch.empty(mid.shape, dtype=torch.float16, device=self.device),
                                   torch.empty(mid.shape, dtype=torch.float16, device=self.device))
            mid_split = self._phi[skey]
        main = torch.cuda.current_stream()
        for i, n in self.stage_a_schedule(N, events is not None):
            plan = self._resnet_plan(n, size, 'A')
            if events is not None:
                for ev in events[i // self.H2D_PIECE:(i + n + self.H2D_PIECE - 1) // self.H2D_PIECE]:
                    main.wait_event(ev)
            plan.set_output(mid[i:i + n], (mid_split[0][i:i + n], mid_split[1][i:i + n]) if mid_split else None)
            if frames is None:
                with _nvtx('resnet root + blocks 1-2 [%d:%d]' % (i, i + n)):
                    plan.run(images[i:i + n], None, st)
            else:
                fr, geom = frames
                H, W = fr.shape[1], fr.shape[2]
                if plan.planes is not None:
                    _lib.check(_lib.lib.hd_process_image(C.c_void_p(fr[i:i + n].data_ptr()), n, H, W, C.c_void_p(geom[i:i + n].data_ptr()), None,
                                                         size, C.c_void_p(plan.planes[0].data_ptr()), C.c_void_p(plan.planes[1].data_ptr()),
                                                         plan.planes[0].shape[2], st), 'hd_process_image')
                    plan.run(None, None, st)
                else:                                 # conv1 without the plane path (simt / tc3 modes): materialise the fp32 crops
                    ckey = ('crops', n, size)
                    if ckey not in self._phi:
                        self._phi[ckey] = torch.empty((n, size, size, 3), dtype=torch.float32, device=self.device)
                    crops = self._phi[ckey]
                    _lib.check(_lib.lib.hd_process_image(C.c_void_p(fr[i:i + n].data_ptr()), n, H, W, C.c_void_p(geom[i:i + n].data_ptr()),
                                                         C.c_void_p(crops.data_ptr()), size, None, None, 0, st), 'hd_process_image')
                    plan.run(crops, None, st)
        for i in range(0, N, cB):
            n = min(cB, N - i)
            plan = self._resnet_plan(n, size, 'B')
            plan.set_input(mid[i:i + n], (mid_split[0][i:i + n], mid_split[1][i:i + n]) if mid_split else None)
            with _nvtx('resnet blocks 3-4 + pool5 [%d:%d]' % (i, i + n)):
                plan.run(None, phi[i:i + n], st)
        return phi

    def encode_images(self, images, out=None):
        """encoder_resnet: (N,H,W,3) float32 CUDA NHWC -> (N,2048)."""
        if not images.is_cuda or images.dtype != torch.float32:
            raise _lib.HDError('encode_images: float32 CUDA tensor required (no CPU fallback exists)')
        if images.dim() != 4 or images.shape[3] != 3 or images.shape[1] != images.shape[2]:
            raise _lib.HDError('encode_images: expected (N,S,S,3) NHWC, got %s' % (tuple(images.shape),))
        images = images.contiguous()
        N = images.shape[0]
        phi = out if out is not None else torch.empty((N, self.resnet.out_dim), dtype=torch.float32, device=images.device)
        if N:
            self._trunk(images, phi)
        return phi

    def encode_images_train(self, images):
        """encoder_resnet(is_training=True): (N,H,W,3) float32 CUDA NHWC -> (N,2048), every batch norm with the moments of these N
        frames (nets.ResNetTrainPlan over the whole batch).  The moving statistics are left alone, as a TF graph leaves them when its
        update ops are not run."""
        from .objective import _TrainTrunk
        if not isinstance(images, torch.Tensor) or not images.is_cuda or images.dtype != torch.float32 or images.dim() != 4:
            raise _lib.HDError('encode_images_train: float32 CUDA tensor (N,S,S,3) required (no CPU fallback exists)')
        if images.shape[0] < 1:
            raise _lib.HDError('encode_images_train: batch statistics need at least one frame')
        if self._train_trunk is None:
            self._train_trunk = _TrainTrunk(self._weights, self.device)
        phi, _ = self._train_trunk(images[None])
        return phi[0]

    def temporal_encode(self, feats):
        """az_fc2_groupnorm ("f_movie"): (B,T,2048) -> (B,T,2048)."""
        if self.fmovie is None:
            raise _lib.HDError('no f_movie weights were loaded')
        B, T = feats.shape[0], feats.shape[1]
        key = (B, T)
        if key not in self._fmovie_plans:
            self._fmovie_plans[key] = FMoviePlan(self.fmovie, B, T, self.impl)
        return self._fmovie_plans[key].run(feats.contiguous())

    def hallucinate(self, feats):
        """fc2_res: (B,T,2048) -> (B,T,2048)   (pred_mode='hal')."""
        if self.hal is None:
            raise _lib.HDError('no fc2_res weights were loaded')
        feats = feats.contiguous()
        N = feats.shape[0] * feats.shape[1]
        if N not in self._hal_plans:
            f32 = dict(dtype=torch.float32, device=feats.device)
            self._hal_plans[N] = [torch.empty((N, 2048), **f32) for _ in range(3)]
        h1, h2, out = self._hal_plans[N]
        st = current_stream()
        self.hal.fc1.bind(feats, N, 1, 1, h1, impl=self.impl).run(st)
        self.hal.fc2.bind(h1, N, 1, 1, h2, impl=self.impl).run(st)
        self.hal.fc3.bind(h2, N, 1, 1, out, res=feats, res_geom=(2048, 1, 1, 1), impl=self.impl).run(st)
        return out.view(feats.shape)

    def theta_mean(self, N):
        if N not in self._theta0:
            self._theta0[N] = self.ief.mean_param.expand(N, 85).contiguous()
        return self._theta0[N]

    def regress(self, feats, omega_start=None, delta_keys=None):
        """call_hmr_ief: feats (N,2048) -> (omega (N,85), {dt: (N,85)})."""
        feats = feats.contiguous()
        N = feats.shape[0]
        keys = tuple(sorted(self.ief.deltas.keys())) if delta_keys is None else tuple(sorted(k for k in delta_keys if k != 0))
        plan = self._ief_plan(N, keys)
        theta0 = self.theta_mean(N) if omega_start is None else omega_start.contiguous()
        return plan.run(feats.view(N, -1), theta0)

    def _ief_plan(self, N, keys):
        pk = (N, tuple(keys))
        if pk not in self._ief_plans:
            self._ief_plans[pk] = IEFPlan(self.ief, N, self.config.num_stage, list(keys), self.impl)
        return self._ief_plans[pk]

    def _out_buffers(self, N, D):
        key = (N, D)
        if key not in self._outs:
            V, K = self.smpl.num_verts, self.smpl.num_kps
            f32 = dict(dtype=torch.float32, device=self.device)

            def mk(rows):
                return {'verts': torch.empty((rows, V, 3), **f32), 'joints': torch.empty((rows, K, 3), **f32),
                        'Rs': torch.empty((rows, 24, 3, 3), **f32), 'Jtr': torch.empty((rows, 24, 3), **f32),
                        'kps': torch.empty((rows, K, 2), **f32)}
            self._outs[key] = (mk(N), mk(N * D) if D else None)
        return self._outs[key]

    # ---------------------------------------------------------------- full window
    def predict(self, images, single_frame=False, on_main_ready=None):
        """Tester.predict on device.  images (B,T,S,S,3) float32 CUDA -> dict of CUDA tensors with the 14
        fetch keys of tester.py:217-255 (+ '_phi', '_movie_strips' for inspection).  Outputs are plan-owned
        buffers that the next predict() of the same shape overwrites."""
        if images.dim() != 5:
            raise _lib.HDError('predict: expected (B,T,S,S,3)')
        B, T = images.shape[0], images.shape[1]
        N = B * T
        key = ('phi', N)
        if key not in self._phi:
            self._phi[key] = torch.empty((N, self.resnet.out_dim), dtype=torch.float32, device=self.device)
        phi = self.encode_images(images.reshape((N,) + tuple(images.shape[2:])), out=self._phi[key])
        return self.predict_from_features(phi.view(B, T, -1), single_frame=single_frame, on_main_ready=on_main_ready)

    def predict_graphed(self, images, single_frame=False):
        """`predict` replayed from a CUDA graph: the ~190 kernel launches of a window are captured once per input buffer /
        shape and afterwards submitted as ONE graph launch (no per-kernel launch gaps, no Python between kernels).
        `images` must stay at the same address (same contract as a TF placeholder fed from a fixed staging buffer);
        outputs are the plan-owned buffers of `predict`.  Returns (out, kernel_nodes)."""
        key = (images.data_ptr(), tuple(images.shape), bool(single_frame))
        ent = self._graphs.get(key)
        if ent is None:
            if len(self._graphs) >= 4:                      # bounded: a graph pins its plans' buffers
                self._graphs.pop(next(iter(self._graphs)))
            self.predict(images, single_frame=single_frame)            # eager warm-up: allocations, plan binding, function attributes
            torch.cuda.synchronize()
            n0 = int(_lib.lib.hd_launch_count())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = self.predict(images, single_frame=single_frame)
            # the graph holds raw device pointers: pin everything the caches held at capture time so a later eviction cannot free it
            keep = [dict(c) for c in (self._resnet_plans, self._fmovie_plans, self._ief_plans, self._hal_plans, self._theta0,
                                      self._phi, self._outs)] + [dict(self.smpl._tc_bufs)]
            ent = (g, out, int(_lib.lib.hd_launch_count()) - n0, images, keep)
            self._graphs[key] = ent
        ent[0].replay()
        return ent[1], ent[2]

    def predict_graphed_split(self, images, on_main_ready):
        """`predict_graphed` in two graphs with a host hook between them: graph A ends when the dt=0 outputs are complete (trunk,
        f_movie, main IEF head, SMPL), `on_main_ready(out)` runs (multi-GPU: starts their gather to rank 0 on a side stream),
        graph B is the delta heads.  Two graph launches per window instead of ~200 kernel launches, and the gather still overlaps
        the delta heads.  Returns (out, kernel_nodes)."""
        key = (images.data_ptr(), tuple(images.shape), 'split')
        ent = self._graphs.get(key)
        if ent is None:
            if len(self._graphs) >= 4:
                self._graphs.pop(next(iter(self._graphs)))
            self.predict(images)                                       # eager warm-up
            torch.cuda.synchronize()
            n0 = int(_lib.lib.hd_launch_count())
            ga, gb = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream())
            box = {}
            with torch.cuda.stream(side):
                ga.capture_begin()

                def boundary(out_main):
                    ga.capture_end()
                    box['main'] = dict(out_main)
                    gb.capture_begin()
                out = self.predict(images, on_main_ready=boundary)
                gb.capture_end()
            torch.cuda.current_stream().wait_stream(side)
            keep = [dict(c) for c in (self._resnet_plans, self._fmovie_plans, self._ief_plans, self._hal_plans, self._theta0,
                                      self._phi, self._outs)] + [dict(self.smpl._tc_bufs)]
            ent = (ga, gb, out, box['main'], int(_lib.lib.hd_launch_count()) - n0, images, keep)
            self._graphs[key] = ent
        ent[0].replay()
        on_main_ready(ent[3])
        ent[1].replay()
        return ent[2], ent[4]

    FETCH_KEYS = tuple(a + b for b in ('', '_delta') for a in ('cams', 'joints', 'kps', 'poses', 'shapes', 'verts', 'omegas'))

    HOST_RING = 2            # result buffer sets handed out in turn: a returned dict stays valid for HOST_RING - 1 more calls

    def predict_host(self, images_host, single_frame=False, fetch=None, bbox_params=None, on_main_ready=None, defer=False):
        """The one host->device->host crossing of `sess.run(fetch_dict, feed_dict)` (tester.py:239-258).

        images_host: (B,T,S,S,3) float32 CPU tensor -- the crops `Tester.predict` is fed -- or, with `bbox_params` (B,T,3),
        (B,T,H,W,3) uint8 video frames that process_image (run_video.py:56-107) crops on the GPU (4x fewer bytes per sample
        over PCIe, and no host-side resize).  Pinned (or cudaHostRegister-ed) memory gives real overlap: frames go up in
        H2D_PIECE pieces on a copy stream while the ResNet consumes earlier pieces; results come back into pinned host
        buffers owned by the engine (a ring of HOST_RING sets).  Returns (dict of CPU tensors, h2d_bytes, d2h_bytes); the
        copies are only complete after `torch.cuda.current_stream().synchronize()`.

        defer=True (streaming): returns (host, h2d, d2h, done_event) without making the current stream wait for the device->host
        copies; the caller overlaps them with the NEXT window (device input buffers alternate, results land in the next ring
        slot) and calls `done_event.synchronize()` before reading `host`.  See Tester.predict_stream."""
        u8 = bbox_params is not None
        if images_host.is_cuda or images_host.dim() != 5 or images_host.dtype != (torch.uint8 if u8 else torch.float32):
            raise _lib.HDError('predict_host: expected a CPU tensor (B,T,S,S,3) float32, or (B,T,H,W,3) uint8 with bbox_params')
        B, T = images_host.shape[0], images_host.shape[1]
        N = B * T
        flat = images_host.reshape((N,) + tuple(images_host.shape[2:]))
        self._stream_step = getattr(self, '_stream_step', 0) + 1
        ring = (self._stream_step & 1) if defer else 0          # streaming: the next window uploads while this one still computes
        key = ('img', N, tuple(flat.shape[1:]), flat.dtype, ring)
        if key not in self._phi:
            self._phi[key] = torch.empty(tuple(flat.shape), dtype=flat.dtype, device=self.device)
        if getattr(self, '_copy_stream', None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._d2h_stream = torch.cuda.Stream(device=self.device)
            self._img_read = {}                                  # device input buffer -> event: its last reader (the trunk) is done
            self._d2h_done = None                                # event: the previous window's results have left the device
        if ('phi', N) not in self._phi:
            self._phi[('phi', N)] = torch.empty((N, self.resnet.out_dim), dtype=torch.float32, device=self.device)
        dev_img, phi = self._phi[key], self._phi[('phi', N)]
        geom_dev = None
        if u8:
            from .preprocess import geometry_table
            g, _ = geometry_table((flat.shape[1], flat.shape[2]), np.asarray(bbox_params, np.float64).reshape(N, 3), int(self.config.img_size))
            gkey = ('geom', N)
            if gkey not in self._phi:
                self._phi[gkey] = (torch.empty((N, 4), dtype=torch.int32, pin_memory=True), torch.empty((N, 4), dtype=torch.int32, device=self.device))
            self._phi[gkey][0].copy_(torch.from_numpy(g))
            geom_dev = self._phi[gkey][1]
        chunk = self.H2D_PIECE
        starts = list(range(0, N, chunk))
        ekey = ('ev', len(starts))
        if ekey not in self._phi:
            self._phi[ekey] = [torch.cuda.Event() for _ in starts]
        events = self._phi[ekey]
        main = torch.cuda.current_stream()
        cs, ds = self._copy_stream, self._d2h_stream
        if defer and key in self._img_read:
            cs.wait_event(self._img_read[key])       # only the window that last used THIS buffer has to be through its trunk
        else:
            cs.wait_stream(main)                     # the previous step may still read dev_img
        with torch.cuda.stream(cs):
            if u8:
                geom_dev.copy_(self._phi[('geom', N)][0], non_blocking=True)
            for ev, i in zip(events, starts):
                n = min(chunk, N - i)
                dev_img[i:i + n].copy_(flat[i:i + n], non_blocking=True)
                ev.record(cs)
        if u8:
            self._trunk(None, phi, events, frames=(dev_img, geom_dev))
        else:
            self._trunk(dev_img, phi, events)
        ev_img = torch.cuda.Event()
        ev_img.record(main)
        self._img_read[key] = ev_img
        if self._d2h_done is not None:               # the heads are about to overwrite the output buffers the previous window's
            main.wait_event(self._d2h_done)          # device->host copies read (long finished by now: a formality, not a stall)
        want = list(fetch or self.FETCH_KEYS)
        host, counted = {}, [0]
        self._host_slot = (getattr(self, '_host_slot', -1) + 1) % self.HOST_RING
        slot = self._host_slot

        def to_host(tensors, stream):
            for k, v in tensors.items():
                if k not in want or k in host:
                    continue
                hk = ('host', slot, k, tuple(v.shape))
                if hk not in self._phi:
                    self._phi[hk] = torch.empty(tuple(v.shape), dtype=torch.float32, pin_memory=True)
                with torch.cuda.stream(stream):
                    self._phi[hk].copy_(v, non_blocking=True)
                host[k] = self._phi[hk]
                counted[0] += v.numel() * 4

        def main_ready(main_out):            # dt=0 outputs: device->host on their own stream, overlapped with the delta heads
            ev = torch.cuda.Event()
            ev.record(main)
            ds.wait_event(ev)
            to_host(main_out, ds)
            if on_main_ready is not None:    # (multi-GPU: the same moment starts the gather towards rank 0)
                on_main_ready(main_out)

        out = self.predict_from_features(phi.view(B, T, -1), single_frame=single_frame, on_main_ready=main_ready)
        ev = torch.cuda.Event()
        ev.record(main)
        ds.wait_event(ev)
        to_host({k: v for k, v in out.items() if not k.startswith('_')}, ds)
        done = torch.cuda.Event()
        done.record(ds)
        self._d2h_done = done
        d2h = counted[0]
        h2d = flat.numel() * flat.element_size() + (N * 16 if u8 else 0)
        if defer:
            return host, h2d, d2h, done
        main.wait_event(done)                 # one synchronisation point for the caller: the current stream
        return host, h2d, d2h

    def predict_from_features(self, phi, single_frame=False, on_main_ready=None):
        B, T = phi.shape[0], phi.shape[1]
        N = B * T
        if single_frame:
            strips = phi
            omega, deltas = self.regress(phi.reshape(N, -1), delta_keys=())
        else:
            mode = self.config.pred_mode
            if mode == 'pred':
                with _nvtx('f_movie'):
                    strips = self.temporal_encode(phi)
            elif mode == 'hal':
                strips = self.hallucinate(phi)
            else:
                raise Exception('Pred mode {} not recognized'.format(mode))
            plan = self._ief_plan(N, tuple(sorted(self.ief.deltas.keys())))
            with _nvtx('IEF main head'):
                omega = plan.run_main(strips.reshape(N, -1), self.theta_mean(N))
            deltas = None
        dts = sorted(self.ief.deltas.keys()) if not single_frame else []
        D = len(dts)
        K, V = self.smpl.num_kps, self.smpl.num_verts
        o0, od = self._out_buffers(N, D)
        cams = omega[:, 0:3]
        # OmegasPred.compute_smpl (omega.py:263-304) for the dt=0 instance ...
        with _nvtx('SMPL dt=0'):
            self.smpl.forward(omega[:, 75:85], omega[:, 3:75], cam=cams, out=o0)
        out = {'cams': cams.reshape(B, T, 3), 'joints': o0['joints'].view(B, T, K, 3), 'kps': o0['kps'].view(B, T, K, 2),
               'poses': o0['Rs'].view(B, T, 24, 3, 3), 'shapes': omega[:, 75:85].reshape(B, T, 10),
               'verts': o0['verts'].view(B, T, V, 3), 'omegas': omega.view(B, T, 85)}
        if on_main_ready is not None:        # the dt=0 results can start their trip to the host while the delta heads compute
            on_main_ready(out)
        if D:
            with _nvtx('IEF delta heads'):
                deltas = self._ief_plan(N, tuple(dts)).run_deltas()
        if D:
            # ... and every delta instance; cams come from the dt=0 prediction (set_cams, tester.py:210-213).
            # Pose n of delta i is written to slot n*D+i, i.e. directly into the [B,T,D,...] stacking of tester.py:252.
            for i, dt in enumerate(dts):
                d = deltas[dt]
                with _nvtx('SMPL dt=%+d' % dt):
                    self.smpl.forward(d[:, 75:85], d[:, 3:75], cam=cams, out=od, slot=(D, i))
            omegas_delta = self._ief_plan(N, tuple(dts)).delta_all.view(B, T, D, 85)
            out.update({'cams_delta': cams.reshape(B, T, 1, 3).expand(B, T, D, 3),
                        'joints_delta': od['joints'].view(B, T, D, K, 3), 'kps_delta': od['kps'].view(B, T, D, K, 2),
                        'poses_delta': od['Rs'].view(B, T, D, 24, 3, 3), 'shapes_delta': omegas_delta[..., 75:85],
                        'verts_delta': od['verts'].view(B, T, D, V, 3), 'omegas_delta': omegas_delta})
        out['_phi'] = phi
        out['_movie_strips'] = strips
        return out

