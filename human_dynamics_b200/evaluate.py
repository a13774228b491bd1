"""Scoring on the GPU: the reference's compute_errors_batched (src/evaluation/eval.py:114-193) over csrc/eval.cu.

`Evaluator(smpl_consts).errors(...)` takes the arguments of compute_errors_batched and returns the same keys, lengths and values;
`errors_many(tubes)` scores any number of tubes (a tfrecord, a dataset) in one pass and returns one such dict per tube.  Inputs may be
numpy arrays or torch tensors, on the host or on the device.  One pass uploads the inputs once, launches

    hd_eval_frames                                                 (always: every 2-D / 3-D / acceleration metric of every frame)
    hd_eval_mesh_tpose, hd_rot2aa, then per chunk of frames
        2 x hd_smpl_forward (2 launches each) + hd_eval_verts_error (with compute_mesh)

with no host synchronisation in between, and fetches one result array.  There is no CPU fallback.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import lib, check, dptr, fptr, current_stream

COLS = _lib.HD_EVAL_COLS
MAX_MESH_CHUNK = 4096          # hd_smpl_forward keeps one kernel configuration (8 poses per block) up to here


def _dev32(x, dev):
    if isinstance(x, torch.Tensor):
        return x.to(device=dev, dtype=torch.float32)
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dev)


def _cat(parts, dev):
    """One upload for host parts (concatenated on the host), a device concatenation for tensors; a single part is used as is."""
    if len(parts) == 1:
        return _dev32(parts[0], dev)
    if all(not isinstance(p, torch.Tensor) for p in parts):
        return _dev32(np.concatenate([np.asarray(p, np.float32) for p in parts]), dev)
    return torch.cat([_dev32(p, dev) for p in parts])


def _rows(t, name):
    """(tensor, row stride in floats) of a [N, A, B] float32 tensor: a view whose frames are packed [A, B] blocks (joints[:, :14] of
    a [N, 25, 3] prediction) is read in place, anything else is made contiguous."""
    if t.dim() != 3:
        raise _lib.HDError('%s must be [N, A, B], got %s' % (name, tuple(t.shape)))
    width = t.shape[1] * t.shape[2]
    if t.stride(2) != 1 or t.stride(1) != t.shape[2] or (t.shape[0] > 1 and t.stride(0) < width):
        t = t.contiguous()
    return t, (t.stride(0) if t.shape[0] > 1 else width)


class Evaluator(object):
    """Device scoring of HMMR predictions.  `smpl_consts` (a human_dynamics_b200.smpl.SMPLConstants) is needed for the meshes only.

    `mesh_chunk` frames are skinned at a time for mesh_posed (2 x mesh_chunk x V x 3 floats of workspace); the result does not depend
    on it."""

    def __init__(self, smpl_consts=None, mesh_chunk=1024, device=None):
        if not 1 <= int(mesh_chunk) <= MAX_MESH_CHUNK:
            raise ValueError('mesh_chunk must be in [1, %d]' % MAX_MESH_CHUNK)
        self.smpl = smpl_consts
        self.mesh_chunk = int(mesh_chunk)
        if device is not None:
            self.device = torch.device(device)
        elif smpl_consts is not None:
            self.device = smpl_consts.device
        else:
            if not torch.cuda.is_available():
                raise _lib.HDError('Evaluator needs a CUDA device (no CPU fallback exists)')
            self.device = torch.device('cuda', torch.cuda.current_device())

    # ------------------------------------------------------------------------------------------------------------------ public
    def errors(self, kps_gt, kps_pred, joints_gt=None, joints_pred=None, poses_gt=None, poses_pred=None, shape_gt=None,
               shapes_pred=None, img_size=224, has_3d=False, min_visible=6, compute_mesh=False):
        """compute_errors_batched (eval.py:114-193) for one tube."""
        tube = dict(kps_gt=kps_gt, kps_pred=kps_pred, joints_gt=joints_gt, joints_pred=joints_pred, poses_gt=poses_gt,
                    poses_pred=poses_pred, shape_gt=shape_gt, shapes_pred=shapes_pred)
        return self.errors_many([tube], img_size=img_size, has_3d=has_3d, min_visible=min_visible, compute_mesh=compute_mesh)[0]

    def errors_many(self, tubes, img_size=224, has_3d=False, min_visible=6, compute_mesh=False):
        """tubes: a list of dicts with the keyword arguments of `errors` (kps_gt, kps_pred, joints_pred and, with has_3d, joints_gt;
        with compute_mesh also poses_gt [n,72], poses_pred [n,24,3,3], shape_gt [10], shapes_pred [n,10]).  One pass over all of
        them; returns the list of per-tube error dicts, each what compute_errors_batched returns for that tube alone."""
        staged = self._stage(tubes, has_3d, compute_mesh)
        out = self._launch(staged, img_size, min_visible)
        return self._split(staged, out.cpu().numpy(), has_3d, compute_mesh)

    # ------------------------------------------------------------------------------------------------------------------ stages
    def _stage(self, tubes, has_3d, compute_mesh):
        """Validate and upload (the only host -> device traffic of a pass)."""
        if not tubes:
            raise ValueError('errors_many needs at least one tube')
        if compute_mesh and has_3d and self.smpl is None:
            raise ValueError('compute_mesh needs the SMPL constants: Evaluator(smpl_consts)')
        lens = []
        for i, t in enumerate(tubes):
            n = len(t['kps_gt'])
            if len(t['kps_pred']) != n or t.get('joints_pred') is None or len(t['joints_pred']) != n:
                raise ValueError('tube %d: kps_gt, kps_pred and joints_pred must have the same number of frames' % i)
            if has_3d and (t.get('joints_gt') is None or len(t['joints_gt']) != n):
                raise ValueError('tube %d: has_3d needs joints_gt with one row per frame' % i)
            lens.append(n)
        dev = self.device
        s = {'lens': lens, 'starts': np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)}
        s['N'] = N = int(s['starts'][-1])
        s['kps_gt'] = _cat([t['kps_gt'] for t in tubes], dev)
        s['kps_pred'] = _cat([t['kps_pred'] for t in tubes], dev)
        s['joints_pred'] = _cat([t['joints_pred'] for t in tubes], dev)
        s['joints_gt'] = _cat([t['joints_gt'] for t in tubes], dev) if has_3d else None
        K = s['kps_gt'].shape[1] if s['kps_gt'].dim() > 1 else 0
        J = s['joints_pred'].shape[1] if s['joints_pred'].dim() > 1 else 0
        if s['kps_gt'].dim() != 3 or s['kps_gt'].shape[2] != 3 or tuple(s['kps_pred'].shape[1:]) != (K, 2):
            raise ValueError('kps_gt must be [n,K,3] and kps_pred [n,K,2]')
        if s['joints_pred'].dim() != 3 or s['joints_pred'].shape[2] != 3 or \
                (has_3d and tuple(s['joints_gt'].shape[1:]) != (J, 3)):
            raise ValueError('joints_pred (and joints_gt) must be [n,J,3]')
        s['K'], s['J'] = K, J
        s['seq_start'] = torch.from_numpy(s['starts'].astype(np.int32)).to(dev)
        if compute_mesh and has_3d:
            for i, t in enumerate(tubes):
                if t.get('poses_gt') is None or t.get('poses_pred') is None or t.get('shape_gt') is None or t.get('shapes_pred') is None:
                    raise ValueError('tube %d: compute_mesh needs poses_gt, poses_pred, shape_gt and shapes_pred' % i)
            s['beta_gt'] = _cat([np.tile(np.asarray(t['shape_gt'], np.float32).reshape(1, 10), (n, 1))
                                 if not isinstance(t['shape_gt'], torch.Tensor) else t['shape_gt'].reshape(1, 10).expand(n, 10)
                                 for t, n in zip(tubes, lens)], dev).reshape(N, 10).contiguous()
            s['beta_pred'] = _cat([t['shapes_pred'] for t in tubes], dev).reshape(N, 10).contiguous()
            s['theta_gt'] = _cat([t['poses_gt'] for t in tubes], dev).reshape(N, 72).contiguous()
            s['Rs_pred'] = _cat([t['poses_pred'] for t in tubes], dev).reshape(N, 216).contiguous()
        return s

    def _launch(self, s, img_size, min_visible):
        """Device work of a pass, no host synchronisation: returns the device result [N, COLS (+2 with meshes)] float64."""
        dev, N, K, J = self.device, s['N'], s['K'], s['J']
        out = torch.empty((N, COLS), dtype=torch.float64, device=dev)
        kg, kg_ld = _rows(s['kps_gt'], 'kps_gt')
        kp, kp_ld = _rows(s['kps_pred'], 'kps_pred')
        jp, jp_ld = _rows(s['joints_pred'], 'joints_pred')
        a = _lib.EvalFramesArgs()
        a.N, a.n_seq, a.seq_start, a.K, a.J = N, len(s['lens']), s['seq_start'].data_ptr(), K, J
        a.kps_gt, a.kps_gt_ld = kg.data_ptr(), kg_ld
        a.kps_pred, a.kps_pred_ld = kp.data_ptr(), kp_ld
        a.joints_pred, a.joints_pred_ld = jp.data_ptr(), jp_ld
        if s['joints_gt'] is not None:
            jg, jg_ld = _rows(s['joints_gt'], 'joints_gt')
            a.joints_gt, a.joints_gt_ld = jg.data_ptr(), jg_ld
        a.img_size, a.min_visible, a.out = float(img_size), int(min_visible), out.data_ptr()
        st = current_stream()
        check(lib.hd_eval_frames(C.byref(a), st), 'hd_eval_frames')
        if 'beta_gt' not in s:
            return out
        tpose = torch.empty(N, dtype=torch.float64, device=dev)
        posed = torch.empty(N, dtype=torch.float64, device=dev)
        sm = self.smpl
        check(lib.hd_eval_mesh_tpose(C.byref(sm.c), fptr(s['beta_gt']), 10, fptr(s['beta_pred']), 10, N, dptr(tpose), st),
              'hd_eval_mesh_tpose')
        theta_pred = torch.empty((N, 72), dtype=torch.float32, device=dev)
        check(lib.hd_rot2aa(fptr(s['Rs_pred']), fptr(theta_pred), N * 24, st), 'hd_rot2aa')
        V, ch = sm.num_verts, max(1, min(self.mesh_chunk, N))
        va = torch.empty((ch, V, 3), dtype=torch.float32, device=dev)
        vb = torch.empty((ch, V, 3), dtype=torch.float32, device=dev)
        ws = torch.empty(int(lib.hd_smpl_workspace_bytes(ch)), dtype=torch.uint8, device=dev)
        for c0 in range(0, N, ch):
            n = min(ch, N - c0)
            for beta, theta, verts in ((s['beta_gt'], s['theta_gt'], va), (s['beta_pred'], theta_pred, vb)):
                check(lib.hd_smpl_forward(C.byref(sm.c), fptr(beta[c0:]), 10, fptr(theta[c0:]), 72, n, fptr(verts), None, None, None,
                                          None, 0, None, 1, 0, dptr(ws), ws.numel(), st), 'hd_smpl_forward')
            check(lib.hd_eval_verts_error(fptr(va), 3 * V, fptr(vb), 3 * V, n, V, dptr(posed[c0:]), st), 'hd_eval_verts_error')
        return torch.cat([out, posed[:, None], tpose[:, None]], dim=1)

    @staticmethod
    def _split(s, res, has_3d, compute_mesh):
        """The per-tube dicts of compute_errors_batched from the fetched rows (eval.py:137-191: lists where the reference builds lists,
        arrays where it builds arrays, -1 for what it does not compute)."""
        out = []
        for a, n in zip(s['starts'][:-1], s['lens']):
            r = res[a:a + n]
            tri = max(n - 2, 0)
            e = {'accel': r[:tri, _lib.HD_EVAL_ACCEL].copy(),
                 'kp': list(r[:, _lib.HD_EVAL_KP]), 'kp_pa': list(r[:, _lib.HD_EVAL_KP_PA]), 'kp_pck': list(r[:, _lib.HD_EVAL_KP_PCK])}
            if has_3d:
                vis = r[:, _lib.HD_EVAL_VIS3D] != 0
                keep = vis[:tri] & vis[1:tri + 1] & vis[2:tri + 2]
                e.update({'accel_error': r[:tri, _lib.HD_EVAL_ACCEL_ERROR][keep],
                          'mesh_posed': r[vis, COLS] if compute_mesh else -1,
                          'mesh_tpose': r[vis, COLS + 1] if compute_mesh else -1,
                          'pose': -1,
                          'joints': list(r[vis, _lib.HD_EVAL_JOINTS]),
                          'joints_pa': list(r[vis, _lib.HD_EVAL_JOINTS_PA]),
                          'shape': -1})
            out.append(e)
        return out
