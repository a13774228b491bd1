"""Host side of the batched SMPL forward: packs the model constants once, then one C-ABI call per batch.

Mirrors `SMPL.__init__` / `SMPL.__call__` of the reference (src/tf_smpl/batch_smpl.py:27-162); the
reference-named class lives in src/tf_smpl/batch_smpl.py and delegates here.
"""
from __future__ import annotations

import ctypes as C
import pickle

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _lib
from ._lib import lib, check, fptr, dptr, current_stream


def _dense(m):
    m = m.r if (hasattr(m, 'r') and not isinstance(m, np.ndarray) and not hasattr(m, 'todense')) else m   # undo_chumpy, batch_smpl.py:22-23
    return np.asarray(m.todense()) if hasattr(m, 'todense') else np.asarray(m)


class _ChStub(object):
    """Stand-in for chumpy objects inside the official SMPL pickles (chumpy is not a dependency here).

    chumpy.Ch pickles as (class, state-dict) with the wrapped ndarray under 'x'; the reference reads it through `.r`
    (`undo_chumpy`, batch_smpl.py:22-23).  Any other attribute of the state is kept but unused."""

    def __setstate__(self, state):
        self.__dict__.update(state if isinstance(state, dict) else {'x': state})

    @property
    def r(self):
        return np.asarray(self.__dict__['x'])


class _SMPLUnpickler(pickle.Unpickler):
    """pickle.Unpickler that maps every class from the `chumpy` package to `_ChStub` (scipy.sparse / numpy load normally)."""

    def find_class(self, module, name):
        if module == 'chumpy' or module.startswith('chumpy.'):
            return _ChStub
        return super().find_class(module, name)


def load_smpl_model(pkl_path_or_dict):
    """The un-pickled SMPL model dict (batch_smpl.py:31-32: `pickle.load(f, encoding='latin1')`), without needing chumpy."""
    if isinstance(pkl_path_or_dict, dict):
        return pkl_path_or_dict
    with open(pkl_path_or_dict, 'rb') as f:
        return _SMPLUnpickler(f, encoding='latin1').load()


class SMPLConstants(object):
    """Device-resident SMPL constants in the layout the kernels want (hd_smpl_consts)."""

    def __init__(self, model, joint_type='cocoplus', device=None, tc=True):
        if joint_type not in ('cocoplus', 'lsp'):
            raise ValueError('BAD!! Unknown joint type: %s, it must be either "cocoplus" or "lsp"' % joint_type)
        dd = load_smpl_model(model)
        dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self.device = dev
        v_template = _dense(dd['v_template']).astype(np.float64)               # (V,3)
        V = v_template.shape[0]
        shapedirs = _dense(dd['shapedirs']).astype(np.float64)                 # (V,3,10)
        nb = shapedirs.shape[-1]
        posedirs = _dense(dd['posedirs']).astype(np.float64)                   # (V,3,207)
        if nb != 10 or posedirs.shape[-1] != 207:
            raise ValueError('expected 10 betas and 207 pose-blend bases, got %d / %d' % (nb, posedirs.shape[-1]))
        Jreg = _dense(dd['J_regressor']).astype(np.float64)                    # (24,V)
        if Jreg.shape != (24, V):
            raise ValueError('J_regressor must be (24, V)')
        weights = _dense(dd['weights']).astype(np.float64)                     # (V,24)
        kreg = _dense(dd['cocoplus_regressor']).astype(np.float64)             # (K,V)
        if joint_type == 'lsp':
            kreg = kreg[:14]                                                   # batch_smpl.py:81-82
        parents = np.asarray(dd['kintree_table'])[0].astype(np.int64).astype(np.int32)   # uint32(-1) -> -1, :66
        self.parents = parents.copy()
        self.num_verts = V
        self.num_kps = kreg.shape[0]
        self.size = [V, 3]
        self.num_betas = nb

        sd = shapedirs.reshape(-1, nb).T                                       # (10, V*3)   :45-48
        pd = posedirs.reshape(-1, 207).T                                       # (207, V*3)  :60-63
        dirs = np.concatenate([sd, pd], axis=0).astype(np.float32)
        # J = (beta.shapedirs + v_template).J_regressor is linear in beta: precompose (float64) once.
        J_template = (Jreg @ v_template).astype(np.float32)                    # (24,3)
        J_shapedirs = np.einsum('jv,vcb->bjc', Jreg, shapedirs).reshape(nb, 72).astype(np.float32)

        nnz = int(max(1, (weights != 0).sum(axis=1).max()))
        if nnz <= 4:
            nnz = 4
        elif nnz < 24:
            nnz = min(24, (nnz + 3) // 4 * 4)
        mask = weights != 0
        order = np.argsort(~mask, axis=1, kind='stable')[:, :nnz]              # non-zero joints first, ascending
        lbs_w = np.take_along_axis(weights, order, 1)
        lbs_idx = np.where(lbs_w != 0, order, 0)

        kp_ptr = [0]
        kp_vidx, kp_w = [], []
        for k in range(kreg.shape[0]):
            nzv = np.nonzero(kreg[k])[0]
            kp_vidx.append(nzv)
            kp_w.append(kreg[k, nzv])
            kp_ptr.append(kp_ptr[-1] + len(nzv))
        kp_vidx = np.concatenate(kp_vidx) if kp_vidx else np.zeros(0, np.int64)
        kp_w = np.concatenate(kp_w) if kp_w else np.zeros(0)

        def f32(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)

        def i32(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)

        self.v_template = f32(v_template.reshape(-1))
        self.dirs = f32(dirs)
        self.J_template = f32(J_template.reshape(-1))
        self.J_shapedirs = f32(J_shapedirs)
        self.lbs_idx = i32(lbs_idx)
        self.lbs_w = f32(lbs_w)
        self.kp_ptr = i32(np.asarray(kp_ptr))
        self.kp_vidx = i32(kp_vidx if len(kp_vidx) else np.zeros(1))
        self.kp_w = f32(kp_w if len(kp_w) else np.zeros(1))
        self.lbs_nnz = nnz

        c = _lib.SmplConsts()
        c.num_verts, c.num_kps, c.lbs_nnz, c.kp_nnz_total = V, self.num_kps, nnz, int(kp_ptr[-1])
        c.v_template = self.v_template.data_ptr()
        c.dirs = self.dirs.data_ptr()
        c.J_template = self.J_template.data_ptr()
        c.J_shapedirs = self.J_shapedirs.data_ptr()
        c.lbs_idx = self.lbs_idx.data_ptr()
        c.lbs_w = self.lbs_w.data_ptr()
        c.kp_ptr = self.kp_ptr.data_ptr()
        c.kp_vidx = self.kp_vidx.data_ptr()
        c.kp_w = self.kp_w.data_ptr()
        for i in range(24):
            c.parents[i] = int(parents[i])
        self.c = c
        self._ws = None
        # Tensor-core blend for large batches: v_posed = [beta | R-I] . dirs + v_template as one [N,256] x [256, V*3] GEMM
        # (fp16 head/remainder split, FP32-class), then HBM-shaped skinning.  Small batches use the fused SIMT kernel.
        self.tc_min_batch = 256
        self.blend = None
        self._tc_bufs = {}
        if tc:
            from .nets import PackedConv, sync_packing
            self.vp_ld = (V * 3 + 3) // 4 * 4
            wb = np.zeros((256, self.vp_ld), np.float32)
            wb[:217, :V * 3] = dirs
            bias = np.zeros(self.vp_ld, np.float32)
            bias[:V * 3] = v_template.reshape(-1)
            with torch.cuda.device(dev):                       # packed on dev's current stream
                self.blend = PackedConv(wb, dev, post_shift=bias, tc='tc3h')
                sync_packing(dev)
            # dense skinning weights as the A operand of the tensor-core skinning GEMM: [roundup128(V), 32] fp16 head + unscaled remainder
            wd = np.zeros(((V + 127) // 128 * 128, 32), np.float32)
            wd[:V, :24] = weights
            w_hi = wd.astype(np.float16)
            self.w_hi = torch.from_numpy(w_hi).to(dev)
            self.w_lo = torch.from_numpy((wd - w_hi.astype(np.float32)).astype(np.float16)).to(dev)
        self.lbs_tc = bool(tc) and (V * 3 * 4) % 8 == 0
        self.lbs_tc_min_batch = 2112                       # 132 SMs x 16 poses
        # host copies for the backward's extra arrays, packed and uploaded on the first backward call (grad_state)
        self._grad_src = (weights, kreg, dirs)
        self._grad = None
        self._bw_bufs = {}

    def workspace(self, N):
        need = int(lib.hd_smpl_workspace_bytes(N))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    def forward(self, beta, theta, cam=None, want_joints=True, want_Rs=True, want_Jtr=True, out=None, slot=(1, 0)):
        """beta (N,10)-view, theta (N,72)-view, cam (N,3)-view: float32 CUDA, unit inner stride, any row stride.

        `out` may hold pre-allocated output tensors; with slot=(D, d) pose n is written to row n*D+d of each
        of them (they must then have N*D leading rows) -- the in-place [B,T,D,...] stacking of tester.py:252.
        Returns dict(verts, joints, Rs, Jtr, kps).
        """
        mul, off = slot
        for name, t, w in (('beta', beta, 10), ('theta', theta, 72)) + ((('cam', cam, 3),) if cam is not None else ()):
            if not t.is_cuda or t.dtype != torch.float32:
                raise _lib.HDError('SMPL %s must be a float32 CUDA tensor (no CPU fallback exists)' % name)
            if t.dim() != 2 or t.shape[1] != w or t.stride(1) != 1:
                raise _lib.HDError('SMPL %s must be (N,%d) with unit inner stride, got %s' % (name, w, tuple(t.shape)))
        N = beta.shape[0]
        if theta.shape[0] != N or (cam is not None and cam.shape[0] != N):
            raise _lib.HDError('SMPL batch mismatch')
        V, K = self.num_verts, self.num_kps
        dev = beta.device
        o = out or {}
        verts = o.get('verts') if 'verts' in o else torch.empty((N * mul, V, 3), dtype=torch.float32, device=dev)
        joints = o.get('joints') if 'joints' in o else (torch.empty((N * mul, K, 3), dtype=torch.float32, device=dev) if want_joints else None)
        Rs = o.get('Rs') if 'Rs' in o else (torch.empty((N * mul, 24, 3, 3), dtype=torch.float32, device=dev) if want_Rs else None)
        Jtr = o.get('Jtr') if 'Jtr' in o else (torch.empty((N * mul, 24, 3), dtype=torch.float32, device=dev) if want_Jtr else None)
        kps = None
        if cam is not None:
            kps = o.get('kps') if 'kps' in o else torch.empty((N * mul, K, 2), dtype=torch.float32, device=dev)
        if N >= self.tc_min_batch and self.blend is not None and self.blend.tc:
            self._forward_tc(beta, theta, cam, N, verts, joints, Rs, Jtr, kps, int(mul), int(off))
        elif N > 0:
            ws = self.workspace(N)
            rc = lib.hd_smpl_forward(C.byref(self.c), fptr(beta), beta.stride(0), fptr(theta), theta.stride(0), N,
                                     fptr(verts), fptr(joints), fptr(Rs), fptr(Jtr),
                                     fptr(cam) if cam is not None else None, cam.stride(0) if cam is not None else 0,
                                     fptr(kps) if kps is not None else None, int(mul), int(off),
                                     dptr(ws), ws.numel(), current_stream())
            check(rc, 'hd_smpl_forward')
        return {'verts': verts, 'joints': joints, 'Rs': Rs, 'Jtr': Jtr, 'kps': kps}

    def _forward_tc(self, beta, theta, cam, N, verts, joints, Rs, Jtr, kps, mul, off):
        """pose -> tensor-core blend GEMM -> skinning -> keypoints (hd_smpl_pose / hd_conv_gemm / hd_smpl_lbs / hd_smpl_joints)."""
        dev = beta.device
        if N not in self._tc_bufs:
            while len(self._tc_bufs) >= 3:                     # bounded cache: an entry holds N * 83 KB of v_posed
                self._tc_bufs.pop(next(iter(self._tc_bufs)))
            f32 = dict(dtype=torch.float32, device=dev)
            coef = (torch.empty((N, 256), dtype=torch.float16, device=dev), torch.empty((N, 256), dtype=torch.float16, device=dev))
            vpos = torch.empty((N, self.vp_ld), **f32)
            a12 = torch.empty((N, 288), **f32)
            rsw = torch.empty((N, 216), **f32)
            # tensor-core skinning walks 16-pose batches, one CTA per batch at a time: below one batch per SM the CUDA-core kernel (one
            # CTA per 16 poses x 128 vertices) fills the chip better
            a12t = (torch.empty((N, 12, 32), dtype=torch.float16, device=dev), torch.empty((N, 12, 32), dtype=torch.float16, device=dev)) \
                if (self.lbs_tc and N >= self.lbs_tc_min_batch) else None
            # operand rows arrive pre-split from the pose kernel: cp.async producer (K = 256)
            op = self.blend.bind(None, N, 1, 1, vpos, inp_split=coef, impl='tc3h')
            self._tc_bufs[N] = (coef, vpos, a12, rsw, op, a12t)
        coef, vpos, a12, rsw, op, a12t = self._tc_bufs[N]
        st = current_stream()
        check(lib.hd_smpl_pose(C.byref(self.c), fptr(beta), beta.stride(0), fptr(theta), theta.stride(0), N, fptr(Rs), fptr(Jtr),
                               fptr(a12), None, 256, C.c_void_p(coef[0].data_ptr()), C.c_void_p(coef[1].data_ptr()),
                               C.c_void_p(a12t[0].data_ptr()) if a12t else None, C.c_void_p(a12t[1].data_ptr()) if a12t else None, mul, off,
                               dptr(rsw), rsw.numel() * 4, st), 'hd_smpl_pose')
        op.run(st)
        if a12t is not None:       # T = W . A on the tensor cores, applied from registers (smpl_lbs_tc.cu)
            check(lib.hd_smpl_lbs_tc(C.c_void_p(self.w_hi.data_ptr()), C.c_void_p(self.w_lo.data_ptr()), C.c_void_p(a12t[0].data_ptr()),
                                     C.c_void_p(a12t[1].data_ptr()), fptr(vpos), self.vp_ld, fptr(verts), N, self.num_verts, mul, off, st),
                  'hd_smpl_lbs_tc')
        else:
            check(lib.hd_smpl_lbs(C.byref(self.c), fptr(vpos), self.vp_ld, fptr(a12), fptr(verts), N, mul, off, st), 'hd_smpl_lbs')
        if (joints is not None or kps is not None) and self.num_kps > 0:
            check(lib.hd_smpl_joints(C.byref(self.c), fptr(verts), fptr(cam) if cam is not None else None,
                                     cam.stride(0) if cam is not None else 0, fptr(joints), fptr(kps) if kps is not None else None,
                                     N, mul, off, st), 'hd_smpl_joints')


    # ---------------------------------------------------------------- backward (smpl_grad.cu) ----------------------------------------

    def grad_state(self):
        """Device arrays of hd_smpl_grad_consts and the packed dirs^T of the dc GEMM, built once on first use."""
        if self._grad is None:
            if self.blend is None:
                raise _lib.HDError('the SMPL backward recomputes v_posed on the tensor-core blend: build SMPLConstants with tc=True')
            from .nets import PackedConv, sync_packing
            weights, kreg, dirs = self._grad_src
            V, dev = self.num_verts, self.device
            pk = pack_grad_arrays(weights, kreg)
            keep = {k: torch.from_numpy(np.ascontiguousarray(v if len(v) else np.zeros(1, v.dtype))).to(dev) for k, v in pk.items()}
            g = _lib.SmplGradConsts()
            g.num_verts, g.num_kps = V, self.num_kps
            g.tile_verts, g.num_tiles = _lib.SMPL_GRAD_TILE, (V + _lib.SMPL_GRAD_TILE - 1) // _lib.SMPL_GRAD_TILE
            for k in ('kpv_ptr', 'kpv_kidx', 'kpv_w', 'lbt_ptr', 'lbt_v', 'lbt_w'):
                setattr(g, k, keep[k].data_ptr())
            # dc = dv_posed . dirs^T: K = vp_ld (zero rows past 3V), Cout = 224 (zero columns past 217), 3xTF32 on the fp32 operand.
            # Gradients carry the loss's arbitrary scale, so they never go through the fp16 head / remainder split.
            wt = np.zeros((self.vp_ld, _lib.SMPL_GRAD_CLD), np.float32)
            wt[:V * 3, :217] = dirs.T
            with torch.cuda.device(dev):
                gemm = PackedConv(wt, dev, tc='tc3')
                sync_packing(dev)
            if gemm.tc != 'tf32':
                raise _lib.HDError('dirs^T did not get the TF32 tensor-core packing (vp_ld %% 32 != 0?)')
            self._grad = (g, keep, gemm)
        return self._grad

    def backward_workspace(self, N):
        """Per-N buffers of one backward (hd_smpl_backward_workspace_bytes layout) plus the two bound GEMMs; bounded cache."""
        if N in self._bw_bufs:
            return self._bw_bufs[N]
        g, keep, gemm = self.grad_state()
        while len(self._bw_bufs) >= 2:
            self._bw_bufs.pop(next(iter(self._bw_bufs)))
        dev = self.device
        ws = torch.empty(int(lib.hd_smpl_backward_workspace_bytes(N, self.num_verts)), dtype=torch.uint8, device=dev)
        views, off = {}, 0
        for name, cols, dt in (('A12', 288, torch.float32), ('dA12', 288, torch.float32), ('dc', _lib.SMPL_GRAD_CLD, torch.float32),
                               ('rs', 216, torch.float32), ('coef_hi', 256, torch.float16), ('coef_lo', 256, torch.float16),
                               ('vpos', self.vp_ld, torch.float32), ('dvpos', self.vp_ld, torch.float32)):
            nb = N * cols * (4 if dt == torch.float32 else 2)
            views[name] = ws[off:off + nb].view(dt).view(N, cols)
            off += (nb + 255) // 256 * 256
        assert off == ws.numel()
        blend = self.blend.bind(None, N, 1, 1, views['vpos'], inp_split=(views['coef_hi'], views['coef_lo']), impl='tc3h')
        dc = gemm.bind(views['dvpos'], N, 1, 1, views['dc'], impl='tc3')
        if dc.d.impl != _lib.HD_IMPL_TC_3XTF32:
            raise _lib.HDError('the dc GEMM must run on the 3xTF32 tensor-core kernel')
        self._bw_bufs[N] = (ws, views, blend, dc)
        return self._bw_bufs[N]

    def backward(self, beta, theta, dverts=None, djoints=None, dRs=None, dJtr=None, dbeta=None, dtheta=None):
        """Gradients of (verts, joints, Rs, Jtr) = forward(beta, theta) w.r.t. beta (N,10) and theta (N,72).

        beta / theta: the forward's inputs (float32 CUDA, unit inner stride, any row stride).  d*: upstream gradients of the outputs,
        dense, or None for zero.  dbeta / dtheta: optional output views (unit inner stride, any row stride), else allocated.
        v_posed is recomputed (hd_smpl_pose + the tensor-core blend), not saved by the forward."""
        for name, t, w in (('beta', beta, 10), ('theta', theta, 72)):
            if not t.is_cuda or t.dtype != torch.float32:
                raise _lib.HDError('SMPL %s must be a float32 CUDA tensor (no CPU fallback exists)' % name)
            if t.dim() != 2 or t.shape[1] != w or t.stride(1) != 1:
                raise _lib.HDError('SMPL %s must be (N,%d) with unit inner stride, got %s' % (name, w, tuple(t.shape)))
        N, V, K = beta.shape[0], self.num_verts, self.num_kps
        if theta.shape[0] != N:
            raise _lib.HDError('SMPL batch mismatch')
        dev = beta.device
        dbeta = torch.empty((N, 10), dtype=torch.float32, device=dev) if dbeta is None else dbeta
        dtheta = torch.empty((N, 72), dtype=torch.float32, device=dev) if dtheta is None else dtheta
        if N == 0:
            return dbeta, dtheta

        def dense(t, shape, name):
            if t is None:
                return None
            if not t.is_cuda or t.dtype != torch.float32 or tuple(t.shape) != shape:
                raise _lib.HDError('SMPL gradient %s must be a float32 CUDA tensor of shape %s' % (name, shape))
            return t.contiguous()
        dverts = dense(dverts, (N, V, 3), 'dverts')
        djoints = dense(djoints, (N, K, 3), 'djoints')
        dRs = dense(dRs, (N, 24, 3, 3), 'dRs')
        dJtr = dense(dJtr, (N, 24, 3), 'dJtr')
        st = current_stream()
        mesh = dverts is not None or (djoints is not None and K > 0)
        dA12, dc = None, None
        if mesh:
            g, _, _ = self.grad_state()
            ws, b, blend, dcop = self.backward_workspace(N)
            if dverts is None:
                dverts = torch.zeros((N, V, 3), dtype=torch.float32, device=dev)
            check(lib.hd_smpl_pose(C.byref(self.c), fptr(beta), beta.stride(0), fptr(theta), theta.stride(0), N, None, None,
                                   fptr(b['A12']), None, 256, dptr(b['coef_hi']), dptr(b['coef_lo']), None, None, 1, 0,
                                   dptr(b['rs']), b['rs'].numel() * 4, st), 'hd_smpl_pose')
            blend.run(st)
            check(lib.hd_smpl_lbs_backward(C.byref(self.c), C.byref(g), fptr(b['vpos']), self.vp_ld, fptr(b['A12']), fptr(dverts),
                                           fptr(djoints) if (djoints is not None and K > 0) else None, fptr(b['dvpos']),
                                           fptr(b['dA12']), N, st), 'hd_smpl_lbs_backward')
            dcop.run(st)
            dA12, dc = b['dA12'], b['dc']
        check(lib.hd_smpl_pose_backward(C.byref(self.c), fptr(beta), beta.stride(0), fptr(theta), theta.stride(0), N,
                                        fptr(dA12) if dA12 is not None else None, fptr(dc) if dc is not None else None,
                                        _lib.SMPL_GRAD_CLD, fptr(dRs) if dRs is not None else None,
                                        fptr(dJtr) if dJtr is not None else None, fptr(dbeta), dbeta.stride(0), fptr(dtheta),
                                        dtheta.stride(0), st), 'hd_smpl_pose_backward')
        return dbeta, dtheta


def pack_grad_arrays(weights, kp_regressor, tile=None):
    """Host packing of the backward's extra SMPL arrays (hd_smpl_grad_consts), from the dense float64 skinning weights [V,24] and
    keypoint regressor [K,V]:
      kpv_ptr / kpv_kidx / kpv_w: the regressor vertex-major (CSR over vertices, keypoint ids ascending);
      lbt_ptr / lbt_v / lbt_w:    the non-zero skinning weights joint-major inside each tile of `tile` vertices."""
    tile = _lib.SMPL_GRAD_TILE if tile is None else tile
    weights = np.asarray(weights, np.float64)
    kreg = np.asarray(kp_regressor, np.float64)
    V = weights.shape[0]
    kv, kk = np.nonzero(kreg.T)                                            # row-major over (v, k): vertices, then keypoints ascending
    kpv_ptr = np.zeros(V + 1, np.int64)
    np.add.at(kpv_ptr, kv + 1, 1)
    ptr, vv, ww = [0], [], []
    for t in range((V + tile - 1) // tile):
        blk = weights[t * tile:(t + 1) * tile]
        for k in range(weights.shape[1]):
            nz = np.nonzero(blk[:, k])[0]
            vv.append(nz + t * tile)
            ww.append(blk[nz, k])
            ptr.append(ptr[-1] + len(nz))
    return {'kpv_ptr': np.cumsum(kpv_ptr).astype(np.int32), 'kpv_kidx': kk.astype(np.int32),
            'kpv_w': kreg.T[kv, kk].astype(np.float32),
            'lbt_ptr': np.asarray(ptr, np.int32), 'lbt_v': np.concatenate(vv).astype(np.int32),
            'lbt_w': np.concatenate(ww).astype(np.float32)}


def _noop():
    pass


def batch_rodrigues(theta):
    """theta (M,3) float32 CUDA -> (M,3,3).  src/tf_smpl/batch_lbs.py:42-60."""
    if not theta.is_cuda:
        raise _lib.HDError('batch_rodrigues: CUDA tensor required (no CPU fallback exists)')
    theta = theta.contiguous().float()
    if theta.dim() != 2 or theta.shape[1] != 3:
        raise _lib.HDError('batch_rodrigues: theta must be (M,3)')
    M = theta.shape[0]
    R = torch.empty((M, 3, 3), dtype=torch.float32, device=theta.device)
    check(lib.hd_rodrigues(fptr(theta), fptr(R), M, current_stream()), 'hd_rodrigues')
    return R


def batch_rot2aa(Rs):
    """Rs (B,3,3) float32 CUDA -> axis-angle (B,3).  src/tf_smpl/batch_lbs.py:63-105."""
    if not Rs.is_cuda:
        raise _lib.HDError('batch_rot2aa: CUDA tensor required (no CPU fallback exists)')
    Rs = Rs.contiguous().float()
    if Rs.dim() != 3 or tuple(Rs.shape[1:]) != (3, 3):
        raise _lib.HDError('batch_rot2aa: Rs must be (B,3,3)')
    aa = torch.empty((Rs.shape[0], 3), dtype=torch.float32, device=Rs.device)
    check(lib.hd_rot2aa(fptr(Rs), fptr(aa), Rs.shape[0], current_stream()), 'hd_rot2aa')
    return aa


def batch_global_rigid_transformation(Rs, Js, parent, rotate_base=False):
    """Rs (N,24,3,3), Js (N,24,3), parent int[24] -> (new_J (N,24,3), A (N,24,4,4)).  batch_lbs.py:133-194."""
    if not (Rs.is_cuda and Js.is_cuda):
        raise _lib.HDError('batch_global_rigid_transformation: CUDA tensors required (no CPU fallback exists)')
    Rs = Rs.contiguous().float()
    Js = Js.contiguous().float()
    N = Rs.shape[0]
    if tuple(Rs.shape[1:]) != (24, 3, 3) or tuple(Js.shape) != (N, 24, 3):
        raise _lib.HDError('batch_global_rigid_transformation: expected Rs (N,24,3,3), Js (N,24,3)')
    par = (C.c_int * 24)(*[(-1 if (int(p) < 0 or int(p) >= 2 ** 31) else int(p)) for p in np.asarray(parent).tolist()])
    new_J = torch.empty((N, 24, 3), dtype=torch.float32, device=Rs.device)
    A = torch.empty((N, 24, 4, 4), dtype=torch.float32, device=Rs.device)
    check(lib.hd_global_rigid(fptr(Rs), fptr(Js), par, fptr(new_J), fptr(A), N, int(bool(rotate_base)), current_stream()),
          'hd_global_rigid')
    return new_J, A


def batch_orth_proj_idrot(X, camera):
    """X (N,P,3), camera (N,3) -> (N,P,2).  src/tf_smpl/projection.py:16-29."""
    if not (X.is_cuda and camera.is_cuda):
        raise _lib.HDError('batch_orth_proj_idrot: CUDA tensors required (no CPU fallback exists)')
    X = X.contiguous().float()
    camera = camera.reshape(-1, 3).contiguous().float()
    N, P = X.shape[0], X.shape[1]
    if X.shape[2] != 3 or camera.shape[0] != N:
        raise _lib.HDError('batch_orth_proj_idrot: expected X (N,P,3) and camera (N,3)')
    out = torch.empty((N, P, 2), dtype=torch.float32, device=X.device)
    check(lib.hd_orth_proj(fptr(X), fptr(camera), fptr(out), N, P, current_stream()), 'hd_orth_proj')
    return out


# ------------------------------------------------------------------------ autograd ---------------------------------------------------
# The four entry points below are what src/tf_smpl/* switch to when grad mode is on and an input requires grad.  Each node saves only
# its inputs (a few hundred bytes per pose for SMPL: v_posed is recomputed in the backward) and is once-differentiable: asking for
# a second derivative raises.

class SMPLFunction(torch.autograd.Function):
    """(beta (N,10), theta (N,72)) -> (verts, joints, Rs, Jtr) of SMPLConstants.forward, differentiable w.r.t. beta and theta."""

    @staticmethod
    def forward(ctx, consts, beta, theta):
        o = consts.forward(beta, theta)
        ctx.consts = consts
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(beta, theta)
        return o['verts'], o['joints'], o['Rs'], o['Jtr']

    @staticmethod
    @once_differentiable
    def backward(ctx, dverts, djoints, dRs, dJtr):
        beta, theta = ctx.saved_tensors
        dbeta, dtheta = ctx.consts.backward(beta, theta, dverts, djoints, dRs, dJtr)
        return None, (dbeta if ctx.needs_input_grad[1] else None), (dtheta if ctx.needs_input_grad[2] else None)


class RodriguesFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, theta):
        theta = theta.contiguous()
        ctx.save_for_backward(theta)
        return batch_rodrigues(theta)

    @staticmethod
    @once_differentiable
    def backward(ctx, dR):
        theta, = ctx.saved_tensors
        dR = dR.contiguous()
        dtheta = torch.empty_like(theta)
        check(lib.hd_rodrigues_backward(fptr(theta), fptr(dR), fptr(dtheta), theta.shape[0], current_stream()), 'hd_rodrigues_backward')
        return dtheta


class GlobalRigidFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, Rs, Js, parent, rotate_base):
        Rs, Js = Rs.contiguous(), Js.contiguous()
        new_J, A = batch_global_rigid_transformation(Rs, Js, parent, rotate_base)
        ctx.par = (C.c_int * 24)(*[(-1 if (int(p) < 0 or int(p) >= 2 ** 31) else int(p)) for p in np.asarray(parent).tolist()])
        ctx.rotate_base = int(bool(rotate_base))
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(Rs, Js)
        return new_J, A

    @staticmethod
    @once_differentiable
    def backward(ctx, dnew_J, dA):
        Rs, Js = ctx.saved_tensors
        N = Rs.shape[0]
        dnew_J = dnew_J.contiguous() if dnew_J is not None else None
        dA = dA.contiguous() if dA is not None else None
        dRs, dJs = torch.empty_like(Rs), torch.empty_like(Js)
        check(lib.hd_global_rigid_backward(fptr(Rs), fptr(Js), ctx.par, fptr(dnew_J) if dnew_J is not None else None,
                                           fptr(dA) if dA is not None else None, fptr(dRs), fptr(dJs), N, ctx.rotate_base,
                                           current_stream()), 'hd_global_rigid_backward')
        return dRs, dJs, None, None


class OrthProjFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X, camera):
        X = X.contiguous()
        cam = camera.reshape(-1, 3).contiguous()
        ctx.cam_shape = camera.shape
        ctx.save_for_backward(X, cam)
        return batch_orth_proj_idrot(X, cam)

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        X, cam = ctx.saved_tensors
        N, P = X.shape[0], X.shape[1]
        dout = dout.contiguous()
        dX, dcam = torch.empty_like(X), torch.empty_like(cam)
        check(lib.hd_orth_proj_backward(fptr(X), fptr(cam), fptr(dout), fptr(dX), fptr(dcam), N, P, current_stream()),
              'hd_orth_proj_backward')
        return dX, dcam.reshape(ctx.cam_shape)


def _needs_grad(*ts):
    return torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in ts)


def _cuda_f32(name, *ts):
    for t in ts:
        if not t.is_cuda:
            raise _lib.HDError('%s: CUDA tensors required (no CPU fallback exists)' % name)
        if t.dtype != torch.float32:
            raise _lib.HDError('%s: the differentiable path takes float32 tensors, got %s' % (name, t.dtype))
