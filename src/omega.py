"""Wrapper classes for predicted variables -- drop-in for the inference side of the reference's src/omega.py.

`OmegasPred` stores B x T x 85 predictions [cams 3 | poses 72 | shapes 10] and computes SMPL + keypoint
projection for all of them at once (omega.py:197-342).  Tensors are float32 CUDA torch.Tensors.
`OmegasGt` (omega.py:161-194) holds the ground truth the training losses read.
"""
import torch

from src.tf_smpl.projection import batch_orth_proj_idrot
from src.models import az_fc2_groupnorm as f_movie   # noqa: F401  (BASELINE.json's name for the temporal encoder)


class Omegas(object):
    """Superclass container (omega.py:16-158)."""

    def __init__(self, config, batch_size=None):
        self.config = config
        self.batch_size = batch_size if batch_size else config.batch_size
        self.length = 0
        dev = torch.device('cuda', torch.cuda.current_device())
        B, K = self.batch_size, self.config.num_kps

        def empty(*shape):
            return torch.empty(shape, dtype=torch.float32, device=dev)
        self.joints = empty(B, 0, K, 3)
        self.kps = empty(B, 0, K, 2)
        self.poses_aa = empty(B, 0, 24, 3)
        self.poses_rot = empty(B, 0, 24, 3, 3)
        self.shapes = empty(B, 0, 10)
        self.deltas_aa = empty(B, 0, 24, 3)
        self.deltas_rot = empty(B, 0, 24, 3, 3)

    def __len__(self):
        return self.length

    def get_joints(self, t=None):
        return self.joints if t is None else self.joints[:, t]

    def get_kps(self, t=None):
        return self.kps if t is None else self.kps[:, t]

    def get_poses_aa(self, t=None):
        return self.poses_aa if t is None else self.poses_aa[:, t]

    def get_poses_rot(self, t=None):
        return self.poses_rot if t is None else self.poses_rot[:, t]

    def get_deltas_aa(self, t=None):
        return self.deltas_aa if t is None else self.deltas_aa[:, t]

    def get_deltas_rot(self, t=None):
        return self.deltas_rot if t is None else self.deltas_rot[:, t]

    def get_shapes(self, t=None):
        return self.shapes if t is None else self.shapes[:, t]

    @staticmethod
    def gather(values, indices):
        """Gathers a subset over time (omega.py:144-158)."""
        idx = torch.as_tensor(indices, dtype=torch.long, device=values.device)
        return values.index_select(1, idx)


class OmegasGt(Omegas):
    """Ground-truth omegas (omega.py:161-194): poses_aa (B,T,24,3) or (B,T,72), shapes (B,10), joints (B,T,14,3), kps (B,T,K,3)."""

    def __init__(self, config, poses_aa, shapes, joints, kps, batch_size=None):
        from src.tf_smpl.batch_lbs import batch_rodrigues
        from src.ops import compute_deltas_batched
        super(OmegasGt, self).__init__(config, batch_size=batch_size)
        self.length = poses_aa.shape[1]
        self.poses_aa = poses_aa
        self.poses_rot = batch_rodrigues(poses_aa.reshape(-1, 3)).reshape(self.batch_size, -1, 24, 3, 3)
        self.shapes = shapes
        self.joints = joints
        self.kps = kps
        self.deltas_rot = compute_deltas_batched(self.poses_rot[:, :-1], self.poses_rot[:, 1:])

    def get_shapes(self, t=None):
        if t is None:
            return self.shapes.unsqueeze(1).expand(-1, self.length, -1)
        return self.shapes

    def get_deltas_aa(self, t=None):
        raise Exception('No axis-aligned deltas.')


class OmegasPred(Omegas):
    """Stores fields for predicted Omegas (omega.py:197-342).

    Unlike the reference, instances are NOT accumulated in a class-level list across Testers
    (omega.py:208,229 leaks them); `compute_all_smpl` takes the instances explicitly, or uses the
    per-owner registry passed as `registry`.
    """

    def __init__(self, config, smpl, use_optcam=False, vis_max_batch=2, vis_t_indices=None, batch_size=None,
                 is_training=True, registry=None):
        super(OmegasPred, self).__init__(config, batch_size)
        self.smpl = smpl
        dev = self.joints.device
        B = self.batch_size
        self.cams = torch.empty((B, 0, 3), dtype=torch.float32, device=dev)
        self.all_verts = torch.empty((0, 6890, 3), dtype=torch.float32, device=dev)
        self.verts = self.all_verts
        self.smpl_computed = False
        self.vis_max_batch = vis_max_batch
        self.vis_t_indices = vis_t_indices
        self.raw = torch.empty((B, 0, 85), dtype=torch.float32, device=dev)
        self.use_optcam = use_optcam
        self.is_training = is_training
        if registry is not None:
            registry.append(self)

    def update_instance_vars(self):
        """omega.py:231-235."""
        self.cams = self.raw[:, :, :3]
        self.poses_aa = self.raw[:, :, 3:3 + 24 * 3].reshape(self.batch_size, -1, 24, 3)
        self.shapes = self.raw[:, :, 3 + 24 * 3:85]
        self.length = self.raw.shape[1]

    def append_batched(self, omegas):
        """Appends multiple omegas (B x T x 85)  (omega.py:237-248)."""
        omegas = omegas.reshape(self.batch_size, -1, 85)
        self.raw = omegas if self.raw.shape[1] == 0 else torch.cat((self.raw, omegas), dim=1)
        self.update_instance_vars()
        self.smpl_computed = False

    def append(self, omega):
        """Appends an omega (B x 85)  (omega.py:250-261)."""
        self.append_batched(omega.reshape(self.batch_size, 1, 85))

    def compute_smpl(self):
        """Batch computation of vertices, joints, rotation matrices, and keypoints (omega.py:263-304)."""
        if self.smpl_computed:
            print('SMPL should only be computed once!')
        B, T = self.batch_size, self.length
        raw = self.raw.reshape(B * T, 85)
        if raw.stride(1) != 1 or raw.stride(0) != 85:
            raw = raw.contiguous()
        verts, joints, poses_rot = self.smpl(beta=raw[:, 75:85], theta=raw[:, 3:75], get_skin=True)
        K = self.config.num_kps
        self.joints = joints.reshape(B, T, K, 3)
        self.poses_rot = poses_rot.reshape(B, T, 24, 3, 3)
        if self.use_optcam and self.is_training:
            kps = joints[:, :, :2]
        else:
            kps = batch_orth_proj_idrot(joints, self.cams.reshape(B * T, 3))
        self.kps = kps.reshape(B, T, K, 2)
        self.all_verts = verts.reshape(B, T, -1, 3)[:self.vis_max_batch]
        self.verts = self.all_verts if self.vis_t_indices is None else Omegas.gather(self.all_verts, self.vis_t_indices)
        self.smpl_computed = True

    def get_cams(self, t=None):
        return self.cams if t is None else self.cams[:, t]

    def set_cams(self, cams):
        """Only used for opt_cam (omega.py:318-323)."""
        assert self.use_optcam
        self.cams = cams

    def get_all_verts(self):
        return self.all_verts

    def get_verts(self):
        return self.verts

    def get_raw(self):
        return self.raw

    @classmethod
    def compute_all_smpl(cls, omegas=()):
        """omega.py:338-342 (instances passed explicitly instead of the leaking class-level list)."""
        for omega in omegas:
            omega.compute_smpl()
