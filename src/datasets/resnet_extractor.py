"""Extracts image features from a sequence of images -- drop-in for src/datasets/resnet_extractor.py:13-98."""
import numpy as np
import torch

from human_dynamics_b200 import augment as _aug
from human_dynamics_b200 import runtime as _rt
from human_dynamics_b200.config import HMMRConfig
from human_dynamics_b200.engine import load_weights
from human_dynamics_b200.nets import PackedResNet, ResNetPlan


class FeatureExtractor(object):
    def __init__(self, model_path, img_size=224, batch_size=64, sess=None, impl='auto'):
        self.model_path = model_path
        self.img_size = img_size
        self.batch_size = batch_size
        w = load_weights(model_path)
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.packed = PackedResNet(w, self.device, tc=(impl if impl != 'simt' else False))
        self.plan = ResNetPlan(self.packed, batch_size, img_size, impl)
        self.phis = torch.empty((batch_size, self.packed.out_dim), dtype=torch.float32, device=self.device)

    def compute_phis(self, images):
        """images (B x H x W x 3) -> phis (B x 2048)   (resnet_extractor.py:58-72)."""
        if tuple(images.shape) != (self.batch_size, self.img_size, self.img_size, 3):
            raise ValueError('images must be %s' % ((self.batch_size, self.img_size, self.img_size, 3),))
        x = torch.as_tensor(np.ascontiguousarray(images, dtype=np.float32)).to(self.device)
        self.plan.run(x, self.phis)
        return self.phis.cpu().numpy()

    def compute_all_phis(self, all_images):
        """all_images (T x H x W x 3) -> (T x 2048); the last partial batch is zero-padded (:88-92)."""
        all_phis = []
        T = len(all_images)
        for i in range(0, T, self.batch_size):
            images = np.asarray(all_images[i:i + self.batch_size], np.float32)
            if len(images) < self.batch_size:
                pad = np.zeros((self.batch_size - len(images), self.img_size, self.img_size, 3), np.float32)
                images = np.vstack((images, pad))
            all_phis.append(self.compute_phis(images))
        return np.vstack(all_phis)[:T]

    def compute_augmented_phis(self, images, image_sizes, labels, centers, poses, gt3ds, augmentor, keep_images=False):
        """The tfrecord converters' two steps (TubePreprocessorDriver, then compute_all_phis) in one device pass: one tube of T
        frames (uint8, or float in [0, 1]) is augmented by `augmentor` (a human_dynamics_b200.augment.TubeAugmentor) straight
        into the plan's conv1 input, batch by batch, and the trunk runs on it.  Returns the augmentor's dict (device tensors:
        labels, poses, gt3ds, centers, the walks) plus phis (T x 2048); `images` (the fp32 crops) only with keep_images."""
        if augmentor.img_size != self.img_size:
            raise ValueError('augmentor img_size %d != extractor img_size %d' % (augmentor.img_size, self.img_size))
        images = images if isinstance(images, torch.Tensor) else np.asarray(images)
        want = np.array(tuple(images.shape[1:3]))
        if (np.asarray(image_sizes).reshape(-1, 2) != want[None]).any():
            raise ValueError("image_sizes must equal the frames' shape %s" % (tuple(want),))
        frames, labels, centers, poses, gt3ds = augmentor.prepare(images, labels, centers, poses, gt3ds)
        T, S, bs, dev = frames.shape[0], self.img_size, self.batch_size, self.device
        walks = augmentor.walks([T])
        new = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)
        lab, cen = new(tuple(labels.shape), torch.float32), new((T, 2), torch.int32)
        pos, g3, geom = new((T, 72), torch.float32), new((T, 14, 3), torch.float32), new((T, _aug.GEOM_WORDS), torch.int32)
        phis = new((T, self.packed.out_dim), torch.float32)
        crops = new((T, S, S, 3), torch.float32) if keep_images else None
        planes = self.plan.planes
        staging = None if planes is not None else torch.zeros((bs, S, S, 3), dtype=torch.float32, device=dev)
        for i in range(0, T, bs):
            n = min(bs, T - i)
            sl = slice(i, i + n)
            w = {k: walks[k][sl] for k in ('trans', 'scale', 'rot', 'flip')}
            outs = dict(labels_out=lab[sl], centers_out=cen[sl], poses_out=pos[sl], gt3ds_out=g3[sl], geom=geom[sl])
            if planes is not None:
                if n < bs:                    # compute_all_phis zero-pads the last batch
                    planes[0][n:].zero_()
                    planes[1][n:].zero_()
                _aug.tube_augment(frames[sl], labels[sl], centers[sl], poses[sl], gt3ds[sl], w, S, augmentor.trans_max,
                                  augmentor.rotate, crops[sl] if crops is not None else None, (planes[0][:n], planes[1][:n]), **outs)
                self.plan.run(None, self.phis)
            else:
                staging[n:].zero_()
                _aug.tube_augment(frames[sl], labels[sl], centers[sl], poses[sl], gt3ds[sl], w, S, augmentor.trans_max,
                                  augmentor.rotate, staging[:n], None, **outs)
                if crops is not None:
                    crops[sl].copy_(staging[:n])
                self.plan.run(staging, self.phis)
            phis[sl].copy_(self.phis[:n])
        res = {'labels': lab, 'poses': pos, 'gt3ds': g3, 'centers': cen, 'trans_walk': walks['trans'],
               'scale_walk': walks['scale'].reshape(-1, 1), 'rot_walk': walks['rot'].reshape(-1, 1), 'geometry': geom[:, :6],
               'phis': phis}
        if crops is not None:
            res['images'] = crops
        return res
