"""Drop-in for src/util/tube_augmentation.py: TubePreprocessor / TubePreprocessorDriver on the GPU (hd_tube_augment).

Same constructor arguments and the same returned keys and shapes as the reference; the walks and the tube's flip are drawn with
torch on the device (TensorFlow's random stream is not reproduced).  `sess` is accepted and ignored.
"""
import numpy as np

from human_dynamics_b200.augment import TubeAugmentor


def _check_sizes(images, image_sizes):
    want = np.array(np.shape(images)[1:3])
    sizes = np.asarray(image_sizes).reshape(-1, 2)
    if len(sizes) != len(images) or (sizes != want[None]).any():
        raise ValueError('image_sizes must equal the frames\' shape %s (all frames of a call have one size)' % (tuple(want),))


class TubePreprocessor(object):

    def __init__(self, img_size=224, trans_max=20, delta_trans_max=3, scale_max=0.3, delta_scale_max=0.05, rotate_max=0,
                 delta_rotate_max=0, seed=None):
        self.output_size = img_size
        self.augmentor = TubeAugmentor(img_size, trans_max, delta_trans_max, scale_max, delta_scale_max, rotate_max,
                                       delta_rotate_max, seed=seed)

    def __call__(self, images, image_sizes, labels, centers, poses, gt3ds, return_walk=False):
        """images (T x H x W x 3) in [0, 1] (float) or uint8, labels (T x 3 x K), centers (T x 2), poses (T x 72), gt3ds (T x 14 x 3)
        -> dict of numpy arrays: images, labels, poses, gt3ds, centers (T x 2 x 1) [, trans_walk, scale_walk, rot_walk]."""
        images = np.asarray(images)
        _check_sizes(images, image_sizes)
        r = self.augmentor(images, labels, centers, poses, gt3ds)
        ret = {'images': r['images'].cpu().numpy(), 'labels': r['labels'].cpu().numpy(), 'poses': r['poses'].cpu().numpy(),
               'gt3ds': r['gt3ds'].cpu().numpy(), 'centers': r['centers'].cpu().numpy()[:, :, None]}
        if return_walk:
            ret.update(trans_walk=r['trans_walk'].cpu().numpy(), scale_walk=r['scale_walk'].cpu().numpy(),
                       rot_walk=r['rot_walk'].cpu().numpy())
        return ret


class TubePreprocessorDriver(object):

    def __init__(self, img_size=224, trans_max=20, delta_trans_max=3, scale_max=0.3, delta_scale_max=0.05, rotate_max=0,
                 delta_rotate_max=0, sess=None, seed=None):
        self.preprocessor = TubePreprocessor(img_size, trans_max, delta_trans_max, scale_max, delta_scale_max, rotate_max,
                                             delta_rotate_max, seed=seed)

    def __call__(self, images, image_sizes, labels, centers, poses, gt3ds):
        """Labels may be T x 3 x K or T x K x 3 (transposed, as the reference's driver does).  Returns the preprocessor's dict
        with the walks."""
        if np.shape(labels)[-1] == 3:
            labels = np.transpose(labels, [0, 2, 1])
        return self.preprocessor(images, image_sizes, labels, centers, poses, gt3ds, return_walk=True)
