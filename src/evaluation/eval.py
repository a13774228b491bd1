"""Evaluates a model on the test tfrecords -- drop-in for the reference's src/evaluation/eval.py.

    python -m src.evaluation.eval --tf_dir <dir with <dataset>/<split>/*.tfrecord> --load_path <checkpoint>
        --smpl_model_path <SMPL pickle> [--test_datasets 3dpw,h36m,penn_action --split test --pred_mode pred]

Same flow, cache files, JSON and summary table as the reference: per tube, cached predictions (prediction.py) of
`Tester.predict_all_images`, then the errors of compute_errors_batched, pickled per tube; per dataset, the nanmean over tfrecords of
each tfrecord's nanmean, rounded to 5 places.  Meshes are scored for the test split of 3DPW only.  No TensorFlow: the tfrecords are
read by src/datasets/common.py, and the metrics run on the GPU (human_dynamics_b200.evaluate.Evaluator) -- all tubes of a tfrecord
whose errors are not cached yet in one pass; the per-tube pickles are what one tube at a time gives.

Deliberate deviations from the reference:
  * pred_mode 'hal' keeps the keys ending in '_hal' (their centre prediction) when the predictions have them and the ordinary keys
    otherwise: the reference's Tester files the hallucinator's output under the ordinary keys, where the reference's branch fails.
  * test_sequence_const takes delta_t as an argument (the flag `delta_t` the reference reads exists in none of its modules); main
    passes --delta_t.
  * --load_path may also name a .npz of TF-named variables (whatever Tester loads).
"""
import json
import os
import pickle
import sys
from glob import glob
from time import time

import numpy as np

from src.datasets.common import read_from_example, tf_record_iterator
from src.evaluation.eval_util import extend_dict_entries, mean_of_dict_values, update_dict_entries
from src.evaluation.prediction import get_eval_path_name, get_predictions, get_result_path_name, decode_frames

SMPL_MODEL_PATH = 'models/neutral_smpl_with_cocoplustoesankles_reg.pkl'
DATASETS_3D = ['3dpw', 'h36m']
CONST_KEYS = ('past', 'past_const', 'present', 'future', 'future_const')

_EVALUATOR = {}


def get_evaluator(smpl=None):
    """The device evaluator over the SMPL constants `smpl` (an SMPLConstants, a pickle path or a model dict), or without SMPL
    constants (no meshes) for smpl=None.  The last one is kept for the next call."""
    from human_dynamics_b200.evaluate import Evaluator
    key = id(smpl) if smpl is not None else None
    if key not in _EVALUATOR:
        consts = smpl
        if smpl is not None and not hasattr(smpl, 'c'):
            from human_dynamics_b200.smpl import SMPLConstants
            consts = SMPLConstants(smpl, joint_type='cocoplus')
        _EVALUATOR.clear()
        _EVALUATOR[key] = Evaluator(consts)
    return _EVALUATOR[key]


def compute_gpu_smpl(poses, shapes, get_joints=False, smpl=None):
    """Vertices (and cocoplus joints) of axis-angle poses [N,72] / [N,24,3] and shapes [N,10] on the GPU (eval.py:68-90)."""
    import torch
    from human_dynamics_b200.smpl import SMPLConstants
    consts = smpl if hasattr(smpl, 'c') else SMPLConstants(smpl if smpl is not None else SMPL_MODEL_PATH, joint_type='cocoplus')
    dev = consts.device
    beta = torch.as_tensor(np.asarray(shapes, np.float32).reshape(-1, 10), device=dev)
    theta = torch.as_tensor(np.asarray(poses, np.float32).reshape(-1, 72), device=dev)
    out = consts.forward(beta, theta, want_joints=get_joints, want_Rs=False, want_Jtr=False)
    verts = out['verts'].cpu().numpy()
    return (verts, out['joints'].cpu().numpy()) if get_joints else verts


def restore_config(config):
    """Restores the settings of the JSON saved beside the checkpoint, except batch_size, load_path, smpl_model_path and T."""
    param_path = glob(os.path.join(os.path.dirname(config.load_path), '*.json'))
    if not param_path:
        return config
    ignore_keys = {'batch_size', 'load_path', 'smpl_model_path', 'T'}
    with open(param_path[0], 'r') as fp:
        prev_config = json.load(fp)
    for k, v in prev_config.items():
        if k not in ignore_keys and hasattr(config, k):
            setattr(config, k, v)
    return config


def compute_errors_batched(kps_gt, kps_pred, joints_gt=None, joints_pred=None, poses_gt=None, poses_pred=None, shape_gt=None,
                           shapes_pred=None, img_size=224, has_3d=False, min_visible=6, compute_mesh=False, smpl=None):
    """The error dict of one tube (eval.py:114-193) computed on the GPU.  The meshes use `smpl` (as for get_evaluator), by default
    the model at SMPL_MODEL_PATH like the reference's compute_gpu_smpl."""
    return get_evaluator(_mesh_model(smpl) if compute_mesh else None).errors(
        kps_gt=kps_gt, kps_pred=kps_pred, joints_gt=joints_gt, joints_pred=joints_pred, poses_gt=poses_gt, poses_pred=poses_pred,
        shape_gt=shape_gt, shapes_pred=shapes_pred, img_size=img_size, has_3d=has_3d, min_visible=min_visible,
        compute_mesh=compute_mesh)


def _mesh_model(smpl):
    return smpl if smpl is not None else SMPL_MODEL_PATH


def _img_size(images):
    """The frame height of a tube: read from the first JPEG's SOF marker (hd_jpeg_parse, no decoding), or from a decoded frame."""
    if len(images) and isinstance(images[0], (bytes, bytearray)):
        from human_dynamics_b200 import jpeg
        try:
            return jpeg.parse(images[0])[0].height
        except jpeg.UnsupportedJPEG:
            pass
    return decode_frames(images[:1]).shape[1]


def _select_preds(preds, pred_mode):
    if pred_mode == 'hal' and any('_hal' in k for k in preds):
        return {k.replace('_hal', ''): v[:, 1] for k, v in preds.items() if '_hal' in k}   # the centre prediction
    return preds


def _tube_args(data, preds):
    return dict(kps_gt=data['kps'], kps_pred=preds['kps'], joints_gt=data['gt3ds'], joints_pred=preds['joints'][:, :14],
                poses_gt=data['poses'], poses_pred=preds['poses'], shape_gt=data['shape'], shapes_pred=preds['shapes'])


def _save(eval_path, errors):
    with open(eval_path, 'wb') as f:
        print('Saving eval to', eval_path)
        pickle.dump(errors, f)


def test_sequence(data, preds, eval_path, pred_mode='pred', has_3d=False, min_visible=6, compute_mesh=False, smpl=None):
    """Errors of one tube, from its pickle when it exists (eval.py:196-243)."""
    preds = _select_preds(preds, pred_mode)
    if os.path.exists(eval_path):
        print('Eval already exists! {}'.format(eval_path))
        with open(eval_path, 'rb') as f:
            return pickle.load(f)
    t0 = time()
    errors = compute_errors_batched(img_size=_img_size(data['images']), has_3d=has_3d, min_visible=min_visible,
                                    compute_mesh=compute_mesh, smpl=smpl, **_tube_args(data, preds))
    _save(eval_path, errors)
    print('Eval time:', time() - t0)
    return errors


def test_sequences(items, pred_mode='pred', has_3d=False, min_visible=6, compute_mesh=False, smpl=None):
    """test_sequence for every (data, preds, eval_path) of `items`, the uncached ones in one device pass."""
    results = [None] * len(items)
    todo = []
    for i, (data, preds, eval_path) in enumerate(items):
        if os.path.exists(eval_path):
            print('Eval already exists! {}'.format(eval_path))
            with open(eval_path, 'rb') as f:
                results[i] = pickle.load(f)
        else:
            todo.append(i)
    if todo:
        t0 = time()
        groups = {}
        for i in todo:                       # one pass per frame size (a tfrecord has one)
            groups.setdefault(_img_size(items[i][0]['images']), []).append(i)
        for img_size, idx in groups.items():
            tubes = [_tube_args(items[i][0], _select_preds(items[i][1], pred_mode)) for i in idx]
            errs = get_evaluator(_mesh_model(smpl) if compute_mesh else None).errors_many(
                tubes, img_size=img_size, has_3d=has_3d, min_visible=min_visible, compute_mesh=compute_mesh)
            for i, e in zip(idx, errs):
                _save(items[i][2], e)
                results[i] = e
        print('Eval time:', time() - t0)
    return results


def test_sequence_const(data, preds, eval_path, has_3d=False, min_visible=6, delta_t=5):
    """The hallucinator's past / present / future predictions against the constant baseline (eval.py:246-327) for predictions that
    carry the '_hal' keys ([n, 3, ...]: past, present, future).  delta_t is an argument here (see the module docstring)."""
    d = delta_t
    kps, joints, poses = preds['kps_hal'], preds['joints_hal'], preds['poses_hal']
    gt_kps, gt3ds, gt_poses = data['kps'], data['gt3ds'], data['poses']
    cases = {
        'present': (slice(None), slice(None), 0),
        'past': (slice(None, -d), slice(d, None), 0),
        'past_const': (slice(None, -d), slice(d, None), 1),
        'future': (slice(d, None), slice(None, -d), 2),
        'future_const': (slice(d, None), slice(None, -d), 1),
    }
    names = list(CONST_KEYS)
    tubes = [dict(kps_gt=gt_kps[cases[k][0]], kps_pred=kps[cases[k][1], cases[k][2]], joints_gt=gt3ds[cases[k][0], :14],
                  joints_pred=joints[cases[k][1], cases[k][2], :14], poses_gt=gt_poses[cases[k][0]],
                  poses_pred=poses[cases[k][1], cases[k][2]]) for k in names]
    errs = get_evaluator().errors_many(tubes, img_size=_img_size(data['images']), has_3d=has_3d, min_visible=min_visible)
    errors_dict = dict(zip(names, errs))
    _save(eval_path, errors_dict)
    return errors_dict


def print_summary(errors_dict):
    title_format = '{:>15}' + '{:>11}' * 8
    row_format = '{:>15}' + '{:>11.5f}' * 8
    keys = ['accel', 'kp', 'kp_pa', 'kp_pck', 'joints', 'joints_pa', 'mesh_posed', 'mesh_tpose']
    print(title_format.format('Data', *keys))
    for dataset, errors in sorted(errors_dict.items()):
        print(row_format.format(dataset, *[errors.get(key, -1) for key in keys]))


def save_results(config, all_dataset_results, json_path=''):
    if json_path:
        with open(json_path, 'w') as f:
            json.dump(all_dataset_results, f)
    if config.pred_mode == 'const':
        for pred_type, predictions in sorted(all_dataset_results.items()):
            print('Predicting', pred_type)
            print_summary(predictions)
    else:
        print_summary(all_dataset_results)


def tfrecord_paths(config, dataset):
    pattern = '*cam03*.tfrecord' if dataset == 'h36m' else '*.tfrecord'
    paths = sorted(glob(os.path.join(config.tf_dir, dataset, config.split, pattern)))
    return paths[::-1] if config.reverse else paths


def main(config, model=None):
    """Evaluates config.load_path on config.test_datasets and writes the JSON summary; returns the results dict.  `model` (a Tester)
    is built from config when not given."""
    t0 = time()
    config = restore_config(config)
    print('-' * 20)
    print('Evaluating {}'.format(config.load_path))
    json_path = get_result_path_name(split=config.split, load_path=config.load_path, pred_mode=config.pred_mode,
                                     datasets=config.test_datasets, pred_dir=config.pred_dir)
    if os.path.exists(json_path):
        print(json_path, 'already exists!')
        with open(json_path, 'r') as f:
            all_dataset_results = json.load(f)
        save_results(config, all_dataset_results)
        print('Total time:', time() - t0)
        print('-' * 20)
        return all_dataset_results

    if model is None:
        from src.evaluation.tester import Tester
        resnet_path = config.resnet_path if getattr(config, 'precomputed_phi', False) else ''
        model = Tester(config, pretrained_resnet_path=resnet_path, sequence_length=config.T)
    const = config.pred_mode == 'const'
    all_dataset_results = {k: {} for k in CONST_KEYS} if const else {}
    for dataset in config.test_datasets:
        print('Evaluating dataset:', dataset)
        dataset_result = {k: {} for k in CONST_KEYS} if const else {}
        tf_paths = tfrecord_paths(config, dataset)
        has_3d = dataset in DATASETS_3D
        compute_mesh = config.split == 'test' and dataset == '3dpw'
        for i, fname in enumerate(tf_paths):
            print('\n', '*' * 10)
            print(dataset, '{}/{}'.format(i, len(tf_paths)))
            print('Running on', os.path.basename(fname))
            path_result = {k: {} for k in CONST_KEYS} if const else {}
            items = []
            for p_id, s_ex in enumerate(tf_record_iterator(fname)):
                data = read_from_example(s_ex, decode_images=False)
                preds = get_predictions(model=model, images=data['images'], load_path=config.load_path, tf_path=fname, p_id=p_id,
                                        pred_dir=config.pred_dir)
                eval_path = get_eval_path_name(load_path=config.load_path, pred_mode=config.pred_mode, tf_path=fname, p_id=p_id,
                                               pred_dir=config.pred_dir, min_visible=config.min_visible)
                if const:
                    errors_dict = test_sequence_const(data=data, preds=preds, eval_path=eval_path, has_3d=has_3d,
                                                      min_visible=config.min_visible, delta_t=config.delta_t)
                    for k in errors_dict:
                        extend_dict_entries(path_result[k], errors_dict[k])
                else:
                    items.append((data, preds, eval_path))
            if not const:
                for errors in test_sequences(items, pred_mode=config.pred_mode, has_3d=has_3d, min_visible=config.min_visible,
                                             compute_mesh=compute_mesh, smpl=model.smpl):
                    extend_dict_entries(path_result, errors)
                update_dict_entries(dataset_result, path_result)
            else:
                for k in path_result:
                    update_dict_entries(dataset_result[k], path_result[k])
        if const:
            for pred_type, result in dataset_result.items():
                mean_of_dict_values(result)
                all_dataset_results[pred_type][dataset] = result
        else:
            mean_of_dict_values(dataset_result)
            all_dataset_results[dataset] = dataset_result

    save_results(config, all_dataset_results, json_path)
    print('Total time:', time() - t0)
    print('-' * 20)
    return all_dataset_results


# ---------------------------------------------------------------------------------------------------------------- flags
def define_flags():
    """The reference's evaluation flags plus the model fields Tester reads (src/config.py defaults)."""
    from absl import flags
    F = flags.FLAGS
    if 'tf_dir' in F:
        return F
    flags.DEFINE_string('resnet_path', '', 'Pretrained ResNet to merge in when precomputed_phi is set.')
    flags.DEFINE_string('pred_mode', 'pred', 'Which prediction track to use (pred, hal, const).')
    flags.DEFINE_string('tf_dir', '', 'Parent directory of tfrecords.')
    flags.DEFINE_string('pred_dir', 'predictions_cache', 'Prediction Directory.')
    flags.DEFINE_list('test_datasets', ['3dpw', 'nba', 'penn_action'], 'Datasets to evaluate.')
    flags.DEFINE_string('split', 'val', 'val or test.')
    flags.DEFINE_integer('min_visible', 6, 'Minimum visible keypoints')
    flags.DEFINE_boolean('reverse', False, 'If True, runs tf records in reverse')
    flags.DEFINE_string('load_path', '', 'Checkpoint to evaluate.')
    flags.DEFINE_string('smpl_model_path', SMPL_MODEL_PATH, 'SMPL model pickle.')
    flags.DEFINE_integer('batch_size', 8, 'Tubes per forward pass.')
    flags.DEFINE_integer('T', 20, 'Frames per window.')
    flags.DEFINE_integer('num_conv_layers', 3, 'Temporal encoder depth.')
    flags.DEFINE_list('delta_t_values', ['-5', '5'], 'Hallucinator offsets.')
    flags.DEFINE_integer('num_kps', 25, 'Keypoints per frame.')
    flags.DEFINE_integer('img_size', 224, 'Input size.')
    flags.DEFINE_boolean('precomputed_phi', False, 'Merge the ResNet of resnet_path into the model.')
    flags.DEFINE_integer('delta_t', 5, 'Offset of the const evaluation.')
    return F


class _Config(object):
    """The flag values as the attribute object main and Tester read."""

    def __init__(self, F):
        for k in ('resnet_path', 'pred_mode', 'tf_dir', 'pred_dir', 'test_datasets', 'split', 'min_visible', 'reverse', 'load_path',
                  'smpl_model_path', 'batch_size', 'T', 'num_conv_layers', 'delta_t_values', 'num_kps', 'img_size', 'precomputed_phi',
                  'delta_t'):
            setattr(self, k, getattr(F, k))
        self.sequence_length = self.T
        self.num_stage = 3
        self.weights = None
        self.smpl_model = None
        self.impl = os.environ.get('HD_IMPL', 'auto')
        self.frame_chunk, self.late_chunk = 160, 640
        self.extra = {}

    def __setattr__(self, k, v):
        object.__setattr__(self, k, v)
        if k == 'T':
            object.__setattr__(self, 'sequence_length', v)


def _run(argv):
    F = define_flags()
    config = _Config(F)
    assert config.load_path, 'Must specify load_path!'
    assert config.tf_dir
    if config.pred_mode == 'hal':
        print('evaluating with the hallucinated track!!')
    main(config)


if __name__ == '__main__':
    define_flags()
    from absl import app
    app.run(_run, argv=sys.argv)
