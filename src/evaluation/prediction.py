"""Cached predictions for the evaluation -- drop-in for the reference's src/evaluation/prediction.py (:22-165).

Same cache layout and pickles, so caches written by either are interchangeable:

    pred_dir/
        <basename(load_path)>/
            <dataset>-<tfrecord>-P<p_id>.pkl           predictions of one tube (everything but the vertices)
            <dataset>-<tfrecord>-P<p_id>-verts.pkl     its vertices (incl_verts)
            results_<pred_mode>_<tfrecord>_P<p_id>[_min-vis<m>].pkl   its errors
            results_<split>_<pred_mode>_<datasets>.json               the summary
"""
import os
import pickle
from time import time

import numpy as np

PRED_DIR = 'predictions_cache'


def get_pred_path_name(load_path, tf_path, p_id, pred_dir=PRED_DIR, incl_verts=False):
    """Path of the cached predictions of tube p_id of a tfrecord (the dataset is the tfrecord's grandparent directory); creates the
    directories.  Returns (path, file name)."""
    vid_id = os.path.basename(tf_path).replace('.tfrecord', '')
    dataset = os.path.basename(os.path.dirname(os.path.dirname(tf_path)))
    output_name = '{}-{}-P{}{}.pkl'.format(dataset, vid_id, p_id, '-verts' if incl_verts else '')
    out_dir = os.path.join(pred_dir, os.path.basename(load_path))
    os.makedirs(out_dir, exist_ok=True)
    return os.path.join(out_dir, output_name), output_name


def get_result_path_name(split, load_path, pred_mode, datasets, pred_dir=PRED_DIR):
    """Path of the JSON summary of an evaluation."""
    output_name = 'results_{}_{}_{}.json'.format(split, pred_mode, '-'.join(datasets))
    return os.path.join(pred_dir, os.path.basename(load_path), output_name)


def get_eval_path_name(load_path, pred_mode, tf_path, p_id, pred_dir=PRED_DIR, min_visible=0):
    """Path of the pickled errors of one tube."""
    vid_id = os.path.basename(tf_path).replace('.tfrecord', '')
    output_name = 'results_{}_{}_P{}'.format(pred_mode, vid_id, p_id)
    if min_visible > 0:
        output_name += '_min-vis{}'.format(min_visible)
    return os.path.join(pred_dir, os.path.basename(load_path), output_name) + '.pkl'


def split_preds(preds):
    """(predictions without the vertices, the vertices)."""
    preds_dict, verts_dict = {}, {}
    for k, v in preds.items():
        (verts_dict if 'vert' in k else preds_dict)[k] = v
    return preds_dict, verts_dict


def decode_frames(images):
    """Frames as an N x H x W x 3 array; JPEG strings (read_from_example(..., decode_images=False)) are decoded here."""
    if len(images) and isinstance(images[0], (bytes, bytearray)):
        from src.datasets.common import decode_jpeg
        images = [decode_jpeg(im) for im in images]
    return np.asarray(images)


def get_predictions(model, images, load_path, tf_path, p_id, pred_dir=PRED_DIR, incl_verts=False):
    """The cached predictions of a tube if they exist, else model.predict_all_images on its frames (cached for next time).  `images`
    may be decoded frames or JPEG strings; JPEGs are decoded only on a cache miss."""
    t0 = time()
    pred_path, _ = get_pred_path_name(load_path, tf_path, p_id, pred_dir=pred_dir, incl_verts=False)
    vert_path, _ = get_pred_path_name(load_path, tf_path, p_id, pred_dir=pred_dir, incl_verts=True)
    if os.path.exists(pred_path) and (not incl_verts or os.path.exists(vert_path)):
        print('Loading existing predictions!')
        with open(pred_path, 'rb') as f:
            preds = pickle.load(f)
        if incl_verts:
            with open(vert_path, 'rb') as f:
                preds.update(pickle.load(f))
    else:
        print('Computing the predictions.')
        images = decode_frames(images)
        if np.max(images) > 1.1:                 # frames in [0, 255] -> [-1, 1], as the reference's sanity check does
            images = (np.array(images) / 255) * 2 - 1
        preds = model.predict_all_images(images)
        preds.update({'tf_path': tf_path, 'p_id': p_id})
        preds, verts = split_preds(preds)
        with open(pred_path, 'wb') as f:
            pickle.dump(preds, f)
        if incl_verts:
            preds.update(verts)
            with open(vert_path, 'wb') as f:
                pickle.dump(verts, f)
    print('Prediction time:', time() - t0)
    return preds
