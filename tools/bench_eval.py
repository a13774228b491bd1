"""Times the GPU evaluation (human_dynamics_b200.evaluate, csrc/eval.cu) on a synthetic test split and prints one JSON line.

Workload: --tubes tubes (default 40) of --frames frames in all (default 35 000; 3DPW's test split is of that order, its exact frame
count is not recorded in this repository), 25 keypoints, 14 joints, meshes on (what eval.py does for 3DPW's test split), the synthetic
SMPL model (6 890 vertices).  Timed, each as the median of --rounds synchronised wall-clock rounds (upload and fetch included):
  split:      Evaluator.errors_many over the whole split, one pass;
  per_tube:   Evaluator.errors once per tube (what eval.test_sequence does for a tube whose errors are not cached);
  launch:     the device work of the one-pass call alone (CUDA events around Evaluator._launch);
  host:       the same scoring as compute_errors_batched written with this repository's numpy eval_util and the src.tf_smpl SMPL
              drop-in, on the first --host-tubes tubes only (reported per frame, with the frame count it was measured on);
  tfrecord:   reading one test record of --record-frames 224^2 JPEG frames (tf_record_iterator with both CRC checks +
              read_from_example), without and with decoding the frames (host only).
The card's name, power limit and max SM clock are read (never set) in the same run.

    python tools/bench_eval.py [--frames 35000] [--tubes 40] [--rounds 5] [--host-tubes 2] [--record-frames 300]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_smpl_grad import card          # noqa: E402


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def host_scoring(t, smpl, img_size=224, min_visible=6):
    """compute_errors_batched (eval.py:114-193, has_3d and compute_mesh on) with numpy eval_util and the src.tf_smpl SMPL drop-in."""
    from src.evaluation import eval_util as eu
    kp, kp_pa, pck = eu.compute_error_kp(t['kps_gt'], (t['kps_pred'] + 1) * 0.5 * img_size, alpha=0.05 * img_size,
                                         min_visible=min_visible)
    accel = eu.compute_accel(t['joints_pred'])
    vis = np.sum(t['kps_gt'][:, :14, 2], axis=1) > min_visible
    accel_err = eu.compute_error_accel(t['joints_gt'], t['joints_pred'], vis)
    n = len(t['kps_gt'])
    shapes_gt = np.tile(t['shape_gt'], (n, 1))
    poses_pred = np.array([eu.rot_mat_to_axis_angle(p) for p in t['poses_pred']])

    def verts(poses, shapes):
        v, _, _ = smpl(torch.from_numpy(np.ascontiguousarray(shapes, np.float32)).cuda(),
                       torch.from_numpy(np.ascontiguousarray(poses, np.float32)).cuda(), get_skin=True)
        return v.cpu().numpy()
    zeros = np.zeros((n, 72))
    tpose = eu.compute_error_verts(verts(zeros, shapes_gt)[vis], verts(zeros, t['shapes_pred'])[vis])
    posed = eu.compute_error_verts(verts(t['poses_gt'], shapes_gt)[vis], verts(poses_pred, t['shapes_pred'])[vis])
    j, jpa = eu.compute_error_3d(t['joints_gt'], t['joints_pred'], vis)
    return kp, kp_pa, pck, accel, accel_err, tpose, posed, j, jpa


def read_record(n):
    """Seconds to read one test record of n 224^2 JPEG frames, without and with JPEG decoding."""
    import tempfile
    from oracle.tfrecord_writer import make_test_example, write_tfrecord
    from src.datasets.common import read_from_example, tf_record_iterator
    yy, xx = np.mgrid[0:224, 0:224]
    imgs = [np.stack([(xx * (f % 7 + 1)) % 256, (yy + 3 * f) % 256, (xx + yy) % 256], -1).astype(np.uint8) for f in range(n)]
    from oracle.eval_ref import make_eval_tubes
    t = make_eval_tubes([n], seed=1, special=False)[0]
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, 'r.tfrecord')
        write_tfrecord(path, [make_test_example(imgs, t['kps_gt'], t['joints_gt'], t['poses_gt'], t['shape_gt'])])
        size = os.path.getsize(path)
        out = {'frames': n, 'bytes': size}
        for name, dec in (('s_no_decode', False), ('s_decode', True)):
            t0 = time.perf_counter()
            for rec in tf_record_iterator(path):
                read_from_example(rec, decode_images=dec)
            out[name] = round(time.perf_counter() - t0, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=35000)
    ap.add_argument('--tubes', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--host-tubes', type=int, default=2)
    ap.add_argument('--record-frames', type=int, default=300)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_eval needs a CUDA device')
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.evaluate import Evaluator
    from human_dynamics_b200.smpl import SMPLConstants
    from src.tf_smpl.batch_smpl import SMPL
    from oracle.eval_ref import make_eval_tubes
    torch.cuda.set_device(0)
    model = synthetic.make_synthetic_smpl(seed=2)
    consts = SMPLConstants(model)
    lens = [a.frames // a.tubes + (1 if i < a.frames % a.tubes else 0) for i in range(a.tubes)]
    tubes = make_eval_tubes(lens, seed=0)
    ev = Evaluator(consts)
    kw = dict(img_size=224, has_3d=True, min_visible=6, compute_mesh=True)
    res = {'tool': 'bench_eval', **card(), 'frames': a.frames, 'tubes': a.tubes, 'vertices': consts.num_verts, 'rounds': a.rounds}

    def split():
        ev.errors_many(tubes, **kw)

    def per_tube():
        for t in tubes:
            ev.errors(**t, **kw)
    staged = ev._stage(tubes, True, True)

    def launch_only():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ev._launch(staged, 224, 6)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)
    split(), per_tube(), launch_only()          # warm-up
    ms = {'split': [], 'per_tube': [], 'launch': []}
    for _ in range(a.rounds):
        ms['split'].append(wall(split))
        ms['per_tube'].append(wall(per_tube))
        ms['launch'].append(launch_only())
    for k, v in ms.items():
        med = statistics.median(v)
        res[k] = {'ms': round(med, 3), 'us_per_frame': round(med * 1e3 / a.frames, 4), 'spread_ms': [round(min(v), 3), round(max(v), 3)]}
    smpl = SMPL(model)
    host = tubes[:a.host_tubes]
    nf = sum(len(t['kps_gt']) for t in host)
    host_scoring(host[0], smpl)                 # warm-up
    t0 = time.perf_counter()
    for t in host:
        host_scoring(t, smpl)
    host_ms = (time.perf_counter() - t0) * 1e3
    res['host'] = {'frames_measured': nf, 'ms': round(host_ms, 1), 'us_per_frame': round(host_ms * 1e3 / nf, 2)}
    res['host_over_split_per_frame'] = round(res['host']['us_per_frame'] / res['split']['us_per_frame'], 1)
    res['tfrecord'] = read_record(a.record_frames)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
