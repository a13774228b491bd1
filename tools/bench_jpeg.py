"""Times JPEG decoding on the GPU (human_dynamics_b200.jpeg, csrc/jpeg.cu) against cv2.imdecode on the same bytes; prints one JSON line.

Workloads (4:2:0, quality 95, seeded synthetic video-like frames from oracle/jpeg_ref.make_image):
  batch_224:   N = 160 frames at 224^2 (a training batch, B*T = 8 x 20);
  batch_300:   N = 640 frames at 300^2 (a batch of the image training path);
  split_224:   N = --split frames at 224^2 (default 35 000, an evaluation split; 512 distinct frames repeated).
For each: `gpu_ms` the median of --rounds synchronised wall-clock calls of jpeg.decode (host parse, the one upload, the launches and
the status check), `kernel_ms` the sum of the four kernels' device time from torch.profiler in a separate call, `host_parse_ms` the
parse alone; `cv2_1t_ms` cv2.imdecode one frame after another in this process with one OpenCV thread, and `cv2_pool_ms` a process pool
over the host cores this process may use (at most 64, reported) decoding the same bytes, both extrapolated from at most --cv2-frames frames.
`get_predictions` times src.evaluation.prediction.get_predictions end to end on one --record-frames-frame 224^2 tube on a prediction
cache miss: `before` with the frames decoded by cv2 on the host (what it did before the GPU decoder), `after` from the JPEG strings.
The card's name, power limit and max SM clock are read (never set) in the same run.

    python tools/bench_jpeg.py [--rounds 5] [--split 35000] [--cv2-frames 2000] [--record-frames 300]
"""
import argparse
import contextlib
import io
import json
import multiprocessing as mp
import os
import statistics
import sys
import tempfile
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


def frames(n, size, distinct=512):
    from oracle import jpeg_ref
    uniq = [jpeg_ref.encode(jpeg_ref.make_image(size, size, seed=i), 95, '420') for i in range(min(n, distinct))]
    return [uniq[i % len(uniq)] for i in range(n)]


def _cv2_chunk(chunk):
    import cv2
    cv2.setNumThreads(1)
    for d in chunk:
        cv2.imdecode(np.frombuffer(d, np.uint8), cv2.IMREAD_COLOR)
    return len(chunk)


def cv2_times(jpegs, limit, pool):
    sub = jpegs[:limit]
    t0 = time.perf_counter()
    _cv2_chunk(sub)
    one = (time.perf_counter() - t0) * 1e3 * len(jpegs) / len(sub)
    n = pool._processes
    parts = [sub[i::n] for i in range(n)]
    pool.map(_cv2_chunk, parts)                          # warm the workers
    t0 = time.perf_counter()
    pool.map(_cv2_chunk, parts)
    many = (time.perf_counter() - t0) * 1e3 * len(jpegs) / len(sub)
    return round(one, 2), round(many, 2)


def kernel_ms(jpegs):
    from torch.profiler import profile, ProfilerActivity
    from human_dynamics_b200 import jpeg
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        jpeg.decode(jpegs)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if 'jpeg_' in e.key and '_kernel' in e.key:
            name = [w for w in ('prep', 'entropy', 'idct', 'color') if w in e.key][0]
            out[name] = round(getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0.0)) / 1e3, 3)
    out['total'] = round(sum(out.values()), 3)
    return out


def parse_ms(jpegs):
    from human_dynamics_b200 import jpeg
    t0 = time.perf_counter()
    for d in jpegs:
        jpeg.parse(d)
    return round((time.perf_counter() - t0) * 1e3, 2)


def get_predictions_times(n, rounds):
    from human_dynamics_b200 import synthetic
    from human_dynamics_b200.config import HMMRConfig
    from src.datasets.common import decode_jpeg
    from src.evaluation.prediction import get_predictions
    from src.evaluation.tester import Tester
    model = Tester(HMMRConfig(batch_size=1, sequence_length=20, weights=synthetic.make_synthetic_weights(seed=1),
                              smpl_model=synthetic.make_synthetic_smpl(seed=2), pred_mode='pred'))
    jpegs = frames(n, 224, distinct=n)
    res = {'frames': n}
    for name, images in (('before', lambda: [decode_jpeg(d) for d in jpegs]), ('after', lambda: jpegs)):
        ts = []
        for r in range(rounds + 1):
            with tempfile.TemporaryDirectory() as td, contextlib.redirect_stdout(io.StringIO()):
                ts.append(wall(lambda: get_predictions(model, images(), 'm', os.path.join(td, 'x', 'test', 'r.tfrecord'), 0,
                                                       pred_dir=td)))
        res[name + '_ms'] = round(statistics.median(ts[1:]), 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--split', type=int, default=35000)
    ap.add_argument('--cv2-frames', type=int, default=2000)
    ap.add_argument('--record-frames', type=int, default=300)
    a = ap.parse_args()
    from human_dynamics_b200 import jpeg
    torch.cuda.init()
    res = dict(card())
    cores = min(len(os.sched_getaffinity(0)), 64)
    res['cv2_pool_processes'] = cores
    pool = mp.get_context('spawn').Pool(cores)
    try:
        for name, n, size in (('batch_224', 160, 224), ('batch_300', 640, 300), ('split_224', a.split, 224)):
            jpegs = frames(n, size)
            jpeg.decode(jpegs)                                       # warm-up: module load, allocator
            ts = [wall(lambda: jpeg.decode(jpegs)) for _ in range(a.rounds)]
            one, many = cv2_times(jpegs, a.cv2_frames, pool)
            res[name] = {'frames': n, 'size': size, 'mbytes': round(sum(map(len, jpegs)) / 1e6, 2),
                         'gpu_ms': round(statistics.median(ts), 2), 'host_parse_ms': parse_ms(jpegs), 'kernel_ms': kernel_ms(jpegs),
                         'cv2_1t_ms': one, 'cv2_pool_ms': many}
            res[name]['gpu_frames_per_s'] = round(n / res[name]['gpu_ms'] * 1e3)
            res[name]['cv2_pool_frames_per_s'] = round(n / many * 1e3)
    finally:
        pool.close()
        pool.join()
    res['get_predictions'] = get_predictions_times(a.record_frames, a.rounds)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
