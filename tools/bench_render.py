"""Times hd_render_mesh on the H100 and prints one JSON line.

Workloads (SMPL's F = 13776 faces; 'smooth' = synthetic.make_smooth_mesh, a closed body-sized surface with realistic coverage,
'capsule' = the real SMPL face table over the synthetic capsule vertices, whose triangles are huge and overlap heavily):
  crop      640 frames at S = 224 over a [-1, 1] background (the crop overlay of one C3 window)
  rotated   640 frames at S = 224, the 90-degree view on white
  frame     640 frames at S = 720 over a background (1280 x 720 video frames rendered as visualize_img_orig does), in
            MeshRenderer's workspace-capped chunks
Each is timed with CUDA events over --iters calls after --warmup calls; per-kernel times come from a separate torch.profiler run of
one call.  Also reported: z-buffer bytes, the card's name and power limit (read in the same run), and the CPU seconds of the
float64 oracle (oracle/render_ref.py) for one 224 frame, for contrast.

    python tools/bench_render.py [--frames 640] [--iters 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def frames_of(base, N, seed):
    rng = np.random.RandomState(seed)
    a = rng.uniform(-0.6, 0.6, N)
    c, s = np.cos(a), np.sin(a)
    Ry = np.zeros((N, 3, 3))
    Ry[:, 0, 0], Ry[:, 0, 2], Ry[:, 1, 1], Ry[:, 2, 0], Ry[:, 2, 2] = c, s, 1, -s, c
    verts = np.einsum('vk,njk->nvj', base.astype(np.float64), Ry).astype(np.float32)
    cams = np.stack([rng.uniform(0.8, 1.1, N), rng.uniform(-0.1, 0.1, N), rng.uniform(-0.1, 0.1, N)], 1).astype(np.float32)
    return torch.from_numpy(verts).cuda(), torch.from_numpy(cams).cuda()


def time_call(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_ms(fn):
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if 'render_' in ev.key:
            name = ev.key.split('render_', 1)[1].split('(')[0].split('<')[0]
            t = getattr(ev, 'device_time_total', None)
            if t is None:
                t = ev.cuda_time_total
            out[name] = round(out.get(name, 0.0) + t / 1000.0, 4)
    return out


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(',')]
        return {'gpu': name, 'power_limit': power, 'max_sm_clock': clock}
    except Exception as e:                    # report, do not guess
        return {'gpu': torch.cuda.get_device_name(0), 'power_limit': 'unknown (%s)' % e}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=640)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_render needs a CUDA device')
    from human_dynamics_b200 import synthetic, _lib
    from human_dynamics_b200.render import MeshRenderer, rotation
    N = args.frames
    smpl_faces = np.load(os.path.join(ROOT, 'src', 'tf_smpl', 'smpl_faces.npy'))
    smooth_v, smooth_f = synthetic.make_smooth_mesh(seed=11)
    capsule_v = synthetic.make_synthetic_smpl(seed=2)['v_template'].astype(np.float32)
    res = {'metric': 'render_frames_per_s', 'frames': N, **card()}
    rot = rotation(90, 'y')
    for mesh, base, faces in (('smooth', smooth_v, smooth_f), ('capsule', capsule_v, smpl_faces)):
        mr = MeshRenderer(faces)
        v, c = frames_of(base, N, seed=1)
        bg224 = torch.rand((N, 224, 224, 3), device='cuda') * 2 - 1
        out224 = torch.empty((N, 224, 224, 3), dtype=torch.uint8, device='cuda')
        jobs = {'crop': (lambda: mr.render(v, c, 224, background=bg224, out=out224), 224),
                'rotated': (lambda: mr.render(v, c, 224, rot=rot, out=out224), 224)}
        bg720 = torch.rand((min(N, mr.chunk_frames(720)), 720, 720, 3), device='cuda') * 2 - 1
        out720 = torch.empty((bg720.shape[0], 720, 720, 3), dtype=torch.uint8, device='cuda')

        def frame_job():
            k = bg720.shape[0]
            for n0 in range(0, N, k):
                n = min(k, N - n0)
                mr.render(v[n0:n0 + n], c[n0:n0 + n], 720, background=bg720[:n], out=out720[:n])
        jobs['frame'] = (frame_job, 720)
        for name, (fn, S) in jobs.items():
            ms = time_call(fn, args.iters, args.warmup)
            res['%s_%s_ms' % (mesh, name)] = round(ms, 3)
            res['%s_%s_frames_per_s' % (mesh, name)] = round(N / ms * 1e3, 1)
            res['%s_%s_kernel_ms' % (mesh, name)] = kernel_ms(fn)
        res['%s_chunk_frames_720' % mesh] = mr.chunk_frames(720)
        del bg224, bg720, out224, out720, mr
        torch.cuda.empty_cache()
    res['zbuffer_bytes_per_frame_224'] = 448 * 448 * 8
    res['zbuffer_bytes_per_frame_720'] = 1440 * 1440 * 8
    res['workspace_bytes_640x224'] = int(_lib.lib.hd_render_workspace_bytes(N, 224, 13776))
    from oracle import render_ref
    t = time.perf_counter()
    render_ref.rasterize(smooth_v, [0.9, 0.0, 0.0], smooth_f, 224)
    res['oracle_cpu_s_per_frame_224_smooth'] = round(time.perf_counter() - t, 3)
    res['goal_ms_640_crops'] = 71.8
    print(json.dumps(res))


if __name__ == '__main__':
    main()
