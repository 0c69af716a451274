#!/usr/bin/env python
"""Top-down view benchmark: f110_render_views (k_render_views) and F110Env.render('rgb_array'), one JSON line on stdout.

    python tools/bench_views.py [--reps 20] [--warmup 3] [--out profiles/h100/bench_views.json]

16384 envs x 2 agents, one heading-up view per agent (32768 views), at 64 x 64 pixels of 0.1 m and 128 x 128 pixels of 0.05 m,
on berlin alone and on the berlin / vegas / skirk / levine canvas stack (env e on map e % 4).  Agents sit on seeded free-space
poses (distance transform >= 0.6 m, random yaw).  Each call writes into a preallocated `out` and is timed alone with CUDA
events, after warm-up, with the L2 flushed (a 256 MiB memset, as bench.py) outside the event pair; figures are means over
--reps calls.  The bytes a call must write (V * H * W) over its time give the write rate, reported against the H100 SXM data
sheet's 3.35 TB/s of HBM3 bandwidth.  rgb_array: F110Env.render for 1 and 64 envs at 800 x 1000 (the classes and the palette
gather), same timing.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np   # noqa: E402

from bench import FLUSH_BYTES, SEED   # noqa: E402
from bench_tracks4 import TRACKS4, gpu_card   # noqa: E402

N, A = 16384, 2
VIEWS = [((64, 64), 0.1), ((128, 128), 0.05)]
HBM_BYTES_PER_S = 3.35e12


def free_poses(hosts, layer_of_env, rng):
    out = np.empty((len(layer_of_env), A, 3))
    tabs = []
    for h in hosts:
        free = np.argwhere(h.dt >= 0.6)
        tabs.append(free[rng.choice(free.shape[0], 4096, replace=False)])
    for e, l in enumerate(layer_of_env):
        h = hosts[l]
        rc = tabs[l][rng.integers(0, 4096, A)]
        out[e, :, 0] = h.orig_x + (rc[:, 1] + rng.random(A)) * h.resolution
        out[e, :, 1] = h.orig_y + (rc[:, 0] + rng.random(A)) * h.resolution
        out[e, :, 2] = rng.uniform(-np.pi, np.pi, A)
    return out


def timed(fn, flush, reps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.mean(ms)), float(np.min(ms)), float(np.max(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    import torch
    import f1tenth_gym_b200 as f110
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    flush = torch.empty(FLUSH_BYTES, dtype=torch.uint8, device=dev)
    tracks = [f110.DeviceMap.from_yaml(f110.maps.resolve_map_path(n), e, dev) for n, e in TRACKS4]
    result = {'metric': 'render_views', 'card': gpu_card(), 'envs': N, 'agents': A, 'views': N * A, 'reps': args.reps,
              'hbm_data_sheet_bytes_per_s': HBM_BYTES_PER_S, 'render_views': [], 'rgb_array': []}
    for name, dmap, hosts, ids in (('berlin', tracks[0], [tracks[0].host], None),
                                   ('tracks4', f110.DeviceMap.stack(tracks), [m.host for m in tracks], np.arange(N) % 4)):
        sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, device=dev, noise_std=0.0)
        sim.set_device_map(dmap, env_map_ids=ids)
        sim.reset(free_poses(hosts, ids if ids is not None else np.zeros(N, int), np.random.default_rng(SEED)))
        for (H, W), s in VIEWS:
            out = torch.empty((N * A, H, W), dtype=torch.uint8, device=dev)
            mean, lo, hi = timed(lambda: sim.render_views(None, (H, W), s, 0.0, True, out=out), flush, args.reps, args.warmup)
            nbytes = N * A * H * W
            counts = torch.bincount(out.view(-1), minlength=256)[:5].cpu().numpy() / float(nbytes)
            result['render_views'].append({
                'map': name, 'size': [H, W], 'metres_per_pixel': s, 'ms_mean': round(mean, 4), 'ms_min': round(lo, 4),
                'ms_max': round(hi, 4), 'bytes_written': nbytes, 'write_GB_per_s': round(nbytes / (mean * 1e-3) / 1e9, 1),
                'share_of_hbm_data_sheet': round(nbytes / (mean * 1e-3) / HBM_BYTES_PER_S, 3),
                'class_fractions': [round(float(c), 4) for c in counts]})
            del out
        del sim
    for K in (1, 64):
        env = f110.F110Env(map='berlin', num_agents=A, num_envs=K, device=dev, scan_noise_std=0.0)
        env.reset(free_poses([tracks[0].host], np.zeros(K, int), np.random.default_rng(SEED + K)))
        envs = list(range(K))
        mean, lo, hi = timed(lambda: env.render(mode='rgb_array', env_ids=envs), flush, args.reps, args.warmup)
        result['rgb_array'].append({'envs': K, 'size': [800, 1000], 'metres_per_pixel': 0.024, 'ms_mean': round(mean, 4),
                                    'ms_min': round(lo, 4), 'ms_max': round(hi, 4), 'bytes_out': K * 800 * 1000 * 3})
        del env
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
