#!/usr/bin/env python
"""Stand-alone scan benchmark: f110_scan_layers (k_scan_lean) against what a user runs today, one JSON line on stdout.

    python tools/bench_scan.py [--reps 20] [--warmup 3] [--out profiles/h100/bench_scan.json]

1080 beams, M = 65 536 and 262 144 poses drawn from seeded per-map start tables (256 free-space poses per map, distance
transform >= 0.6 m, as tools/bench_tracks4.py builds them, each pose jittered by up to 0.5 m and given a random yaw), on:
  berlin        alone (metres)                      today: f110_scan (k_raymarch)
  example_map   alone (cell units)                  today: f110_scan (k_raymarch)
  maps6         the six bundled maps, mixed_resolution stack; pose k on layer k % 6
  rot4          berlin, vegas, skirk and levine with the origin yaws of bench_tracks4's rot4, rotated_origins stack
For the stacks, today's way is one f110_scan call per layer on that map's own DeviceMap with that layer's poses; its time is
the sum of those calls.  Every call is timed alone with CUDA events, after warm-up, with the L2 flushed (a 256 MiB memset, as
bench.py) outside the event pair; the figures are means over --reps calls.  The fp32 outputs of the two arms are compared
bit for bit.  The card name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np   # noqa: E402

from bench import FLUSH_BYTES, SEED   # noqa: E402
from bench_tracks4 import MAPS6, ROT4_YAWS, TRACKS4, gpu_card   # noqa: E402

B = 1080
SIZES = (65536, 262144)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    args = ap.parse_args()
    import torch
    import f1tenth_gym_b200 as f110
    from f1tenth_gym_b200 import _native as nat
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    lib = nat.lib()
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    flush = torch.empty(FLUSH_BYTES, dtype=torch.uint8, device=dev)
    load = lambda n, e: f110.DeviceMap.from_yaml(f110.maps.resolve_map_path(n), e, dev)  # noqa: E731

    def rotated(m, yaw):
        h = m.host
        return f110.DeviceMap(f110.maps.HostMap(h.dt, h.resolution, (h.orig_x, h.orig_y, yaw)), dev)
    six = [load(n, e) for n, e in MAPS6]
    rot4 = [rotated(m, y) for m, y in zip(six[:4], ROT4_YAWS)]
    workloads = [('berlin', six[0], [six[0]]), ('example_map', six[5], [six[5]]),
                 ('maps6', f110.DeviceMap.stack(six, mixed_resolution=True), six),
                 ('rot4', f110.DeviceMap.stack(rot4, rotated_origins=True), rot4)]
    beams = f110.DeviceBeams(B, 4.7, f110.maps.DEFAULT_PARAMS, dev)

    def poses_for(layers, M):
        rng = np.random.default_rng(SEED)
        out = np.zeros((M, 3))
        ids = np.arange(M) % len(layers)
        for l, m in enumerate(layers):
            h = m.host
            free = np.argwhere(h.dt >= 0.6)
            sel = free[rng.choice(free.shape[0], 256, replace=False)]
            k = np.flatnonzero(ids == l)
            pick = sel[rng.integers(0, 256, k.size)]
            xr = (pick[:, 1] + 0.5) * h.resolution + rng.uniform(-0.5, 0.5, k.size)
            yr = (pick[:, 0] + 0.5) * h.resolution + rng.uniform(-0.5, 0.5, k.size)
            out[k, 0] = h.orig_x + (h.orig_c * xr - h.orig_s * yr)
            out[k, 1] = h.orig_y + (h.orig_s * xr + h.orig_c * yr)
            out[k, 2] = rng.uniform(0, 2 * np.pi, k.size)
        return torch.from_numpy(out).to(dev), torch.from_numpy(ids.astype(np.int32)).to(dev)

    def timed(fn, reps, warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize(dev)
        e0 = [torch.cuda.Event(enable_timing=True) for _ in range(reps)]
        e1 = [torch.cuda.Event(enable_timing=True) for _ in range(reps)]
        for r in range(reps):
            flush.zero_()
            e0[r].record()
            fn()
            e1[r].record()
        torch.cuda.synchronize(dev)
        return np.array([a.elapsed_time(b) for a, b in zip(e0, e1)])

    results = {}
    for name, dmap, layers in workloads:
        for M in SIZES:
            p, ids = poses_for(layers, M)
            out_new = torch.empty((M, B), dtype=torch.float32, device=dev)
            out_old = torch.empty((M, B), dtype=torch.float32, device=dev)

            def new():
                nat.check(lib.f110_scan_layers(C.byref(dmap.c), C.byref(beams.c), p.data_ptr(), ids.data_ptr(), M,
                                               out_new.data_ptr(), None, None, stream))
            new()
            record = lib.f110_debug_last_launch().decode()
            t_new = timed(new, args.reps, args.warmup)
            # today: f110_scan on each map's own DeviceMap, with that map's poses
            parts = []
            for l, m in enumerate(layers):
                k = torch.nonzero(ids == l).flatten()
                pl = p[k].contiguous()
                ol = torch.empty((k.numel(), B), dtype=torch.float32, device=dev)
                parts.append((m, k, pl, ol))
            old_ms = np.zeros(args.reps)
            for m, k, pl, ol in parts:
                def old(m=m, pl=pl, ol=ol):
                    nat.check(lib.f110_scan(C.byref(m.c), C.byref(beams.c), pl.data_ptr(), pl.shape[0], ol.data_ptr(),
                                            None, None, stream))
                old_ms += timed(old, args.reps, args.warmup)
                out_old[k] = ol
            torch.cuda.synchronize(dev)
            identical = bool(torch.equal(out_new, out_old))
            results['%s_M%d' % (name, M)] = {
                'maps': len(layers), 'poses': M, 'lean_ms': float(t_new.mean()), 'today_ms': float(old_ms.mean()),
                'lean_ms_range': [float(t_new.min()), float(t_new.max())],
                'lean_poses_per_s': M / (t_new.mean() * 1e-3), 'today_poses_per_s': M / (old_ms.mean() * 1e-3),
                'today_over_lean': float(old_ms.mean() / t_new.mean()), 'outputs_identical': identical,
                'lean_launch': record}
            del out_new, out_old, parts
            torch.cuda.empty_cache()
    line = {'metric': 'stand-alone scan time', 'unit': 'ms per call', 'num_beams': B, 'reps': args.reps,
            'warmup': args.warmup, 'gpu': gpu_card(),
            'arms': {'lean': 'one f110_scan_layers call (k_scan_lean) over all poses',
                     'today': 'f110_scan (k_raymarch) on each map\'s own DeviceMap, one call per map, times summed'},
            'poses': 'seeded free-space start tables (256 per map, DT >= 0.6 m), +-0.5 m jitter, random yaw; pose k on '
                     'layer k % L',
            'measurement': 'CUDA events around each call, L2 flushed (256 MiB memset) outside the event pair, mean over reps',
            'workloads': results}
    text = json.dumps(line)
    print(text)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(text + '\n')
    if not all(r['outputs_identical'] for r in results.values()):
        sys.exit('outputs of the two arms differ')


if __name__ == '__main__':
    main()
