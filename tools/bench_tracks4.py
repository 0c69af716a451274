#!/usr/bin/env python
"""Multi-track batch benchmark (the `tracks4`, `maps6` and `rot4` workloads): one JSON line on stdout.

    python tools/bench_tracks4.py [--workload tracks4|maps6|rot4] [--steps 300] [--warmup 30]

16384 envs x 2 agents over berlin, vegas, skirk and levine in ONE simulator (a canvas stack, DESIGN.md §2; env e on
map e % 4; k_march_lean_het), random actions, env level and per-map auto-reset replayed from a CUDA graph as bench.py's
cfg3.  The same run times each map alone at 16384 x 2 on the single-map path and reports them under `workloads`, so the
cost of mixing is visible.  Timing, L2 flush and metric follow bench.py (its constants are imported from there).
Committed line: profiles/h100/bench_tracks4.json.

`--workload maps6`: the same over all six bundled maps (env e on map e % 6), which come in three resolutions (0.05, 0.0504
and 0.0625 m), so they are stacked with mixed_resolution=True and every layer runs in metres on k_march_lean_het_res;
example_map alone runs on its cell-unit kernel.  Committed line: profiles/h100/bench_maps6.json.

`--workload rot4`: the four tracks of `tracks4`, each with its yaml origin given a different yaw (ROT4_YAWS), stacked with
rotated_origins=True on k_march_lean_rot; start tables are built in each map's rotated frame.  Each rotated map alone is
timed three ways: on k_march_lean_rot (`<map>_alone`), on the literal k_raymarch through debug variant 13
(`<map>_raymarch_alone`, the path rotated maps took before k_march_lean_rot), and as the unrotated original on its
default kernel (`<map>_unrotated_alone`).  Committed line: profiles/h100/bench_rot4.json.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402

from bench import FLUSH_BYTES, METRIC, POSE_GAP, SEED, UNIT   # noqa: E402

TRACKS4 = [('berlin', '.png'), ('vegas', '.png'), ('skirk', '.png'), ('levine', '.pgm')]
MAPS6 = TRACKS4 + [('stata_basement', '.png'), ('example_map', '.png')]
# rot4: the origin yaw of each of the four tracks (rad)
ROT4_YAWS = [0.35, -0.8, 1.9, 3.0]
# workload -> (maps, DeviceMap.stack(mixed_resolution=...), origin yaws or None)
WORKLOADS = {'tracks4': (TRACKS4, False, None), 'maps6': (MAPS6, True, None), 'rot4': (TRACKS4, False, ROT4_YAWS)}


def gpu_card():
    """Card name and power limit, read in the same run as the measurement."""
    import subprocess
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(',')]
        return {'name': name, 'power_limit': limit}
    except Exception as e:
        return {'error': repr(e)}


def run_tracks4(args):
    """The multi-track workload: 16384 envs x 2 agents over the workload's maps in ONE simulator (canvas stack, env e on
    map e % L; tracks4: berlin, vegas, skirk and levine on k_march_lean_het), random actions, env level and per-map auto-reset in a CUDA graph as cfg3.  Start
    poses come from seeded per-map tables of free-space poses (distance transform >= 0.6 m): only example_map ships a
    raceline.  The same run measures each map alone at 16384 x 2 on the single-map path (`workloads`), which shows what
    mixing costs."""
    import torch
    import f1tenth_gym_b200 as f110
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    K, W = args.steps, args.warmup
    names, mixed_resolution, yaws = WORKLOADS[args.workload]
    N, A, B, L = 16384, 2, 1080, len(names)
    plain = [f110.DeviceMap.from_yaml(f110.maps.resolve_map_path(n), e, dev) for n, e in names]
    maps = plain if yaws is None else \
        [f110.DeviceMap(f110.maps.HostMap(m.host.dt, m.host.resolution, (m.host.orig_x, m.host.orig_y, y)), dev)
         for m, y in zip(plain, yaws)]

    def start_tables(ms):
        """256 seeded free-space poses per map, at cell centres of the map's own (rotated) frame, in world coordinates."""
        rng = np.random.default_rng(SEED)
        out = []
        for m in ms:
            h = m.host
            free = np.argwhere(h.dt >= 0.6)
            sel = free[rng.choice(free.shape[0], 256, replace=False)]
            xr, yr = (sel[:, 1] + 0.5) * h.resolution, (sel[:, 0] + 0.5) * h.resolution
            out.append(np.stack([h.orig_x + (h.orig_c * xr - h.orig_s * yr), h.orig_y + (h.orig_s * xr + h.orig_c * yr),
                                 rng.uniform(0, 2 * np.pi, sel.shape[0])], axis=1))
        return out, [torch.from_numpy(t).to(dev) for t in out]
    tables, dtabs = start_tables(maps)
    flush = torch.empty(FLUSH_BYTES, dtype=torch.uint8, device=dev)

    def measure(dmap, ids, tabs, host_tabs, steps, warmup):
        sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, num_beams=B, device=dev)
        sim.set_device_map(dmap, env_map_ids=ids)
        layer = np.zeros(N, int) if ids is None else ids
        prng = np.random.default_rng(SEED + 1)
        poses = np.zeros((N, A, 3))
        for e in range(N):
            t = host_tabs[layer[e]]
            k = int(prng.integers(0, t.shape[0]))
            poses[e] = [t[(k - POSE_GAP * i) % t.shape[0]] for i in range(A)]
        sim.env_reset(poses)
        gen = torch.Generator(device=dev)
        gen.manual_seed(SEED)
        P = min(steps + warmup, 256)
        pool = torch.rand((P, N * A, 2), generator=gen, device=dev, dtype=torch.float64)
        pool[..., 0] = -0.4189 + 0.8378 * pool[..., 0]
        pool[..., 1] = 8.0 * pool[..., 1]
        abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
        sim.capture_graph(abuf, autoreset_poses=tabs, pose_gap=POSE_GAP, autoreset_seed=SEED, env_level=True)
        record = f110._native.lib().f110_debug_last_launch().decode()
        for t in range(warmup):
            abuf.copy_(pool[t % P])
            sim.replay()
        torch.cuda.synchronize(dev)
        ev0 = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        ev1 = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        for t in range(steps):
            flush.zero_()
            abuf.copy_(pool[(warmup + t) % P])
            ev0[t].record()
            sim.replay()
            ev1[t].record()
        torch.cuda.synchronize(dev)
        step_ms = np.array([a.elapsed_time(b) for a, b in zip(ev0, ev1)])
        kms = np.zeros(3)
        for t in range(20):
            flush.zero_()
            kms += np.array(sim.step_profile(pool[t % P].view(N, A, 2)))
            sim.env_post_step()
            sim.autoreset(tabs, POSE_GAP, SEED)
        kms /= 20
        del sim
        torch.cuda.empty_cache()
        return {'value': steps * N * A / (step_ms.sum() * 1e-3), 'ms_per_step': float(step_ms.mean()), 'steps': steps,
                'warmup': warmup, 'step_ms_percentiles': {'p5': float(np.percentile(step_ms, 5)),
                                                          'p50': float(np.percentile(step_ms, 50)),
                                                          'p95': float(np.percentile(step_ms, 95))},
                'kernel_ms': {'k_dynamics': kms[0], 'k_march': kms[1], 'k_tail': kms[2]}, 'launch': record}

    ids = np.arange(N) % L
    main = measure(f110.DeviceMap.stack(maps, mixed_resolution=mixed_resolution, rotated_origins=yaws is not None), ids,
                   dtabs, tables, K, W)
    singles = {}
    for l, (name, _) in enumerate(names):
        singles[name] = measure(maps[l], None, dtabs[l], [tables[l]], K, W)
    if yaws is not None:
        lib = f110._native.lib()
        ptables, pdtabs = start_tables(plain)
        for l, (name, _) in enumerate(names):
            lib.f110_debug_set_variant(13)
            try:
                singles[name + '_raymarch'] = measure(maps[l], None, dtabs[l], [tables[l]], K, W)
            finally:
                lib.f110_debug_set_variant(0)
            singles[name + '_unrotated'] = measure(plain[l], None, pdtabs[l], [ptables[l]], K, W)
    line = {'metric': METRIC, 'value': main['value'], 'unit': UNIT, 'n_gpus': 1, 'steps': K, 'warmup': W,
            'ms_per_step': main['ms_per_step'], 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
            'dtype': 'f64', 'data': 'synthetic',
            'config': {'workload': args.workload, 'maps': [n for n, _ in names], 'env_map_ids': 'e %% %d' % L,
                       'num_envs_per_gpu': N, 'num_agents': A, 'num_beams': B, 'integrator': 'RK4', 'timestep': 0.01,
                       'scan_noise': 'off', 'actions': 'steer~U[-0.4189,0.4189], speed~U[0,8] i.i.d. per tick',
                       'auto_reset': 'ego collision -> hashed pose from the map\'s own table of 256 seeded free-space '
                                     'poses (distance transform >= 0.6 m)'},
            'measurement': {'timing': 'sum of per-step CUDA-event times around a CUDA-graph replay (tick with env level '
                                      'and auto-reset)', 'l2': 'flushed between timed steps (256 MiB memset outside the '
                                      'event pairs)', 'kernel_ms': 'f110_step_profile over 20 ticks'},
            'gpu': gpu_card(), 'step_ms_percentiles': main['step_ms_percentiles'], 'kernel_ms': main['kernel_ms'],
            'launch': main['launch'],
            'workloads': {'%s_alone' % n: r for n, r in singles.items()}}
    if mixed_resolution:
        line['config']['mixed_resolution'] = True
    if yaws is not None:
        line['config']['rotated_origins'] = True
        line['config']['origin_yaws'] = dict(zip([n for n, _ in names], yaws))
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', choices=sorted(WORKLOADS), default='tracks4')
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=30)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error('--steps must be at least 1')
    args.warmup = max(args.warmup, 3)
    run_tracks4(args)


if __name__ == '__main__':
    main()
