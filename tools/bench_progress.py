#!/usr/bin/env python
"""Centerline progress benchmark: f110_track_progress (k_track_progress) alone, and the tick with and without it, one JSON line.

    python tools/bench_progress.py [--reps 50] [--ticks 100] [--rounds 5] [--out profiles/h100/bench_progress.json]

Two workloads at 16384 envs x 2 agents: example_map with its raceline as the centerline (782 segments), and a stack of four
generated tracks (trackgen.random_tracks(21, 4), 291-365 segments each; env e on track e % 4) with per-map auto-reset.  Agents
start on their centerline, 5 waypoints apart, and run 50 ticks of fixed random actions before the timing, so that most of them
are tracked.  The update alone is timed with CUDA events around one launch, after warm-up, with the L2 flushed (a 256 MiB
memset, as bench.py) outside the event pair (mean, median, min and max of --reps launches), in two arms:
  tracking   every agent as the ticks left it (the windowed search of 65 segments; agents the last tick reset re-acquire);
  acquiring  every agent unacquired (seg = -1, set outside the event pair): the global search, the worst case after a mass
             reset.
The tick is timed as CUDA-graph replays (f110_tick with env level and auto-reset, as bench.py's cfg3), one graph without the
update and one of an identical simulator with it appended (capture_graph(progress=True)), alternated in --rounds blocks of
--ticks replays; no flush there.  The card name and power limit are read in the same run.
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
from bench_tracks4 import gpu_card   # noqa: E402

N, A = 16384, 2
GAP = 5


def workloads(f110, dev):
    """name -> (DeviceMap, env_map_ids or None, centerline tables, per-layer start tables (device), start poses (N, A, 3))."""
    rng = np.random.default_rng(SEED)
    wp = np.loadtxt(os.path.join(ROOT, 'f1tenth_gym_b200', 'maps', 'example_waypoints.csv'), delimiter=';', skiprows=3)
    em = f110.DeviceMap.from_yaml(f110.maps.resolve_map_path('example_map'), '.png', dev)
    starts = f110.maps.load_waypoints()[:-1]
    K = starts.shape[0]
    ks = rng.integers(0, K, N)
    poses = np.stack([starts[(ks - GAP * a) % K] for a in range(A)], axis=1)
    out = {'example_map': (em, None, wp[:, 1:3], torch_table(starts, dev), poses)}
    tracks = f110.trackgen.random_tracks(21, 4)
    stacked, _ = f110.trackgen.device_maps(tracks, dev)
    ids = np.arange(N) % 4
    st = [np.stack([t.start_pose(k) for k in range(t.waypoints.shape[0])]) for t in tracks]
    ks = rng.integers(0, 10 ** 6, N)
    poses = np.stack([np.stack([st[l][(k - GAP * a) % st[l].shape[0]] for a in range(A)]) for l, k in zip(ids, ks)])
    out['tracks4_generated'] = (stacked, ids, [t.waypoints for t in tracks], [torch_table(s, dev) for s in st], poses)
    return out


def torch_table(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def make_sim(f110, dev, dmap, ids, poses, centerline):
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, device=dev, noise_std=0.0)
    sim.set_device_map(dmap, env_map_ids=ids)
    sim.set_centerlines(centerline)
    sim.env_reset(poses)
    return sim


def time_events(fn, flush, reps, warmup, before=None):
    import torch
    for _ in range(warmup):
        if before:
            before()
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        if before:
            before()
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return {'ms_mean': round(float(np.mean(ms)), 5), 'ms_median': round(float(np.median(ms)), 5),
            'ms_min': round(float(np.min(ms)), 5), 'ms_max': round(float(np.max(ms)), 5)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--ticks', type=int, default=100)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100', 'bench_progress.json'))
    args = ap.parse_args()
    import torch
    import f1tenth_gym_b200 as f110
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    flush = torch.empty(FLUSH_BYTES, dtype=torch.uint8, device=dev)
    result = {'metric': 'track_progress', 'card': gpu_card(), 'envs': N, 'agents': A, 'window': [8, 56],
              'reps': args.reps, 'workloads': []}
    rng = np.random.default_rng(SEED + 1)
    act = torch.from_numpy(np.stack([rng.uniform(-0.3, 0.3, N * A), rng.uniform(1.0, 6.0, N * A)], axis=1)).to(dev)
    for name, (dmap, ids, centerline, tables, poses) in workloads(f110, dev).items():
        sim = make_sim(f110, dev, dmap, ids, poses, centerline)
        ar = tables
        for _ in range(50):
            sim.tick(act, env_level=True, autoreset_poses=ar, pose_gap=GAP, seed=SEED)
            sim.update_progress()
        torch.cuda.synchronize()
        seg_snapshot = sim.track_seg.clone()
        tracked = float((sim.steer_cnt != 0).double().mean().item())
        w = {'workload': name, 'segments': sim.centerlines.num_segments, 'tracked_fraction': round(tracked, 4)}
        w['update_tracking'] = time_events(sim.update_progress, flush, args.reps, args.warmup,
                                           before=lambda: sim.track_seg.copy_(seg_snapshot))
        w['update_acquiring'] = time_events(sim.update_progress, flush, args.reps, args.warmup,
                                            before=lambda: sim.track_seg.fill_(-1))
        sim.track_seg.copy_(seg_snapshot)
        # the tick with and without the update, as CUDA graphs of two identical simulators, alternated
        plain = make_sim(f110, dev, dmap, ids, poses, centerline)
        with_p = make_sim(f110, dev, dmap, ids, poses, centerline)
        abuf = act.clone()
        graphs = {'tick': plain.capture_graph(abuf, autoreset_poses=ar, pose_gap=GAP, autoreset_seed=SEED, env_level=True),
                  'tick_with_update': with_p.capture_graph(abuf, autoreset_poses=ar, pose_gap=GAP, autoreset_seed=SEED,
                                                           env_level=True, progress=True)}
        for g in graphs.values():
            for _ in range(20):
                g.replay()
        torch.cuda.synchronize()
        per = {k: [] for k in graphs}
        for _ in range(args.rounds):
            for k, g in graphs.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.ticks):
                    g.replay()
                b.record()
                b.synchronize()
                per[k].append(a.elapsed_time(b) / args.ticks)
        for k, v in per.items():
            w[k] = {'ms_per_tick_mean': round(float(np.mean(v)), 5), 'ms_per_tick_min': round(float(np.min(v)), 5),
                    'ms_per_tick_max': round(float(np.max(v)), 5), 'rounds': args.rounds, 'ticks_per_round': args.ticks}
        assert torch.equal(plain.state, with_p.state) and torch.equal(plain.scans, with_p.scans)
        w['tick_outputs_identical'] = True
        result['workloads'].append(w)
        del sim, plain, with_p, graphs
        torch.cuda.synchronize()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
