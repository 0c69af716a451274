"""k_tail2 on the H100: its time per tick under the default block shape and under forced shapes (f110_debug_set_tail2).

    python tools/bench_tail2.py [--workloads cfg3,cfg2x2] [--shapes default,128:-8,128:-42] [--rounds 4] [--ticks 20]
                                [--out FILE]

Each workload is set up as bench.py sets it up (example_map, 1080 beams, raceline start poses with the second agent 23 waypoints
behind, random actions, auto-reset on an ego collision).  A shape is `default` or `threads:agents`, passed to
f110_debug_set_tail2 as they are: a negative agent count forces that many agents per block exactly, bypassing the whole-wave rule.
Ticks run through Simulator.step_profile, which times k_dynamics, the ray march and the tail with CUDA events, with the L2 flushed
before each tick as bench.py flushes it.  The shapes are alternated in rounds of `--ticks` ticks each; the report holds, per shape,
the median tail time over all its ticks and the spread of the round medians.  The card's name and power limit are read in the
same run.  Without a GPU it fails.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {'cfg3': (16384, 2), 'cfg2x2': (4096, 2), 'cfg3_a3': (16384, 3), 'cfg3_a4': (16384, 4)}
POSE_GAP, SEED, BEAMS = 23, 12345, 1080
FLUSH_BYTES = 256 << 20


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--workloads', default='cfg3,cfg2x2')
    ap.add_argument('--shapes', default='default')
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--ticks', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--out', default=None)
    a = ap.parse_args(argv)
    a.workloads = [w for w in a.workloads.split(',') if w]
    for w in a.workloads:
        if w not in WORKLOADS:
            ap.error('unknown workload %r' % w)
    a.shapes = [s for s in a.shapes.split(',') if s]
    for s in a.shapes:
        if s != 'default' and len(s.split(':')) != 2:
            ap.error('bad shape %r' % s)
    return a


def card():
    q = 'name,power.limit,clocks.max.sm'
    r = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None


def set_shape(L, shape):
    if shape == 'default':
        L.f110_debug_set_tail2(256, 64)          # the built-in rule
    else:
        t, ag = (int(x) for x in shape.split(':'))
        L.f110_debug_set_tail2(t, ag)


def run_workload(name, args, f110, torch, L):
    N, A = WORKLOADS[name]
    dev = torch.device('cuda:0')
    dmap = f110.DeviceMap.from_yaml(f110.maps.resolve_map_path('example_map'), '.png', dev)
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, num_beams=BEAMS, device=dev)
    sim.set_device_map(dmap)
    wp_np = f110.maps.load_waypoints()
    wp = torch.from_numpy(wp_np).to(dev)
    ks = np.array([np.random.default_rng(SEED + e).integers(0, wp_np.shape[0]) for e in range(N)])
    sim.env_reset(np.stack([wp_np[(ks - POSE_GAP * i) % wp_np.shape[0]] for i in range(A)], axis=1))
    gen = torch.Generator(device=dev)
    gen.manual_seed(SEED)
    flush = torch.empty(FLUSH_BYTES, dtype=torch.uint8, device=dev)

    def tick():
        u = torch.rand((N, A, 2), generator=gen, device=dev, dtype=torch.float64)
        u[..., 0] = -0.4189 + 0.8378 * u[..., 0]
        u[..., 1] = 8.0 * u[..., 1]
        flush.zero_()
        d = sim.step_profile(u)
        sim.env_post_step()
        sim.autoreset(wp, POSE_GAP, SEED)
        return d

    set_shape(L, 'default')
    for _ in range(args.warmup):
        tick()
    per = {s: [] for s in args.shapes}
    rounds = {s: [] for s in args.shapes}
    for _ in range(args.rounds):
        for s in args.shapes:
            set_shape(L, s)
            tick()                                  # first tick of a shape: not timed
            ms = [tick()[2] for _ in range(args.ticks)]
            per[s] += ms
            rounds[s].append(statistics.median(ms))
    set_shape(L, 'default')
    out = {}
    for s in args.shapes:
        out[s] = {'tail_us_median': 1e3 * statistics.median(per[s]),
                  'round_medians_us': [1e3 * x for x in rounds[s]],
                  'spread_us': 1e3 * (max(rounds[s]) - min(rounds[s]))}
    return out


def main(argv=None):
    args = parse(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_tail2: no GPU')
    import f1tenth_gym_b200 as f110
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    res = {'card': card(), 'workloads': {}}
    for w in args.workloads:
        res['workloads'][w] = run_workload(w, args, f110, torch, L)
        print(w, json.dumps(res['workloads'][w]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
