"""Action repeat on the H100: K plain ticks in one CUDA graph against tick_repeat(K) in one CUDA graph.

    python tools/bench_repeat.py [--out profiles/h100/bench_repeat.json] [--blocks 6] [--replays 40] [--quick]

Workloads cfg3 (16384 x 2), cfg2 (4096 x 1), cfg2x2 (4096 x 2) on example_map and tracks4 (4096 x 2 on the four-track
canvas); K in {1, 2, 4, 8}; random actions (the benchmark policy) and, on example_map, pure pursuit.  Per workload and K both
arms run in the same process from the same reset, alternated in blocks of graph replays timed with CUDA events; the report holds
the median and the spread of the blocks per arm, agent-physics-steps/s, the marched fraction (device counter), per-kernel
times of the short path (torch.profiler, a run of its own) and a hash of state + final scans that must match between the arms.
The card's name and power limit are read in the same run.  Without a GPU it fails; --dry-run parses the arguments and prints
the plan.
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {'cfg3': ('example_map', 16384, 2), 'cfg2': ('example_map', 4096, 1), 'cfg2x2': ('example_map', 4096, 2),
             'tracks4': ('tracks4', 4096, 2)}
TRACKS = [('berlin', '.png'), ('vegas', '.png'), ('skirk', '.png'), ('levine', '.pgm')]
KS = (1, 2, 4, 8)
POSE_GAP, SEED = 23, 12345


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100', 'bench_repeat.json'))
    ap.add_argument('--workloads', default=','.join(WORKLOADS))
    ap.add_argument('--ks', default=','.join(str(k) for k in KS))
    ap.add_argument('--blocks', type=int, default=6, help='timed blocks per arm, alternated')
    ap.add_argument('--replays', type=int, default=40, help='graph replays (policy steps) per block')
    ap.add_argument('--warmup', type=int, default=60, help='policy steps before the first timed block')
    ap.add_argument('--quick', action='store_true', help='cfg2 only, K = 4, two blocks')
    ap.add_argument('--dry-run', action='store_true')
    a = ap.parse_args(argv)
    a.workloads = [w for w in a.workloads.split(',') if w]
    a.ks = [int(k) for k in a.ks.split(',') if k]
    for w in a.workloads:
        if w not in WORKLOADS:
            ap.error('unknown workload %r' % w)
    if any(not 1 <= k <= 64 for k in a.ks) or a.blocks < 1 or a.replays < 1:
        ap.error('K in [1, 64], blocks and replays >= 1')
    if a.quick:
        a.workloads, a.ks, a.blocks = ['cfg2'], [4], 2
    return a


def plan(a):
    return [(w, pol, k) for w in a.workloads for pol in (('random', 'pure_pursuit') if WORKLOADS[w][0] == 'example_map' else ('random',))
            for k in a.ks]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


class Arm(object):
    """One simulator and its captured graph: `repeat` = K runs tick_repeat(K), 0 runs K plain ticks in one graph."""

    def __init__(self, f110, torch, dev, dmap, ids, poses, tables, K, short, policy, wp):
        N, A = poses.shape[:2]
        self.torch, self.K, self.N, self.A, self.policy = torch, K, N, A, policy
        self.sim = sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, device=dev)
        sim.set_device_map(dmap, env_map_ids=ids)
        sim.env_reset(poses)
        self.abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
        self.gen = torch.Generator(device=dev)
        self.gen.manual_seed(SEED)
        if policy == 'pure_pursuit':
            from f1tenth_gym_b200.planner import PurePursuitPlanner
            self.planner = PurePursuitPlanner(device=dev)
        if short:
            sim.capture_graph(self.abuf, autoreset_poses=tables, pose_gap=POSE_GAP, autoreset_seed=SEED, env_level=True, repeat=K)
            self.graph = sim._graph
        else:
            sim.capture_graph(self.abuf, autoreset_poses=tables, pose_gap=POSE_GAP, autoreset_seed=SEED, env_level=True)
            one = sim._graph
            # K plain ticks in ONE graph: captured from K replays' worth of launches
            L, C, nat = f110._native.lib(), __import__('ctypes'), f110._native
            table, n = sim._start_table(tables)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(K):
                    nat.check(L.f110_tick_ex(C.byref(sim.c), C.byref(sim._map_struct), C.byref(sim._march_tables),
                                             C.byref(sim.beams.c), nat.ptr(self.abuf), 1, nat.ptr(table), n, POSE_GAP, SEED,
                                             C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
            self.graph, self._keep = g, (one, table)

    def act(self):
        torch, sim = self.torch, self.sim
        if self.policy == 'random':
            u = torch.rand((self.N * self.A, 2), generator=self.gen, device=self.abuf.device, dtype=torch.float64)
            self.abuf[:, 0] = -0.4189 + 0.8378 * u[:, 0]
            self.abuf[:, 1] = 8.0 * u[:, 1]
        else:
            # the reference example's settings (examples/waypoint_follow.py: lookahead 0.82461887897713965, vgain 0.90338203837889)
            self.planner.plan_into(sim.state[0], sim.state[1], sim.state[4], 0.82461887897713965, 0.90338203837889, self.abuf)

    def steps(self, n):
        for _ in range(n):
            self.act()
            self.graph.replay()

    def digest(self):
        h = hashlib.sha1()
        h.update(self.sim.state.cpu().numpy().tobytes())
        h.update(self.sim.scans.cpu().numpy().tobytes())
        return h.hexdigest()


def build_case(f110, torch, dev, workload):
    maps_dir = os.path.join(ROOT, 'f1tenth_gym_b200', 'maps')
    kind, N, A = WORKLOADS[workload]
    rng = np.random.default_rng(N + A)
    if kind == 'example_map':
        dmap = f110.DeviceMap.from_yaml(os.path.join(maps_dir, 'example_map.yaml'), '.png', dev)
        wp = f110.maps.load_waypoints()
        k = rng.integers(0, wp.shape[0], N)
        poses = np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1)
        return dmap, None, poses, torch.from_numpy(wp).to(dev), wp
    layers = [f110.DeviceMap.from_yaml(os.path.join(maps_dir, n + '.yaml'), e, dev) for n, e in TRACKS]
    ids = np.arange(N) % len(layers)
    tabs = []
    for m in layers:
        h = m.host
        free = np.argwhere(h.dt >= 0.6)
        sel = free[rng.choice(free.shape[0], 256, replace=False)]
        tabs.append(np.stack([sel[:, 1] * h.resolution + h.orig_x + 0.013, sel[:, 0] * h.resolution + h.orig_y + 0.007,
                              rng.uniform(0, 2 * np.pi, 256)], axis=1))
    poses = np.zeros((N, A, 3))
    for e in range(N):
        t = tabs[ids[e]]
        j = rng.integers(0, t.shape[0])
        for i in range(A):
            poses[e, i] = t[(j - POSE_GAP * i) % t.shape[0]]
    return f110.DeviceMap.stack(layers), ids, poses, [torch.from_numpy(t).to(dev) for t in tabs], None


def kernel_times(torch, arm, steps=10):
    """Mean device time per launch of the short path's kernels, from torch.profiler (a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        arm.steps(steps)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in ('k_ttc_select', 'k_march_ttc', 'k_tail_noscan', 'k_dynamics', 'k_march_lean', 'k_tail2', 'k_tail<'):
            if name in e.key:
                t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
                out.setdefault(name, [0.0, 0])
                out[name][0] += t
                out[name][1] += e.count
    return {k: round(v[0] / max(v[1], 1), 2) for k, v in out.items()}


def measure(f110, torch, dev, a, workload, policy, K, case):
    dmap, ids, poses, tables, wp = case
    arms = {'plain': Arm(f110, torch, dev, dmap, ids, poses, tables, K, False, policy, wp),
            'repeat': Arm(f110, torch, dev, dmap, ids, poses, tables, K, True, policy, wp)}
    for arm in arms.values():
        arm.steps(a.warmup)
    torch.cuda.synchronize()
    assert arms['plain'].digest() == arms['repeat'].digest(), 'the arms diverged during the warm-up'
    if K > 1:
        arms['repeat'].sim.marched_agents.zero_()
    times = {k: [] for k in arms}
    for _ in range(a.blocks):
        for name, arm in arms.items():           # alternated: plain, repeat, plain, repeat, ...
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arm.steps(a.replays)
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e3 / a.replays)
    N, A = poses.shape[:2]
    steps = a.blocks * a.replays
    marched = float(arms['repeat'].sim.marched_agents.item()) / max(1, steps * (K - 1) * N * A) if K > 1 else None
    same = arms['plain'].digest() == arms['repeat'].digest()
    row = {'workload': workload, 'policy': policy, 'K': K, 'envs': N, 'agents': A, 'hash_equal': same,
           'marched_fraction': marched, 'launch': f110._native.lib().f110_debug_last_launch().decode()}
    for name, ts in times.items():
        med = statistics.median(ts)
        row[name] = {'us_per_policy_step': round(med, 2), 'min': round(min(ts), 2), 'max': round(max(ts), 2),
                     'agent_physics_steps_per_s': round(N * A * K / (med * 1e-6))}
    row['speedup'] = round(row['plain']['us_per_policy_step'] / row['repeat']['us_per_policy_step'], 3)
    if K > 1:
        row['kernel_us'] = kernel_times(torch, arms['repeat'])
    return row


def main(argv=None):
    a = parse(argv)
    todo = plan(a)
    if a.dry_run:
        print(json.dumps({'plan': todo, 'out': a.out}))
        return 0
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_repeat needs a CUDA device: timings on anything else mean nothing')
    import f1tenth_gym_b200 as f110
    dev = torch.device('cuda:0')
    rows, cases = [], {}
    for workload, policy, K in todo:
        if workload not in cases:
            cases = {workload: build_case(f110, torch, dev, workload)}
        row = measure(f110, torch, dev, a, workload, policy, K, cases[workload])
        print(json.dumps(row), flush=True)
        rows.append(row)
    report = {'card': card(), 'blocks': a.blocks, 'replays_per_block': a.replays, 'warmup_steps': a.warmup, 'rows': rows}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, 'w') as f:
        json.dump(report, f, indent=1)
    ok = all(r['hash_equal'] for r in rows)
    print(json.dumps({'card': report['card'], 'rows': len(rows), 'all_hashes_equal': ok}))
    return 0 if ok else 1


if __name__ == '__main__':
    sys.exit(main())
