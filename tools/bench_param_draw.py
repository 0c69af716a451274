"""Per-episode parameter draws on the H100: what the per-env parameter table and the draw launch cost a captured call.

    python tools/bench_param_draw.py [--out profiles/h100/bench_param_draw.json] [--blocks 6] [--replays 100] [--quick]

Workloads cfg3 (16384 x 2) and cfg2x2 (4096 x 2) on example_map without scan noise; policies random actions (the benchmark
policy) and pure pursuit on every slot.  Modes: the plain auto-reset tick (f110_tick_lidar with the start table, as bench.py
replays it), the episode tick (f110_tick_episodes, max_ticks 200) and tick_repeat(a, 4) with the in-call auto-reset.  Arms:
'shared' (the [A][18] table), 'per_env' (the [N*A][18] table, no draws) and 'per_env_draw' (the same plus the draws of
Simulator.set_param_draw: mu, C_Sf, C_Sr, m, I, a_max, v_max, with m and I in one group).  Per workload, policy and mode every arm
runs in the same process from the same reset, one CUDA graph of one call per arm, alternated in blocks of replays timed with
CUDA events after a warm-up; the report holds the median and the spread of the blocks per arm, and the time per launch of
k_param_draw and k_dynamics from torch.profiler over un-captured calls (a run of its own).  The card's name, power limit and
clocks are read in the same run.  Without a GPU it fails; --dry-run parses the arguments and prints the plan.
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

WORKLOADS = {'cfg3': (16384, 2), 'cfg2x2': (4096, 2)}
POLICIES = ('random', 'pure_pursuit')
MODES = ('autoreset', 'episodes', 'repeat4')
ARMS = ('shared', 'per_env', 'per_env_draw')
POSE_GAP, SEED = 23, 12345
DRAW = {'mu': (0.6, 1.4), 'C_Sf': (3.5, 6.0), 'C_Sr': (4.0, 7.0), 'm': (3.0, 4.5), 'I': (0.035, 0.06), 'a_max': (6.0, 12.0),
        'v_max': (12.0, 25.0)}
KERNELS = ('k_param_draw', 'k_dynamics')


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100', 'bench_param_draw.json'))
    ap.add_argument('--workloads', default=','.join(WORKLOADS))
    ap.add_argument('--modes', default=','.join(MODES))
    ap.add_argument('--blocks', type=int, default=6, help='timed blocks per arm, alternated')
    ap.add_argument('--replays', type=int, default=100, help='graph replays per block')
    ap.add_argument('--warmup', type=int, default=100, help='calls per arm before timing')
    ap.add_argument('--quick', action='store_true', help='2 blocks of 20 replays, 20 warm-up calls')
    ap.add_argument('--dry-run', action='store_true')
    a = ap.parse_args(argv)
    a.workloads = [w for w in a.workloads.split(',') if w]
    a.modes = [m for m in a.modes.split(',') if m]
    if a.quick:
        a.blocks, a.replays, a.warmup = 2, 20, 20
    return a


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


class Arm(object):
    def __init__(self, f110, torch, dev, dmap, poses, table, mode, arm, policy):
        N, A = poses.shape[:2]
        self.torch, self.N, self.A, self.policy, self.mode = torch, N, A, policy, mode
        self.sim = sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, device=dev)
        sim.set_device_map(dmap)
        sim.env_reset(poses)
        if arm != 'shared':
            sim.update_params(f110.maps.DEFAULT_PARAMS, env_mask=np.ones(N, bool))
        if arm == 'per_env_draw':
            sim.set_param_draw(DRAW, groups=[['m', 'I']], seed=SEED)
            sim.redraw_params()
        if mode == 'episodes':
            sim.set_episodes(200)
        self.table = table
        self.K = 4 if mode == 'repeat4' else 1
        self.abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
        self.gen = torch.Generator(device=dev)
        self.gen.manual_seed(SEED)
        if policy == 'pure_pursuit':
            self.planner = f110.PurePursuitPlanner(device=dev)
        sim.capture_graph(self.abuf, autoreset_poses=table, pose_gap=POSE_GAP, autoreset_seed=SEED, env_level=True, repeat=self.K)

    def act(self):
        torch, sim = self.torch, self.sim
        if self.policy == 'random':
            u = torch.rand((self.N * self.A, 2), generator=self.gen, device=self.abuf.device, dtype=torch.float64)
            self.abuf[:, 0] = -0.4189 + 0.8378 * u[:, 0]
            self.abuf[:, 1] = 8.0 * u[:, 1]
        else:
            self.planner.plan_into(sim.state[0], sim.state[1], sim.state[4], 0.82461887897713965, 0.90338203837889, self.abuf)

    def steps(self, n, eager=False):
        s = self.sim
        for _ in range(n):
            self.act()
            if not eager:
                s.replay()
            elif self.K > 1:
                s.tick_repeat(self.abuf, self.K, autoreset_poses=self.table, pose_gap=POSE_GAP, seed=SEED)
            else:
                s.tick(self.abuf, autoreset_poses=self.table, pose_gap=POSE_GAP, seed=SEED)


def kernel_times(torch, arm, steps=20):
    """Mean device time per launch (us) and launches per call of each kernel in KERNELS."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        arm.steps(steps, eager=True)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in KERNELS:
            if name in e.key:
                t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
                out.setdefault(name, [0.0, 0])
                out[name][0] += t
                out[name][1] += e.count
    return {k: {'us_per_launch': round(v[0] / max(v[1], 1), 2), 'launches_per_call': v[1] / steps} for k, v in out.items()}


def measure(f110, torch, dev, a, workload, policy, mode, case):
    N, A = WORKLOADS[workload]
    dmap, poses, table = case
    arms = {name: Arm(f110, torch, dev, dmap, poses, table, mode, name, policy) for name in ARMS}
    for arm in arms.values():
        arm.steps(a.warmup)
    torch.cuda.synchronize()
    times = {m: [] for m in arms}
    for _ in range(a.blocks):
        for m, arm in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arm.steps(a.replays)
            e1.record()
            e1.synchronize()
            times[m].append(e0.elapsed_time(e1) * 1e3 / a.replays)
    row = {'workload': workload, 'policy': policy, 'mode': mode, 'envs': N, 'agents': A, 'arms': {}}
    for m, arm in arms.items():
        row['arms'][m] = {'us_per_call': round(statistics.median(times[m]), 2), 'min': round(min(times[m]), 2),
                          'max': round(max(times[m]), 2)}
    for m, arm in arms.items():
        row['arms'][m]['kernels'] = kernel_times(torch, arm)
    base = row['arms']['shared']['us_per_call']
    row['cost_vs_shared'] = {m: round(row['arms'][m]['us_per_call'] / base - 1.0, 4) for m in arms}
    for arm in arms.values():
        del arm.sim
    torch.cuda.empty_cache()
    return row


def build_case(f110, torch, dev, workload):
    N, A = WORKLOADS[workload]
    rng = np.random.default_rng(N + A)
    dmap = f110.DeviceMap.from_yaml(os.path.join(ROOT, 'f1tenth_gym_b200', 'maps', 'example_map.yaml'), '.png', dev)
    wp = f110.maps.load_waypoints()
    k = rng.integers(0, wp.shape[0], N)
    poses = np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1)
    return dmap, poses, torch.from_numpy(wp).to(dev)


def main(argv=None):
    a = parse(argv)
    todo = [(w, p, m) for w in a.workloads for p in POLICIES for m in a.modes]
    if a.dry_run:
        print(json.dumps({'plan': todo, 'arms': ARMS, 'out': a.out}))
        return 0
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_param_draw needs a CUDA device: timings on anything else mean nothing')
    import f1tenth_gym_b200 as f110
    dev = torch.device('cuda:0')
    report = {'card': card(), 'blocks': a.blocks, 'replays_per_block': a.replays, 'warmup_calls': a.warmup, 'rows': []}
    cases = {w: build_case(f110, torch, dev, w) for w in a.workloads}
    for workload, policy, mode in todo:
        row = measure(f110, torch, dev, a, workload, policy, mode, cases[workload])
        print(json.dumps(row), flush=True)
        report['rows'].append(row)
    report['card_after'] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, 'w') as f:
        json.dump(report, f, indent=1)
    print(json.dumps({'card': report['card'], 'rows': len(report['rows'])}))
    return 0


if __name__ == '__main__':
    sys.exit(main())
