"""Episode mode on the H100: a captured episode tick against today's captured tick with the auto-reset.

    python tools/bench_episodes.py [--out profiles/h100/bench_episodes.json] [--blocks 6] [--replays 100] [--quick]

Workloads cfg3 (16384 x 2) and cfg2x2 (4096 x 2) on example_map without scan noise; policies random actions (the benchmark
policy) and pure pursuit on every slot.  Arms: 'autoreset' (f110_tick_lidar with the start table, as bench.py replays it) and
'episodes' with max_ticks 0 and 200 (f110_tick_episodes).  Per workload and policy every arm runs in the same process from the
same reset, one CUDA graph of one tick per arm, alternated in blocks of replays timed with CUDA events after a warm-up; the
report holds the median and the spread of the blocks per arm, the restarted share of envs per tick (episode arms: envs that
ended, counted over the blocks; the auto-reset arm: envs whose ego collided) and per-kernel times from torch.profiler over
un-captured ticks (a run of its own).  The card's name, power limit and clocks are read in the same run.  Without a GPU it
fails; --dry-run parses the arguments and prints the plan.
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
ARMS = (('autoreset', None), ('episodes_max0', 0), ('episodes_max200', 200))
POSE_GAP, SEED = 23, 12345
KERNELS = ('k_dynamics', 'k_march_lean', 'k_tail2', 'k_episode_end', 'k_episode_dyn', 'k_restart_march', 'k_episode_cast',
           'k_episode_tail')


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100', 'bench_episodes.json'))
    ap.add_argument('--workloads', default=','.join(WORKLOADS))
    ap.add_argument('--blocks', type=int, default=6, help='timed blocks per arm, alternated')
    ap.add_argument('--replays', type=int, default=100, help='graph replays per block')
    ap.add_argument('--warmup', type=int, default=200, help='ticks per arm before timing')
    ap.add_argument('--quick', action='store_true', help='2 blocks of 20 replays, 20 warm-up ticks')
    ap.add_argument('--dry-run', action='store_true')
    a = ap.parse_args(argv)
    a.workloads = [w for w in a.workloads.split(',') if w]
    if a.quick:
        a.blocks, a.replays, a.warmup = 2, 20, 20
    return a


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


class Arm(object):
    def __init__(self, f110, torch, dev, dmap, poses, table, max_ticks, policy):
        N, A = poses.shape[:2]
        self.torch, self.N, self.A, self.policy, self.episodes = torch, N, A, policy, max_ticks is not None
        self.sim = sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, device=dev)
        sim.set_device_map(dmap)
        sim.env_reset(poses)
        if self.episodes:
            sim.set_episodes(max_ticks)
        self.table = table
        self.abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
        self.gen = torch.Generator(device=dev)
        self.gen.manual_seed(SEED)
        self.ended = torch.zeros((), dtype=torch.int64, device=dev)
        if policy == 'pure_pursuit':
            self.planner = f110.PurePursuitPlanner(device=dev)
        sim.capture_graph(self.abuf, autoreset_poses=table, pose_gap=POSE_GAP, autoreset_seed=SEED, env_level=True)

    def act(self):
        torch, sim = self.torch, self.sim
        if self.policy == 'random':
            u = torch.rand((self.N * self.A, 2), generator=self.gen, device=self.abuf.device, dtype=torch.float64)
            self.abuf[:, 0] = -0.4189 + 0.8378 * u[:, 0]
            self.abuf[:, 1] = 8.0 * u[:, 1]
        else:
            self.planner.plan_into(sim.state[0], sim.state[1], sim.state[4], 0.82461887897713965, 0.90338203837889, self.abuf)

    def steps(self, n, eager=False, count=False):
        s = self.sim
        for _ in range(n):
            self.act()
            if eager:
                s.tick(self.abuf, autoreset_poses=self.table, pose_gap=POSE_GAP, seed=SEED)
            else:
                s.replay()
            if count:           # device-side sums: no host synchronisation inside the timed block
                if self.episodes:
                    self.ended += (s.ep_terminated | s.ep_truncated).sum()
                else:
                    self.ended += (s.collisions.view(self.N, self.A)[:, 0] != 0).sum()


def kernel_times(torch, arm, steps=20):
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
    return {k: round(v[0] / max(v[1], 1), 2) for k, v in out.items()}


def measure(f110, torch, dev, a, workload, policy, case):
    N, A = WORKLOADS[workload]
    dmap, poses, table = case
    arms = {name: Arm(f110, torch, dev, dmap, poses, table, T, policy) for name, T in ARMS}
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
    # the restarted share over a separate, counted stretch (the sums are extra launches, kept out of the timed blocks)
    for arm in arms.values():
        arm.ended.zero_()
        arm.steps(a.replays, count=True)
    row = {'workload': workload, 'policy': policy, 'envs': N, 'agents': A, 'arms': {}}
    for m, arm in arms.items():
        med = statistics.median(times[m])
        arm.sim.tick(arm.abuf, autoreset_poses=table, pose_gap=POSE_GAP, seed=SEED)      # one eager tick for the launch record
        row['arms'][m] = {'us_per_tick': round(med, 2), 'min': round(min(times[m]), 2), 'max': round(max(times[m]), 2),
                          'restarted_share_per_tick': float(arm.ended.item()) / (a.replays * N),
                          'launch': f110._native.lib().f110_debug_last_launch().decode()}
    for m, arm in arms.items():
        row['arms'][m]['kernel_us'] = kernel_times(torch, arm)
    base = row['arms']['autoreset']['us_per_tick']
    row['cost_vs_autoreset'] = {m: round(row['arms'][m]['us_per_tick'] / base - 1.0, 4) for m in arms}
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
    todo = [(w, p) for w in a.workloads for p in POLICIES]
    if a.dry_run:
        print(json.dumps({'plan': todo, 'arms': [m for m, _ in ARMS], 'out': a.out}))
        return 0
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_episodes needs a CUDA device: timings on anything else mean nothing')
    import f1tenth_gym_b200 as f110
    dev = torch.device('cuda:0')
    report = {'card': card(), 'blocks': a.blocks, 'replays_per_block': a.replays, 'warmup_ticks': a.warmup, 'rows': []}
    for workload, policy in todo:
        row = measure(f110, torch, dev, a, workload, policy, build_case(f110, torch, dev, workload))
        print(json.dumps(row), flush=True)
        report['rows'].append(row)
    report['card_after'] = card()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, 'w') as f:
        json.dump(report, f, indent=1)
    print(json.dumps({'card': report['card'], 'rows': len(report['rows'])}))
    return 0


if __name__ == '__main__':
    sys.exit(main())
