"""Episodes under a held action on the H100: captured calls of tick_repeat in episode mode against captured tick_repeat calls
with the in-call auto-reset.

    python tools/bench_episode_repeat.py [--out profiles/h100/bench_episode_repeat.json] [--blocks 6] [--replays 50] [--quick]

Workloads cfg3 (16384 x 2) and cfg2x2 (4096 x 2) on example_map without scan noise; K in {2, 4, 8}; policies random actions (the
benchmark policy) and pure pursuit on every slot.  Arms: 'autoreset' (f110_tick_repeat with the start table, as a frame-skip
loop without episodes runs it) and 'episodes' (f110_tick_repeat_episodes without a time limit, so that both arms end envs on
the same events).  Per workload, K and policy both arms run in the same process from the same reset, one CUDA graph of
one call per arm, alternated in blocks of replays timed with CUDA events after a warm-up; the report holds the median and the
spread of the blocks per arm, the share of envs per call that ended on a tick before the last (episodes) and per-kernel times
from torch.profiler over un-captured calls (a run of its own).  A twin check then runs both arms eagerly from one reset under
one action stream and compares, after every call, a hash of the state rows of the envs that neither arm ended.  The card's
name, power limit and clocks are read in the same run.  Without a GPU it fails; --dry-run prints the plan.
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
REPEATS = (2, 4, 8)
ARMS = ('autoreset', 'episodes')
POSE_GAP, SEED = 23, 12345
KERNELS = ('k_dynamics', 'k_ttc_select', 'k_march_ttc', 'k_march_lean', 'k_tail_noscan', 'k_tail2', 'k_repeat_done',
           'k_episode_latch', 'k_episode_restart', 'k_episode_dyn', 'k_restart_march', 'k_episode_cast', 'k_episode_tail')


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100', 'bench_episode_repeat.json'))
    ap.add_argument('--workloads', default=','.join(WORKLOADS))
    ap.add_argument('--repeats', default=','.join(str(k) for k in REPEATS))
    ap.add_argument('--blocks', type=int, default=6, help='timed blocks per arm, alternated')
    ap.add_argument('--replays', type=int, default=50, help='graph replays per block')
    ap.add_argument('--warmup', type=int, default=50, help='calls per arm before timing')
    ap.add_argument('--quick', action='store_true', help='2 blocks of 10 replays, 10 warm-up calls')
    ap.add_argument('--dry-run', action='store_true')
    a = ap.parse_args(argv)
    a.workloads = [w for w in a.workloads.split(',') if w]
    a.repeats = [int(k) for k in a.repeats.split(',') if k]
    if a.quick:
        a.blocks, a.replays, a.warmup = 2, 10, 10
    return a


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


class Arm(object):
    def __init__(self, f110, torch, dev, dmap, poses, table, K, episodes, policy, capture=True):
        N, A = poses.shape[:2]
        self.torch, self.N, self.A, self.K, self.policy, self.episodes = torch, N, A, K, policy, episodes
        self.sim = sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, device=dev)
        sim.set_device_map(dmap)
        sim.env_reset(poses)
        if episodes:
            sim.set_episodes(0)
        self.table = table
        self.abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
        self.gen = torch.Generator(device=dev)
        self.gen.manual_seed(SEED)
        self.mid = torch.zeros((), dtype=torch.int64, device=dev)
        if policy == 'pure_pursuit':
            self.planner = f110.PurePursuitPlanner(device=dev)
        if capture:
            sim.capture_graph(self.abuf, autoreset_poses=table, pose_gap=POSE_GAP, autoreset_seed=SEED, env_level=True, repeat=K)

    def act(self):
        torch, sim = self.torch, self.sim
        if self.policy == 'random':
            u = torch.rand((self.N * self.A, 2), generator=self.gen, device=self.abuf.device, dtype=torch.float64)
            self.abuf[:, 0] = -0.4189 + 0.8378 * u[:, 0]
            self.abuf[:, 1] = 8.0 * u[:, 1]
        else:
            self.planner.plan_into(sim.state[0], sim.state[1], sim.state[4], 0.82461887897713965, 0.90338203837889, self.abuf)

    def call(self):
        return self.sim.tick_repeat(self.abuf, self.K, autoreset_poses=self.table, pose_gap=POSE_GAP, seed=SEED)

    def steps(self, n, eager=False, count=False):
        s = self.sim
        for _ in range(n):
            self.act()
            if eager:
                self.call()
            else:
                s.replay()
            if count and self.episodes:     # device-side sums: no host synchronisation inside the counted stretch
                self.mid += ((s.end_tick >= 0) & (s.end_tick < self.K - 1)).sum()


def kernel_times(torch, arm, calls=10):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        arm.steps(calls, eager=True)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in KERNELS:
            if name in e.key:
                t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
                out.setdefault(name, [0.0, 0])
                out[name][0] += t
                out[name][1] += e.count
    # microseconds per call (all launches of the kernel in a call) and launches per call
    return {k: {'us_per_call': round(v[0] / calls, 2), 'launches_per_call': round(v[1] / calls, 2)} for k, v in out.items()}


def twin_hashes(f110, torch, dev, case, K, policy, calls=30):
    """Both arms eagerly from one reset under the autoreset arm's actions: after each call, a hash of the state rows of the envs
    that neither arm ended (the autoreset arm: done on no tick of the call; the episode arm: end_tick = -1) must agree."""
    dmap, poses, table = case
    x = Arm(f110, torch, dev, dmap, poses, table, K, False, policy, capture=False)
    y = Arm(f110, torch, dev, dmap, poses, table, K, True, policy, capture=False)
    equal, compared = True, 0
    for _ in range(calls):
        x.act()
        y.abuf.copy_(x.abuf)
        ox, oy = x.call(), y.call()
        keep = (ox['done_any'] == 0) & (oy['end_tick'] < 0)
        sx, sy = x.sim.state.view(7, x.N, x.A)[:, keep], y.sim.state.view(7, y.N, y.A)[:, keep]
        hx = int(sx.contiguous().view(torch.int64).sum().item())
        hy = int(sy.contiguous().view(torch.int64).sum().item())
        equal = equal and hx == hy and torch.equal(sx, sy)
        compared += int(keep.sum().item())
        # the envs either arm ended restart differently: continue both from the autoreset arm's state
        for n in ('state', 'steer_buf', 'steer_cnt', 'current_time', 'lap_times', 'lap_counts', 'toggle_list', 'near_starts',
                  'start_xs', 'start_ys', 'start_thetas', 'start_rot', 'done', 'checkpoint_done', 'collisions', 'collision_idx',
                  'wall_flag', 'scans', 'tick_counter'):
            getattr(y.sim, n).copy_(getattr(x.sim, n))
        y.sim.ep_ticks.zero_()
    return {'equal': bool(equal), 'env_calls_compared': compared}


def measure(f110, torch, dev, a, workload, K, policy, case):
    N, A = WORKLOADS[workload]
    dmap, poses, table = case
    arms = {m: Arm(f110, torch, dev, dmap, poses, table, K, m == 'episodes', policy) for m in ARMS}
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
    arms['episodes'].mid.zero_()
    arms['episodes'].steps(a.replays, count=True)
    row = {'workload': workload, 'K': K, 'policy': policy, 'envs': N, 'agents': A, 'arms': {}}
    for m, arm in arms.items():
        med = statistics.median(times[m])
        arm.call()      # one eager call for the launch record
        row['arms'][m] = {'us_per_call': round(med, 2), 'min': round(min(times[m]), 2), 'max': round(max(times[m]), 2),
                          'launch': f110._native.lib().f110_debug_last_launch().decode()}
    row['arms']['episodes']['ended_mid_call_share'] = float(arms['episodes'].mid.item()) / (a.replays * N)
    for m, arm in arms.items():
        row['arms'][m]['kernel_us'] = kernel_times(torch, arm)
    row['episodes_vs_autoreset'] = round(row['arms']['episodes']['us_per_call'] / row['arms']['autoreset']['us_per_call'] - 1.0, 4)
    row['non_ended_state_hash'] = twin_hashes(f110, torch, dev, case, K, policy)
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
    todo = [(w, K, p) for w in a.workloads for K in a.repeats for p in POLICIES]
    if a.dry_run:
        print(json.dumps({'plan': todo, 'arms': list(ARMS), 'out': a.out}))
        return 0
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_episode_repeat needs a CUDA device: timings on anything else mean nothing')
    import f1tenth_gym_b200 as f110
    dev = torch.device('cuda:0')
    report = {'card': card(), 'blocks': a.blocks, 'replays_per_block': a.replays, 'warmup_calls': a.warmup, 'rows': []}
    cases = {}
    for workload, K, policy in todo:
        if workload not in cases:
            cases[workload] = build_case(f110, torch, dev, workload)
        row = measure(f110, torch, dev, a, workload, K, policy, cases[workload])
        print(json.dumps({k: v for k, v in row.items() if k != 'arms'} |
                         {m: row['arms'][m]['us_per_call'] for m in ARMS}), flush=True)
        report['rows'].append(row)
    report['card_after'] = card()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, 'w') as f:
        json.dump(report, f, indent=1)
    print(json.dumps({'card': report['card'], 'rows': len(report['rows'])}))
    return 0


if __name__ == '__main__':
    sys.exit(main())
