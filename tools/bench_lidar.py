"""Agents without a lidar on the H100: one captured tick per policy step with the lidar mask all / ego only / none.

    python tools/bench_lidar.py [--out profiles/h100/bench_lidar.json] [--blocks 6] [--replays 100] [--quick]

Workloads cfg3 (16384 x 2) and cfg2x2 (4096 x 2) with the masks all / ego / none, cfg2 (4096 x 1) with all / none, on
example_map without scan noise (the short path needs it off); policies random actions (the benchmark policy) and pure pursuit on
every slot.  Per workload and policy every arm runs in the same process from the same reset, one CUDA graph of one tick with the
env level and the auto-reset per arm, alternated in blocks of replays timed with CUDA events after a warm-up; the report holds
the median and the spread of the blocks per arm.  Within a workload the hash of state, collisions, lap arrays and done must be
equal across the arms, and so must the hash of the scans of the slots that have a lidar in the arm: the script fails otherwise.
Per-kernel times come from torch.profiler over un-captured ticks (a run of its own), and the fraction of sensorless agents listed
for the iTTC march from f110_lidar.listed.  The card's name, power limit and clocks are read in the same run.  Without a GPU it
fails; --dry-run parses the arguments and prints the plan.
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

WORKLOADS = {'cfg3': (16384, 2, ('all', 'ego', 'none')), 'cfg2x2': (4096, 2, ('all', 'ego', 'none')),
             'cfg2': (4096, 1, ('all', 'none'))}
POLICIES = ('random', 'pure_pursuit')
POSE_GAP, SEED = 23, 12345
KERNELS = ('k_dynamics', 'k_lidar_order', 'k_march_lean', 'k_ttc_select', 'k_march_ttc', 'k_lidar_cast', 'k_tail_noscan', 'k_tail2',
           'k_tail<')


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100', 'bench_lidar.json'))
    ap.add_argument('--workloads', default=','.join(WORKLOADS))
    ap.add_argument('--blocks', type=int, default=6, help='timed blocks per arm, alternated')
    ap.add_argument('--replays', type=int, default=100, help='graph replays (ticks) per block')
    ap.add_argument('--warmup', type=int, default=100, help='ticks before the first timed block')
    ap.add_argument('--quick', action='store_true', help='cfg2 only, two blocks')
    ap.add_argument('--dry-run', action='store_true')
    a = ap.parse_args(argv)
    a.workloads = [w for w in a.workloads.split(',') if w]
    for w in a.workloads:
        if w not in WORKLOADS:
            ap.error('unknown workload %r' % w)
    if a.blocks < 1 or a.replays < 1:
        ap.error('blocks and replays >= 1')
    if a.quick:
        a.workloads, a.blocks = ['cfg2'], 2
    return a


def mask_of(name, A):
    return {'all': None, 'ego': [i == 0 for i in range(A)], 'none': [False] * A}[name]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


class Arm(object):
    def __init__(self, f110, torch, dev, dmap, poses, table, mask, policy):
        N, A = poses.shape[:2]
        self.torch, self.N, self.A, self.policy = torch, N, A, policy
        self.mask = [True] * A if mask is None else mask
        self.sim = sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, device=dev)
        sim.set_device_map(dmap)
        sim.env_reset(poses)
        sim.set_lidar(mask)
        self.table = table
        self.abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
        self.gen = torch.Generator(device=dev)
        self.gen.manual_seed(SEED)
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
            # the reference example's settings (examples/waypoint_follow.py: lookahead 0.82461887897713965, vgain 0.90338203837889)
            self.planner.plan_into(sim.state[0], sim.state[1], sim.state[4], 0.82461887897713965, 0.90338203837889, self.abuf)

    def steps(self, n, eager=False):
        for _ in range(n):
            self.act()
            if eager:
                self.sim.tick(self.abuf, autoreset_poses=self.table, pose_gap=POSE_GAP, seed=SEED)
            else:
                self.sim.replay()

    def digests(self):
        s = self.sim
        h = hashlib.sha1()
        for t in (s.state, s.collisions, s.collision_idx, s.lap_times, s.lap_counts, s.toggle_list, s.done):
            h.update(t.cpu().numpy().tobytes())
        on = [i for i in range(self.A) if self.mask[i]]
        scans = s.scans.view(self.N, self.A, -1)[:, on].cpu().numpy()
        return h.hexdigest(), on, scans


def kernel_times(torch, arm, steps=20):
    """Mean device time per launch of the tick's kernels over un-captured ticks (torch.profiler, a run of its own)."""
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
    N, A, masks = WORKLOADS[workload]
    dmap, poses, table = case
    arms = {m: Arm(f110, torch, dev, dmap, poses, table, mask_of(m, A), policy) for m in masks}
    for arm in arms.values():
        arm.steps(a.warmup)
    torch.cuda.synchronize()
    for arm in arms.values():
        if arm.sim.lidar_listed is not None:
            arm.sim.lidar_listed.zero_()
    times = {m: [] for m in arms}
    for _ in range(a.blocks):
        for m, arm in arms.items():              # alternated: all, ego, none, all, ...
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arm.steps(a.replays)
            e1.record()
            e1.synchronize()
            times[m].append(e0.elapsed_time(e1) * 1e3 / a.replays)
    ref_hash, _, ref_scans = arms['all'].digests()
    row = {'workload': workload, 'policy': policy, 'envs': N, 'agents': A, 'arms': {}}
    ok = True
    ticks = a.blocks * a.replays
    for m, arm in arms.items():
        h, on, scans = arm.digests()
        same_state = h == ref_hash
        same_scans = bool(np.array_equal(scans.view(np.int32), ref_scans[:, on].view(np.int32)))
        ok = ok and same_state and same_scans
        med = statistics.median(times[m])
        sensorless = N * (A - len(on))
        listed = arm.sim.lidar_listed
        arm.sim.tick(arm.abuf, autoreset_poses=table, pose_gap=POSE_GAP, seed=SEED)     # one eager tick for the launch record
        row['arms'][m] = {'us_per_tick': round(med, 2), 'min': round(min(times[m]), 2), 'max': round(max(times[m]), 2),
                          'agent_steps_per_s': round(N * A / (med * 1e-6)), 'state_hash_equal': same_state,
                          'lidar_scans_equal': same_scans,
                          'listed_fraction': (float(listed.item()) / (ticks * sensorless)) if (listed is not None and sensorless)
                          else None,
                          'launch': f110._native.lib().f110_debug_last_launch().decode()}
    for m, arm in arms.items():
        row['arms'][m]['kernel_us'] = kernel_times(torch, arm)
    row['speedup_vs_all'] = {m: round(row['arms']['all']['us_per_tick'] / row['arms'][m]['us_per_tick'], 3) for m in arms}
    return row, ok


def build_case(f110, torch, dev, workload):
    N, A, _ = WORKLOADS[workload]
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
        print(json.dumps({'plan': todo, 'out': a.out}))
        return 0
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_lidar needs a CUDA device: timings on anything else mean nothing')
    import f1tenth_gym_b200 as f110
    dev = torch.device('cuda:0')
    report = {'card': card(), 'blocks': a.blocks, 'replays_per_block': a.replays, 'warmup_ticks': a.warmup, 'rows': []}
    ok = True
    for workload, policy in todo:
        row, good = measure(f110, torch, dev, a, workload, policy, build_case(f110, torch, dev, workload))
        print(json.dumps(row), flush=True)
        report['rows'].append(row)
        ok = ok and good
    report['card_after'] = card()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, 'w') as f:
        json.dump(report, f, indent=1)
    print(json.dumps({'card': report['card'], 'rows': len(report['rows']), 'all_hashes_equal': ok}))
    return 0 if ok else 1


if __name__ == '__main__':
    sys.exit(main())
