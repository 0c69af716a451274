"""What static box obstacles cost on the flagship workload: 16384 envs x 2 agents on example_map, 1080 beams, a captured
graph with lap logic and auto-reset (bench.py's cfg3), random actions and pure pursuit (the actions are computed between the
replays, inside the timed window), K in {0, 1, 4, 8} boxes per env drawn from obstacle_candidates along example_waypoints.csv
and redrawn at every auto-reset; and K = 4 under tick_repeat(a, 4).

    python tools/bench_obstacles.py [--ticks 400] [--warmup 50] [--out profiles/h100/bench_obstacles.json]

Reports per case the time per tick from CUDA events around whole timed windows of graph replays, the fraction of agents with
a present box within max_range + half its diagonal (the ones k_obstacles clips against), the GPU name and power limit read in
the same run, and the times of k_obstacles and k_env_tail_obst: CUDA events the library records around the two launches
(f110_debug_set_obst_events) over un-captured ticks after the timed window, mean per tick.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import f1tenth_gym_b200 as f110     # noqa: E402

N, A, SEED, POSE_GAP = 16384, 2, 12345, 23


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(','))
        return name, limit
    except Exception as e:      # the card name still comes from torch
        return torch.cuda.get_device_name(0), 'unknown (%s)' % e


def run(dmap, K, repeat, ticks, warmup, dev, policy='random', kernel_ticks=50):
    wp = f110.maps.load_waypoints()
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, device=dev)
    sim.set_device_map(dmap)
    rng = np.random.default_rng(SEED)
    ks = rng.integers(0, wp.shape[0], N)
    sim.env_reset(np.stack([wp[(ks - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1))
    if K:
        cand = f110.obstacle_candidates(wp[:, :2], 4096, lateral=(-0.8, 0.8), seed=SEED)
        sim.set_obstacles(np.zeros((K, 5)), np.zeros(K, bool))
        sim.set_obstacle_draw(cand, count=(K, K), clearance=2.0, seed=SEED)
        sim.respawn_obstacles()
    tab = torch.from_numpy(wp).to(dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(SEED)
    pool = torch.rand((64, N * A, 2), generator=gen, device=dev, dtype=torch.float64)
    pool[..., 0] = -0.4189 + 0.8378 * pool[..., 0]
    pool[..., 1] = 8.0 * pool[..., 1]
    abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
    planner = None
    if policy == 'pure_pursuit':
        from f1tenth_gym_b200.planner import PurePursuitPlanner
        planner = PurePursuitPlanner(device=dev)

    def act(t):
        if planner is None:
            abuf.copy_(pool[t % 64])
        else:
            planner.plan_into(sim.state[0], sim.state[1], sim.state[4], 0.82461887897713965, 0.90338203837889, abuf)
    sim.capture_graph(abuf, autoreset_poses=tab, pose_gap=POSE_GAP, autoreset_seed=SEED, env_level=True, repeat=repeat)
    calls = max(1, ticks // repeat)
    for t in range(max(1, warmup // repeat)):
        act(t)
        sim.replay()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    near = 0.0
    e0.record()
    for t in range(calls):
        act(t)
        sim.replay()
    e1.record()
    torch.cuda.synchronize(dev)
    ms = e0.elapsed_time(e1)
    if K:
        b, on = sim.obstacle_boxes, sim.obstacle_active.bool()
        xy = sim.state[:2].T.reshape(N, A, 1, 2)
        d = torch.linalg.norm(b[:, None, :, :2] - xy, dim=-1)
        reach = dmap.c.max_range + 0.5 * torch.linalg.norm(b[:, :, 3:5], dim=-1)[:, None, :]
        near = float(((d <= reach) & on[:, None, :]).any(-1).double().mean())
    k_obst = k_tail = None
    if K and repeat == 1:
        L = f110._native.lib()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        for e in ev:
            e.record()      # creates the CUDA event behind e.cuda_event
        L.f110_debug_set_obst_events(*[e.cuda_event for e in ev])
        k_obst = k_tail = 0.0
        try:
            for t in range(kernel_ticks):
                act(t)
                sim.tick(abuf, env_level=True, autoreset_poses=tab, pose_gap=POSE_GAP, seed=SEED)
                torch.cuda.synchronize(dev)
                k_obst += ev[0].elapsed_time(ev[1]) * 1e3 / kernel_ticks
                k_tail += ev[1].elapsed_time(ev[2]) * 1e3 / kernel_ticks
        finally:
            L.f110_debug_set_obst_events(None, None, None)
    return dict(K=K, repeat=repeat, policy=policy, ticks=calls * repeat, us_per_tick=1e3 * ms / (calls * repeat),
                agents_with_box_in_range=near, k_obstacles_us=k_obst, k_env_tail_obst_us=k_tail)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ticks', type=int, default=400)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--out', default=os.path.join('profiles', 'h100', 'bench_obstacles.json'))
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    dmap = f110.DeviceMap.from_yaml(os.path.join(os.path.dirname(f110.__file__), 'maps', 'example_map.yaml'), '.png', dev)
    name, limit = card()
    cases = [run(dmap, K, 1, args.ticks, args.warmup, dev, pol) for pol in ('random', 'pure_pursuit') for K in (0, 1, 4, 8)]
    cases += [run(dmap, K, 4, args.ticks, args.warmup, dev) for K in (0, 4)]
    out = dict(gpu=name, power_limit=limit, workload='cfg3: 16384 x 2, example_map, 1080 beams, graph, lap logic + auto-reset',
               cases=cases)
    for c in cases:
        print(json.dumps(c))
    os.makedirs(os.path.dirname(args.out) or '.', exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(dict(gpu=name, power_limit=limit)))


if __name__ == '__main__':
    main()
