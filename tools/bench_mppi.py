"""Time one MPPI planner iteration (f110_mppi_sample, f110_predict_scored, f110_mppi_update, each with CUDA events) against the
scoring route available without the scored rollout: predict(record_states, record_clearance), project_centerline on every
predicted pose, then the cost, softmin weights and weighted mean in torch.  Writes profiles/h100/bench_mppi.json (or --out)
with the card name and power limit read in the same run.

    python tools/bench_mppi.py [--maps example_map,tracks4] [--M 256,4096] [--K 64,256,1024] [--H 10,30] [--reps 5] [--out PATH]

Per (map, M, K, H): microseconds of each planner launch, of f110_predict on the same samples (the rollout without the cost),
of the route, the route's peak memory, and how far
the route's costs are from the scored ones (the route projects every pose globally where the scored rollout tracks a window,
so the two differ where the global projection jumps to another part of the track).  The route is skipped (null) where it does
not fit in memory.  example_map tracks its bundled waypoints; tracks4 has no bundled centerlines, so each layer tracks an
ellipse around its cars (the timing depends on the table size and the re-acquire rate, not on the shape).  Then the closed
loop of tests/test_gpu_mppi.py (tick + pure pursuit + MPPI for the ego, H = 30, K = 256) as a replayed CUDA graph: ticks per
second at 64 and 1024 envs x 2 agents.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from bench_predict import card, load_map   # noqa: E402


def event_time(fn, reps):
    """Median microseconds of fn between two CUDA events over reps calls, after one warm-up call."""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1) * 1000.0)
    return round(float(np.median(t)), 1)


def route_cost(sim, ids, act, w, L):
    """The cost of include/f110_mppi.h from recorded futures, with a global projection of every pose, in torch."""
    M, K, H = act.shape[:3]
    out = sim.predict(act, agent_ids=ids, record_states=True, record_clearance=True)
    st = out['states']
    ids_t = torch.as_tensor(ids, device=st.device, dtype=torch.long)
    src = sim.state[:, ids_t].t()[:, [0, 1, 4]]
    tables = None
    if sim.centerlines.num_tables > 1:
        layer = sim.env_layer.long()[ids_t // sim.num_agents]
        tables = torch.cat([layer, layer.repeat_interleave(K * H)]).int()
    poses = torch.cat([src, st[..., [0, 1, 4]].reshape(-1, 3)])
    proj = sim.project_centerline(poses, table_ids=tables)
    s0 = proj[:M, 3]
    p = proj[M:].reshape(M, K, H, 5)
    s = torch.cat([s0[:, None, None].expand(M, K, 1), p[..., 3]], dim=2)
    Lm = L[sim.env_layer.long()[ids_t // sim.num_agents]] if tables is not None else torch.full((M,), L[0], device=st.device,
                                                                                                    dtype=torch.float64)
    delta = s[..., 1:] - s[..., :-1]
    half = (Lm * 0.5)[:, None, None]
    delta = torch.where(delta > half, delta - Lm[:, None, None], torch.where(delta < -half, delta + Lm[:, None, None], delta))
    u = act
    du = torch.cat([torch.zeros_like(u[:, :, :1]), u[:, :, 1:] - u[:, :, :-1]], dim=2)
    pen = torch.clamp(w['clear_min'] - out['clearance'].double(), min=0.0)
    c = (w['w_lat'] * p[..., 2] ** 2 + w['w_head'] * p[..., 4] ** 2 + w['w_clear'] * pen ** 2 + w['w_dsteer'] * du[..., 0] ** 2
         + w['w_dspeed'] * du[..., 1] ** 2).sum(2) - w['w_prog'] * delta.sum(2) + (out['wall_step'] >= 0) * w['w_wall']
    c = torch.where(torch.isfinite(c), c, torch.full_like(c, float('inf')))
    wk = torch.exp(-(c - c.min(1, keepdim=True).values) / 1.0)
    U = (wk[:, :, None, None] * act).sum(1) / wk.sum(1)[:, None, None]
    return c, U


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--maps', default='example_map,tracks4')
    ap.add_argument('--M', default='256,4096')
    ap.add_argument('--K', default='64,256,1024')
    ap.add_argument('--H', default='10,30')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--loop-ticks', type=int, default=500)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100', 'bench_mppi.json'))
    a = ap.parse_args()
    import f1tenth_gym_b200 as f110
    from f1tenth_gym_b200 import _native as nat
    from test_gpu_multimap import mixed_population
    from test_gpu_mppi import closed_loop, layer_centerlines
    import ctypes as C
    dev = torch.device('cuda:0')
    name, power = card()
    rows = []
    w = dict(f110.simulator.COST_DEFAULTS)
    L = nat.lib()
    for mname in a.maps.split(','):
        dm, hosts = load_map(f110, dev, mname)
        for M in (int(v) for v in a.M.split(',')):
            rng = np.random.default_rng(0)
            layers = np.arange(M) % len(hosts)
            sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 1, num_envs=M, device=dev)
            sim.set_device_map(dm, env_map_ids=layers if len(hosts) > 1 else None)
            if mname == 'example_map':
                wp = f110.maps.load_waypoints()
                sim.reset(wp[rng.integers(0, wp.shape[0], M)][:, None, :])
                sim.set_centerlines(wp[:, :2])
            else:
                sim.reset(mixed_population(hosts, layers, rng, 1))
                sim.set_centerlines(layer_centerlines(sim, layers, len(hosts)))
            for _ in range(20):
                sim.step(np.stack([rng.uniform(-0.1, 0.1, (M, 1)), rng.uniform(1, 4, (M, 1))], axis=2))
            Ls = torch.as_tensor([r[-1, 5] + r[-1, 6] for r in
                                  [f110.simulator.centerline_segments(t)[0] for t in
                                   ([wp[:, :2]] if mname == 'example_map' else layer_centerlines(sim, layers, len(hosts)))]],
                                 device=dev, dtype=torch.float64)
            ids = np.arange(M)
            for K in (int(v) for v in a.K.split(',')):
                for H in (int(v) for v in a.H.split(',')):
                    p = f110.MPPIPlanner(sim, ids, H, K, seed=1)
                    p._nominal[..., 1] = 3.0
                    st = f110.simulator._stream_ptr(dev)
                    out = torch.zeros((M, 2), dtype=torch.float64, device=dev)
                    t_sample = event_time(lambda: L.f110_mppi_sample(C.byref(sim.c), C.byref(p._mppi_c), None,
                                                                     nat.ptr(p.samples_actions), st), a.reps)
                    t_pred = event_time(lambda: L.f110_predict_scored(
                        C.byref(sim.c), C.byref(sim._map_struct), C.byref(sim._march_tables), C.byref(sim.beams.c),
                        C.byref(sim.centerlines.c), C.byref(p._args), C.byref(p._cost_c), st), a.reps)
                    t_plain = event_time(lambda: L.f110_predict(
                        C.byref(sim.c), C.byref(sim._map_struct), C.byref(sim._march_tables), C.byref(sim.beams.c),
                        C.byref(p._args), st), a.reps)
                    t_update = event_time(lambda: L.f110_mppi_update(C.byref(p._mppi_c), nat.ptr(p.samples_actions),
                                                                     nat.ptr(p.cost), nat.ptr(out), M, None, None, st), a.reps)
                    t_iter = event_time(lambda: p.plan_into(out), a.reps)
                    # the route without the scored rollout, on the samples the planner drew last
                    L.f110_mppi_sample(C.byref(sim.c), C.byref(p._mppi_c), None, nat.ptr(p.samples_actions), st)
                    L.f110_predict_scored(C.byref(sim.c), C.byref(sim._map_struct), C.byref(sim._march_tables),
                                          C.byref(sim.beams.c), C.byref(sim.centerlines.c), C.byref(p._args),
                                          C.byref(p._cost_c), st)
                    act = p.samples_actions
                    scored = p.cost.clone()
                    row = dict(map=mname, M=M, K=K, H=H, sample_us=t_sample, scored_predict_us=t_pred, predict_us=t_plain, update_us=t_update,
                               iteration_us=t_iter, nan_cost_share=float(torch.isnan(scored).float().mean()))
                    try:
                        torch.cuda.synchronize()
                        torch.cuda.reset_peak_memory_stats()
                        base = torch.cuda.memory_allocated()
                        t_route = event_time(lambda: route_cost(sim, ids, act, w, Ls), a.reps)
                        peak = torch.cuda.max_memory_allocated() - base
                        c_route, _ = route_cost(sim, ids, act, w, Ls)
                        fin = torch.isfinite(scored) & torch.isfinite(c_route)
                        diff = (c_route - scored).abs()[fin]
                        rel = diff / scored.abs()[fin].clamp(min=1.0)
                        row.update(route_us=t_route, route_peak_bytes=int(peak),
                                   route_differs_share=float((rel > 1e-9).float().mean()),
                                   route_max_rel_diff=float(rel.max()) if rel.numel() else None)
                        del c_route
                    except torch.cuda.OutOfMemoryError:
                        row.update(route_us=None, route_peak_bytes=None)
                    sim._predict_buf = None
                    torch.cuda.empty_cache()
                    print(json.dumps(row), flush=True)
                    rows.append(row)
                    del p
            del sim
            torch.cuda.empty_cache()
    loop = []
    for N in (64, 1024):
        for graph in (True,):
            import time
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            closed_loop(f110, dev, N, a.loop_ticks, 'mppi', graph=graph)
            dt = time.perf_counter() - t0
            r = dict(envs=N, agents=2, ticks=a.loop_ticks, graph=graph, ticks_per_s_incl_setup=round(a.loop_ticks / dt, 1))
            # steady state: time a second run's replays only
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            closed_loop(f110, dev, N, 2 * a.loop_ticks, 'mppi', graph=graph)
            dt2 = time.perf_counter() - t0
            r['ticks_per_s'] = round(a.loop_ticks / max(dt2 - dt, 1e-9), 1)
            print(json.dumps(r), flush=True)
            loop.append(r)
    res = dict(gpu=name, power_limit=power, cost=w, rows=rows, closed_loop=loop)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(dict(gpu=name, power_limit=power, rows=len(rows))))


if __name__ == '__main__':
    main()
