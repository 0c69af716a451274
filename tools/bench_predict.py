"""Time Simulator.predict against the route it replaces: copy the source rows into a sensorless replica of M * K envs x 1 agent,
then H ticks.  Writes profiles/h100/bench_predict.json (or --out) with the card name and power limit read in the same run.

    python tools/bench_predict.py [--maps example_map,tracks4] [--K 64,256,1024] [--H 10,30] [--reps 5] [--out PATH]

Per (map, K, H, distribution): microseconds per call of each arm, sample-steps per second, the share of sample-steps that
failed the pre-test (marched; from the replica's listed-agent count), and a hash of final_state / wall_step that must be equal
between the arms.  Distributions: 'held' (each car's current steering and speed held, plus noise) and 'uniform' (uniform random
actions).  The replica arm is skipped (route_us null) where the tick refuses a replica that large (M * K * beams >= 2^32).
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (v.strip() for v in out.split(','))
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), 'unknown'


def load_map(f110, dev, name):
    maps = os.path.join(ROOT, 'f1tenth_gym_b200', 'maps')
    if name == 'tracks4':
        from test_gpu_multimap import TRACKS
        layers = [f110.DeviceMap.from_yaml(os.path.join(maps, n + '.yaml'), e, dev) for n, e in TRACKS]
        return f110.DeviceMap.stack(layers), [m.host for m in layers]
    m = f110.DeviceMap.from_yaml(os.path.join(maps, name + '.yaml'), '.png', dev)
    return m, [m.host]


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1000.0)
    return float(np.median(times))


def digest(*ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.contiguous().cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--maps', default='example_map,tracks4')
    ap.add_argument('--M', type=int, default=4096)
    ap.add_argument('--K', default='64,256,1024')
    ap.add_argument('--H', default='10,30')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100', 'bench_predict.json'))
    a = ap.parse_args()
    import f1tenth_gym_b200 as f110
    from test_gpu_multimap import mixed_population
    dev = torch.device('cuda:0')
    name, power = card()
    rows = []
    for mname in a.maps.split(','):
        dm, hosts = load_map(f110, dev, mname)
        N, A = a.M, 1
        layers = np.arange(N) % len(hosts)
        rng = np.random.default_rng(0)
        src = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 1, num_envs=N, device=dev)
        src.set_device_map(dm, env_map_ids=layers if len(hosts) > 1 else None)
        src.reset(mixed_population(hosts, layers, rng, A))
        for _ in range(20):
            src.step(np.stack([rng.uniform(-0.2, 0.2, (N, A)), rng.uniform(1, 5, (N, A))], axis=2))
        M = N * A
        for K in (int(v) for v in a.K.split(',')):
            rep = None
            for H in (int(v) for v in a.H.split(',')):
                for dist in ('held', 'uniform'):
                    if dist == 'uniform':
                        act = np.stack([rng.uniform(-0.4189, 0.4189, (M, K, H)), rng.uniform(-5, 20, (M, K, H))], axis=3)
                    else:       # the current steering and speed held, with noise: mostly wall-free futures
                        st = src.state.cpu().numpy()
                        base = np.stack([st[2], np.maximum(st[3], 2.0)], axis=1)[:, None, None, :]
                        act = base + rng.normal(0, 1, (M, K, H, 2)) * np.array([0.03, 0.5])
                    act = torch.as_tensor(np.ascontiguousarray(act), device=dev)
                    t_pred = timed(lambda: src.predict(act), a.reps)
                    out = src.predict(act)
                    h_pred = digest(out['final_state'], out['wall_step'])
                    if rep is None:
                        rep = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 1, num_envs=M * K, device=dev)
                        rep.set_device_map(dm, env_map_ids=np.repeat(layers, K) if len(hosts) > 1 else None)
                        rep.set_lidar([False])
                    idx = torch.arange(M, device=dev).repeat_interleave(K)
                    acts = [act[:, :, h].reshape(M * K, 2).contiguous() for h in range(H)]

                    def route():
                        rep.state.copy_(src.state[:, idx])
                        rep.steer_buf.copy_(src.steer_buf[:, idx])
                        rep.steer_cnt.copy_(src.steer_cnt[idx])
                        for h in range(H):
                            rep.tick(acts[h], env_level=False)
                    try:
                        t_route = timed(route, a.reps)
                    except f110._native.F110Error:
                        row = dict(map=mname, M=M, K=K, H=H, dist=dist, predict_us=round(t_pred, 1), route_us=None,
                                   predict_sample_steps_per_s=M * K * H / (t_pred * 1e-6),
                                   wall_share=float((out['wall_step'] >= 0).float().mean()), hash_predict=h_pred, hash_route=None)
                        print(json.dumps(row), flush=True)
                        rows.append(row)
                        continue
                    walls = []
                    rep.state.copy_(src.state[:, idx]); rep.steer_buf.copy_(src.steer_buf[:, idx])
                    rep.steer_cnt.copy_(src.steer_cnt[idx])
                    listed = 0
                    for h in range(H):
                        rep.tick(acts[h], env_level=False)
                        walls.append(rep.wall_flag.clone())
                        listed += int(rep.lidar_list_count[0].item()) if rep.lidar_list_count is not None else 0
                    w = torch.stack(walls, 1) != 0
                    first = torch.where(w.any(1), w.int().argmax(1), torch.full_like(w[:, 0], -1, dtype=torch.int64)).int()
                    h_route = digest(rep.state.t().reshape(M, K, 7), first.reshape(M, K))
                    row = dict(map=mname, M=M, K=K, H=H, dist=dist, predict_us=round(t_pred, 1), route_us=round(t_route, 1),
                               predict_sample_steps_per_s=M * K * H / (t_pred * 1e-6),
                               marched_share=listed / float(M * K * H), wall_share=float((out['wall_step'] >= 0).float().mean()),
                               hash_predict=h_pred, hash_route=h_route)
                    print(json.dumps(row), flush=True)
                    rows.append(row)
            del rep
            torch.cuda.empty_cache()
    res = dict(gpu=name, power_limit=power, rows=rows)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(dict(gpu=name, power_limit=power, equal_hashes=all(r['hash_predict'] == r['hash_route'] for r in rows if r['hash_route']))))


if __name__ == '__main__':
    main()
