#!/usr/bin/env python
"""Same-box A/B of the ray-march kernel variants (measurement aid, not the product path).

    python tools/ab_march.py [--workloads cfg2,cfg3] [--variants 0,1,20,21,22,6] [--ticks 40] > gpurun_out/ab_march.json

For every (workload, variant): reset to the same start poses, replay the same action sequence, time each kernel of
the tick with CUDA events (f110_step_profile, L2 flushed between ticks) and the whole tick as a CUDA-graph replay,
and hash the scans / state so that the variants are shown to produce identical results.
Variants (F110_MARCH_VARIANT): 0 lean fp64 table, 64 warps/SM, 4 x 512 threads per SM, first half of every block's share dealt
statically and the rest claimed dynamically (--dyn static_pct:ahead); 66 / 60 / 61 static dealing with 4 x 512 / 2 x 1024 / 8 x 256
threads per SM; 42 dynamic with 2 x 1024; 62-65 thread-block clusters sharing
one ticket counter through DSMEM; 40 / 41 dynamic queue tail; 30 / 31 TMA tile; 21 lean at 48 warps/SM (40 registers);
20 / 22 lean, u8 rank-coded table + shared-memory LUT (64 / 48 warps); 1 round-1 persistent kernel; 6 round-1 coded;
7 no queue (block per 64-beam tile); 90 the padded row-major table instead of the 4 x 4-cell brick table (f110_march_tables);
30+ see csrc/f110_b200.cu.
The first and last lines name the card with its power limit and SM clock (nvidia-smi, read only).
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import re
import subprocess

import numpy as np   # noqa: E402
import torch         # noqa: E402

import bench         # noqa: E402
import f1tenth_gym_b200 as f110   # noqa: E402
from f1tenth_gym_b200 import _native as nat   # noqa: E402


def run(workload, variant, ticks, dev, chunk=3, dyn=(50, 4), pdl=0, tail=8, tail2=(256, 64), ipt=(-1, -1, -1, -1)):
    m = re.match(r'^n(\d+)a(\d+)(?:b(\d+))?$', workload)      # ad-hoc size: n<envs>a<agents>[b<beams>]
    w = dict(num_envs=int(m.group(1)), num_agents=int(m.group(2)), num_beams=int(m.group(3) or 1080)) if m else bench.WORKLOADS[workload]
    N, A, B = w['num_envs'], w['num_agents'], w['num_beams']
    NA = N * A
    L = nat.lib()
    L.f110_debug_set_variant(int(variant))
    L.f110_debug_set_chunk(int(chunk))
    L.f110_debug_set_dyn(int(dyn[0]), int(dyn[1]))
    L.f110_debug_set_pdl(int(pdl))
    L.f110_debug_set_ipt(*[int(x) for x in ipt])
    L.f110_debug_set_tail(int(tail))
    L.f110_debug_set_tail2(int(tail2[0]), int(tail2[1]))
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, bench.SEED, num_envs=N, num_beams=B, device=dev)
    sim.set_map(f110.maps.resolve_map_path('example_map'), '.png')
    wp_np = f110.maps.load_waypoints()
    wp = torch.from_numpy(wp_np).to(dev)
    ks = np.array([np.random.default_rng(bench.SEED + e).integers(0, wp_np.shape[0]) for e in range(N)])
    poses = np.stack([wp_np[(ks - bench.POSE_GAP * i) % wp_np.shape[0]] for i in range(A)], axis=1)
    sim.env_reset(poses)
    gen = torch.Generator(device=dev)
    gen.manual_seed(bench.SEED)
    P = 2 * ticks + 8
    u = torch.rand((P, NA, 2), generator=gen, device=dev, dtype=torch.float64)
    u[..., 0] = -0.4189 + 0.8378 * u[..., 0]
    u[..., 1] = 8.0 * u[..., 1]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    # settle (mixed speeds, resets) with the eager tick, timing each kernel
    kms = np.zeros(3)
    for t in range(ticks + 8):
        flush.zero_()
        d = sim.step_profile(u[t].view(N, A, 2))
        sim.env_post_step()
        sim.autoreset(wp, bench.POSE_GAP, bench.SEED)
        if t >= 8:
            kms += np.array(d)
    kms /= ticks
    torch.cuda.synchronize(dev)
    h = hashlib.sha1()
    h.update(sim.scans.cpu().numpy().tobytes())
    h.update(sim.state.cpu().numpy().tobytes())
    h.update(sim.collisions.cpu().numpy().tobytes())
    # whole tick as a graph replay
    abuf = torch.zeros((NA, 2), dtype=torch.float64, device=dev)
    sim.capture_graph(abuf, autoreset_poses=wp, pose_gap=bench.POSE_GAP, autoreset_seed=bench.SEED, env_level=True)
    ev0 = [torch.cuda.Event(enable_timing=True) for _ in range(ticks)]
    ev1 = [torch.cuda.Event(enable_timing=True) for _ in range(ticks)]
    for t in range(5):
        abuf.copy_(u[ticks + 8 + t]); sim.replay()
    for t in range(ticks):
        flush.zero_()
        abuf.copy_(u[(ticks + 8 + t) % P])
        ev0[t].record(); sim.replay(); ev1[t].record()
    torch.cuda.synchronize(dev)
    tick_us = 1e3 * float(np.median([a.elapsed_time(b) for a, b in zip(ev0, ev1)]))
    return {'workload': workload, 'variant': variant, 'chunk': chunk, 'dyn': list(dyn), 'pdl': pdl, 'tail_minb': tail, 'tail2': list(tail2), 'ipt': list(ipt), 'dyn_us': 1e3 * kms[0], 'march_us': 1e3 * kms[1],
            'tail_us': 1e3 * kms[2], 'tick_graph_us': tick_us, 'agent_steps_per_s': NA / (tick_us * 1e-6),
            'hash': h.hexdigest()[:16]}


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu'
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', '0'], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = 'nvidia-smi failed: %s' % e
    return {'card': torch.cuda.get_device_name(0), 'nvidia_smi': dict(zip(q.split(','), [x.strip() for x in out.split(',')]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='cfg2,cfg2x2,cfg3')
    ap.add_argument('--variants', default='1,0,21,20,22')
    ap.add_argument('--chunks', default='3')
    ap.add_argument('--dyn', default='50:4', help='static_pct:ahead[,static_pct:ahead...] for the dynamic-tail variants 40/41')
    ap.add_argument('--pdl', default='0')
    ap.add_argument('--tail', default='8', help='k_tail register budget: 4 (128 regs), 5 (96), 8 (64); -1 = always k_tail, -2 = always the two-phase k_tail2')
    ap.add_argument('--tail2', default='256:64', help='k_tail2 block shape threads:agents[,threads:agents...]')
    ap.add_argument('--ipt', default='-1:-1:-1:-1', help='log2(entries per ticket) veryheavy:heavy:light:dyntail[,...] for variant 0; -1 = default (0:1:2:by class)')
    ap.add_argument('--ticks', type=int, default=40)
    ap.add_argument('--repeat', type=int, default=2)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    print(json.dumps(card()), flush=True)
    rows = []
    for wl in args.workloads.split(','):
        for rep in range(args.repeat):
            for v in [int(x) for x in args.variants.split(',')]:
                for ch in [int(x) for x in args.chunks.split(',')]:
                    for dy in (args.dyn.split(',') if v in (0, 40, 41, 42, 43, 45, 57, 58) or 81 <= v <= 86 else ['50:4']):
                        for pdl in [int(x) for x in args.pdl.split(',')]:
                            for tl in [int(x) for x in args.tail.split(',')]:
                                for t2 in args.tail2.split(','):
                                    for ip in (args.ipt.split(',') if v == 0 else ['-1:-1:-1:-1']):
                                        r = run(wl, v, args.ticks, dev, ch, tuple(int(x) for x in dy.split(':')), pdl, tl,
                                                tuple(int(x) for x in t2.split(':')), tuple(int(x) for x in ip.split(':')))
                                        r['rep'] = rep
                                        rows.append(r)
                                        print(json.dumps(r), flush=True)
        hs = {r['hash'] for r in rows if r['workload'] == wl}
        print(json.dumps({'workload': wl, 'identical_results_across_variants': len(hs) == 1}), flush=True)
    print(json.dumps(card()), flush=True)


if __name__ == '__main__':
    main()
