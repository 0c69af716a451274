"""CPU model of k_tail2's opponent ray-cast: how many beams a task visits, and how many beam intervals its record needs.

    python tools/tail_cast_study.py [--envs 16384] [--seed 0]

Poses as bench.py's cfg3 draws them: raceline waypoints of example_map with the second agent 23 waypoints behind, plus 0.3 m or
1.5 m of position jitter and a matching yaw jitter.  Per (ego, opponent) pair it restates phase 1 of k_tail2 in numpy: the
opponent's corners, get_blocked_view_indices (nearest beam of each corner), the wide-window cone asin(half_diag / dist) + 0.05
and the intervals around (phi - yaw) + m pi that the record stores.  It reports the share of wide windows, the beams visited per
env, the warp iterations per env that the warp-per-ego loop needed (ceil(len / 32) per interval), and the beams saved if the
cone's 0.05 rad slack or the mirror intervals (m odd) were dropped.  `task_intervals` is the restatement the host tests use for
the interval-count bound.  No GPU is used.
"""
import argparse
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

IVALS = 4            # F110_TAIL2_IVALS


def task_intervals(lo, hi, phi, yaw, cone, fov, angle_increment, ivals=IVALS):
    """k_tail2 phase 1: the beam intervals of one task -> (list of (i0, i1), whole).  `whole`: the task visits [lo, hi] (a narrow
    window, cone >= 3.5, or more intervals than the record holds)."""
    if not (cone < 3.5 and hi - lo >= 96):
        return [(lo, hi)], True
    d = phi - yaw
    base = d - 2 * math.pi * np.rint(d * (1.0 / (2 * math.pi)))
    half, inv_inc = fov / 2., 1.0 / angle_increment
    m0 = max(-3, int(math.floor((-half - cone - 0.02 - base) * (1.0 / math.pi))))
    m1 = min(5, int(math.ceil((half + cone + 0.02 - base) * (1.0 / math.pi))))
    out, nxt = [], lo
    for m in range(m0, m1 + 1):
        c = base + m * math.pi
        f0, f1 = (c - cone + half) * inv_inc - 2.0, (c + cone + half) * inv_inc + 2.0
        if f1 < lo or f0 > hi:
            continue
        i0, i1 = max(nxt, int(math.floor(max(f0, lo)))), min(hi, int(math.ceil(min(f1, hi))))
        if i0 > i1:
            continue
        if len(out) == ivals:
            return [(lo, hi)], True
        out.append((i0, i1))
        nxt = i1 + 1
    return out, False


def corners(x, y, th, length, width):
    c, s = math.cos(th), math.sin(th)
    pts = []
    for sl, sw in ((1, 1), (1, -1), (-1, -1), (-1, 1)):
        pts.append((x + sl * c * length / 2 - sw * s * width / 2, y + sl * s * length / 2 + sw * c * width / 2))
    return pts


def nearest_beam(angle, B, fov, inc):
    return int(min(max(round((angle + fov / 2) / inc), 0), B - 1))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--envs', type=int, default=16384)
    ap.add_argument('--seed', type=int, default=0)
    a = ap.parse_args(argv)
    from f1tenth_gym_b200 import maps
    wp = maps.load_waypoints()
    p = maps.DEFAULT_PARAMS
    length, width = p['length'], p['width']
    half_diag = 0.5 * math.hypot(length, width)
    B, fov = 1080, 4.7
    inc = fov / (B - 1)
    rng = np.random.default_rng(a.seed)
    for jit in (0.3, 1.5):
        k = rng.integers(0, wp.shape[0], a.envs)
        wide = visited = iters = no_slack = no_mirror = 0
        for e in range(a.envs):
            pos = [wp[(k[e] - 23 * i) % wp.shape[0]] + np.r_[rng.normal(0, jit, 2), rng.normal(0, jit / 5)] for i in range(2)]
            for ego in range(2):
                x, y, yaw = pos[ego]
                ox, oy, oth = pos[1 - ego]
                dist = math.hypot(ox - x, oy - y)
                if dist > 30.0 + half_diag:
                    continue
                idx = []
                for cx, cy in corners(ox, oy, oth, length, width):
                    ang = math.atan2(math.sin(yaw), math.cos(yaw)) - math.atan2(cy - y, cx - x)
                    ang = ang - 2 * math.pi if ang > math.pi else ang + 2 * math.pi if ang < -math.pi else ang
                    idx.append(nearest_beam(-ang, B, fov, inc))
                lo, hi = min(idx), max(idx)
                phi = math.atan2(oy - y, ox - x)
                cone = 4.0
                if hi - lo >= 96 and dist > 1.25 * half_diag:
                    cone = math.asin(half_diag / dist) + 0.05
                iv, _ = task_intervals(lo, hi, phi, yaw, cone, fov, inc)
                wide += hi - lo >= 96
                n = sum(i1 - i0 + 1 for i0, i1 in iv)
                visited += n
                iters += sum((i1 - i0) // 32 + 1 for i0, i1 in iv)
                if hi - lo >= 96 and cone < 3.5:
                    ivs, _ = task_intervals(lo, hi, phi, yaw, cone - 0.05, fov, inc)
                    no_slack += n - sum(i1 - i0 + 1 for i0, i1 in ivs)
                    # the mirror intervals: those whose centre is nearer (phi - yaw) + pi than (phi - yaw), modulo 2 pi
                    for i0, i1 in iv:
                        mid = -fov / 2 + 0.5 * (i0 + i1) * inc
                        dd = (mid - (phi - yaw) + math.pi) % (2 * math.pi) - math.pi
                        if abs(dd) > math.pi / 2:
                            no_mirror += i1 - i0 + 1
        print('jitter %.1f m: wide windows %.1f %% of egos, %.1f beams and %.2f warp iterations per env, '
              'slack 0.05 rad = %.1f %% of beams, mirror intervals = %.1f %% of beams' % (
                  jit, 100.0 * wide / (2 * a.envs), visited / a.envs, iters / a.envs, 100.0 * no_slack / max(visited, 1),
                  100.0 * no_mirror / max(visited, 1)))


if __name__ == '__main__':
    main()
