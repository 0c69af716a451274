#!/usr/bin/env python
"""CPU model of the cell-unit ray march's DT gathers on a map, for choosing the layout of the table (DESIGN.md §3.2).

    python tools/march_layout_study.py [--map example_map] [--agents 96] [--lane-agents 384] [--layouts rowmajor,brick4x4]

Agents sit on the map's raceline (bundled waypoints) with N(0, 0.3 m) of position and N(0, 0.35 rad) of heading jitter; each
marches 1080 beams over 4.7 rad as the reference's trace_ray does (numpy fp64, lookups on the padded table: an off-map cell
reads dt[-1,-1]).  Printed:

  * lane figures, one warp per 32 consecutive beams of an agent: lookups per agent, and the busy share of the lanes
    (sum of lookups / (32 * sum over items of the longest beam)) for the beams in order, for an oracle that sorts every
    agent's beams by their own count, and for regroupings by the counts of the previous tick (the agents moved on by one
    timestep: 2 classes at several thresholds, 5 classes, fully sorted);
  * for every layout: distinct 32-byte sectors and distinct 128-byte lines that one warp gather touches (every gather
    with a live lane, the live lanes only).

A layout is a function (r, c, width) -> element index of cell (r, c) of the (H+1) x (W+1) padded fp64 table; add one to
LAYOUTS to study it.  Nothing here needs a GPU.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from f1tenth_gym_b200 import maps   # noqa: E402

B, FOV, MAX_RANGE, EPS = 1080, 4.7, 30.0, 0.0001


def brick(rows, cols, sector_rows=1):
    """Bricks of rows x cols cells (rows * cols = 16: one 128-byte line), row-major over the brick grid.  sector_rows = 1:
    row-major inside a brick; 2: 2 x 2-cell sectors (cols must be 2 * k), sectors row-major inside the brick."""
    def index(r, c, width):
        bw = -(-(width + 1) // cols)
        base = ((r // rows) * bw + c // cols) * 16
        rr, cc = r % rows, c % cols
        if sector_rows == 1:
            return base + rr * cols + cc
        return base + ((rr // 2) * (cols // 2) + cc // 2) * 4 + (rr % 2) * 2 + cc % 2
    return index


LAYOUTS = {
    'rowmajor': lambda r, c, width: r * (width + 1) + c,
    'brick4x4': brick(4, 4),
    'brick8x2': brick(8, 2),           # 8 rows x 2 columns: each 32-byte sector holds 2 x 2 cells
    'brick2x8': brick(2, 8),           # 2 rows x 8 columns: each sector holds 4 cells of one row
    'brick2x8s': brick(2, 8, 2),       # 2 rows x 8 columns, each sector 2 x 2 cells
}


def population(wp, n, rng):
    k = rng.integers(0, wp.shape[0], n)
    return (wp[k, 0] + rng.normal(0, 0.3, n), wp[k, 1] + rng.normal(0, 0.3, n),
            wp[k, 2] + rng.normal(0, 0.35, n))


class Marcher(object):
    def __init__(self, h):
        self.dt, self.res, self.ox, self.oy = h.dt, h.resolution, h.orig_x, h.orig_y
        self.H, self.W = h.dt.shape
        self.ang = -FOV / 2 + np.arange(B) * FOV / (B - 1)

    def cells(self, X, Y):
        """(row, column) of the padded table: an off-map point reads the padding row / column (dt[-1,-1])."""
        c = np.floor((X - self.ox) / self.res).astype(np.int64)
        r = np.floor((Y - self.oy) / self.res).astype(np.int64)
        off = (c < 0) | (r < 0) | (c >= self.W) | (r >= self.H)
        return np.where(off, self.H, r), np.where(off, self.W, c)

    def value(self, r, c):
        return np.where((r == self.H) | (c == self.W), self.dt[-1, -1],
                        self.dt[np.minimum(r, self.H - 1), np.minimum(c, self.W - 1)])

    def march(self, x, y, th, on_gather=None):
        """Lookups per beam [agents][B]; on_gather(r, c, live) is called for every gather after the first lookup."""
        X = np.repeat(x[:, None], B, 1)
        Y = np.repeat(y[:, None], B, 1)
        a = th[:, None] + self.ang[None, :]
        co, si = np.cos(a), np.sin(a)
        D = self.value(*self.cells(X, Y))
        T = D.copy()
        n = np.ones(D.shape, np.int64)
        live = (D > EPS) & (T <= MAX_RANGE)
        while live.any():
            X = np.where(live, X + D * co, X)
            Y = np.where(live, Y + D * si, Y)
            r, c = self.cells(X, Y)
            if on_gather is not None:
                on_gather(r, c, live)
            Dn = self.value(r, c)
            D = np.where(live, Dn, D)
            T = np.where(live, T + Dn, T)
            n += live
            live = live & (D > EPS) & (T <= MAX_RANGE)
        return n


def warp_iterations(n, perm=None):
    tot = 0
    for a in range(n.shape[0]):
        row = n[a] if perm is None else n[a][perm[a]]
        tot += int(row[:(B // 32) * 32].reshape(-1, 32).max(1).sum())
        if B % 32:
            tot += int(row[(B // 32) * 32:].max())
    return tot


def lane_study(m, wp, agents, rng):
    x, y, th = population(wp, agents, rng)
    v = rng.uniform(0, 8, agents)
    n0 = m.march(x, y, th)
    n1 = m.march(x + 0.01 * v * np.cos(th), y + 0.01 * v * np.sin(th), th + rng.normal(0, 0.01, agents))
    look = n1.sum()
    out = {'lookups_per_agent': n1.sum(1).mean(), 'busy_share_in_order': look / (32 * warp_iterations(n1)),
           'busy_share_oracle_sort': look / (32 * warp_iterations(n1, np.argsort(n1, axis=1, kind='stable')))}
    for thr in (8, 12, 16, 24, 32):
        perm = np.argsort((n0 < thr).astype(int), axis=1, kind='stable')
        out['busy_share_prev_2class_%d' % thr] = look / (32 * warp_iterations(n1, perm))
    perm = np.argsort(np.digitize(n0, [6, 10, 16, 28]), axis=1, kind='stable')
    out['busy_share_prev_5class'] = look / (32 * warp_iterations(n1, perm))
    out['busy_share_prev_sorted'] = look / (32 * warp_iterations(n1, np.argsort(n0, axis=1, kind='stable')))
    return out


def line_study(m, wp, agents, rng, layouts):
    x, y, th = population(wp, agents, rng)
    stats = {k: [0, 0] for k in layouts}
    gathers = [0]
    nw = (B + 31) // 32

    def on_gather(r, c, live):
        for name in layouts:
            addr = LAYOUTS[name](r, c, m.W) * 8
            for a in range(r.shape[0]):
                for j in range(nw):
                    sl = slice(32 * j, 32 * j + 32)
                    lv = live[a, sl]
                    if not lv.any():
                        continue
                    ad = addr[a, sl][lv]
                    stats[name][0] += np.unique(ad >> 5).size
                    stats[name][1] += np.unique(ad >> 7).size
                    if name == layouts[0]:
                        gathers[0] += 1
    m.march(x, y, th, on_gather)
    return {k: (s / gathers[0], l / gathers[0]) for k, (s, l) in stats.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--map', default='example_map')
    ap.add_argument('--agents', type=int, default=96, help='agents of the sector / line count')
    ap.add_argument('--lane-agents', type=int, default=384, help='agents of the lane figures (0: skip)')
    ap.add_argument('--layouts', default=','.join(LAYOUTS))
    ap.add_argument('--seed', type=int, default=1)
    args = ap.parse_args()
    path = maps.resolve_map_path(args.map)
    h = maps.load_map(path, '.pgm' if args.map == 'levine' else '.png')
    m = Marcher(h)
    wp = maps.load_waypoints()
    if args.lane_agents > 0:
        for k, v in lane_study(m, wp, args.lane_agents, np.random.default_rng(args.seed)).items():
            print('%-28s %.3f' % (k, v))
    layouts = args.layouts.split(',')
    for name, (sec, ln) in line_study(m, wp, args.agents, np.random.default_rng(args.seed), layouts).items():
        print('%-10s sectors/gather %.2f  lines/gather %.2f' % (name, sec, ln))


if __name__ == '__main__':
    main()
