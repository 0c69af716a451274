"""Host-side checks of f110_predict (C ABI include/f110_predict.h, csrc/predict.cuh; no GPU).

  * The ctypes mirror of f110_predict_args against the header, the export, and the ABI version (still 6).
  * Every refusal returns its code before anything is enqueued: NULL pointers, M / K / H bounds, M * K >= 2^31, the sim, map and
    beam rules, and a map / beam setup on which the held-action short path cannot run; F110_ERR_NO_MAP without a table.
  * k_predict's registers and stack, one instance per map kind, with no local memory (no spills).
  * The per-step clearance rule: fp32 of the first lookup at the scan pose, as k_predict computes it on cell-unit tables
    (cell_index on x / res, times res) and on metre tables (xy_2_rc with the IEEE quotient, rotated or not), equals fp32 of the
    oracle's dt_lookup at that pose on every bundled map and a rotated one, over poses on the map, near cell edges and off it.
"""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, '..', 'include', 'f110_predict.h')
BUNDLED = ('berlin', 'skirk', 'levine', 'vegas', 'stata_basement', 'example_map')


def test_predict_args_match_c_layout(tmp_path):
    from f1tenth_gym_b200 import _native as nat
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){',
             'printf("size %zu\\n", sizeof(f110_predict_args));']
    for f, _ in nat.F110PredictArgs._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(f110_predict_args, %s));' % (f, f))
    lines.append('printf("maxh %d\\n", F110_PREDICT_MAX_H);')
    lines.append('printf("abi %d\\n", F110_ABI_VERSION); return 0;}')
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out['size']) == ctypes.sizeof(nat.F110PredictArgs)
    for f, _ in nat.F110PredictArgs._fields_:
        assert int(out[f]) == getattr(nat.F110PredictArgs, f).offset, f
    assert int(out['maxh']) == nat.PREDICT_MAX_H == 4096
    assert int(out['abi']) == nat.ABI_VERSION == 6


def test_predict_entry_point_exported():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    declared = set(re.findall(r'^\S[^(;]*?\b(f110_\w+)\s*\(', open(HEADER).read(), re.M))
    assert declared == set(nat.PREDICT_SIGNATURES) == {'f110_predict'}
    assert hasattr(L, 'f110_predict')


def _lean_setup(buf):
    """A sim, map and beams that pass every host rule up to the short-path test, on host addresses: nothing may ever be
    launched with them, so every call below must be refused."""
    from f1tenth_gym_b200 import _native as nat
    p = ctypes.addressof(buf)
    sim = nat.F110Sim()
    sim.num_envs, sim.num_agents, sim.integrator, sim.timestep = 4, 2, 1, 0.01
    for f in ('params', 'state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'scans', 'wall_flag', 'collisions',
              'collision_idx', 'march_cost', 'march_order', 'march_count', 'march_rec'):
        setattr(sim, f, p)
    sim.march_ipa = (1080 + 31) // 32
    mp = nat.F110Map()
    mp.height, mp.width, mp.resolution, mp.orig_c = 100, 120, 0.05, 1.0
    mp.eps, mp.max_range, mp.theta_dis, mp.dt_min_positive = 1e-4, 30.0, 2000, 0.05
    for f in ('dt', 'sines', 'cosines', 'sincos', 'sincos2'):
        setattr(mp, f, p)
    bm = nat.F110Beams()
    bm.num_beams, bm.fov, bm.theta_index_increment = 1080, 4.7, 1.0
    bm.scan_angles = bm.cosines = bm.side_distances = bm.cos_side = p
    bm.side_max = 0.3
    return sim, mp, bm


def test_predict_rejects_before_any_launch():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    buf = (ctypes.c_double * 64)()
    p = ctypes.addressof(buf)
    sim, mp, bm = _lean_setup(buf)

    def args(**over):
        a = nat.F110PredictArgs(p, p, 2, 3, 5, p, p, None, None)
        for k, v in over.items():
            setattr(a, k, v)
        return a

    def call(a, s=sim, m=mp, b=bm):
        return L.f110_predict(ctypes.byref(s) if s is not None else None, ctypes.byref(m) if m is not None else None, None,
                              ctypes.byref(b) if b is not None else None, ctypes.byref(a) if a is not None else None, None)

    # NULL pointers and bounds
    assert call(None) == -1
    assert call(args(), s=None) == -1
    for f in ('agent_ids', 'actions', 'final_state', 'wall_step'):
        assert call(args(**{f: None})) == -1, f
    for over in ({'M': 0}, {'M': -1}, {'K': 0}, {'H': 0}, {'H': 4097}, {'M': 65536, 'K': 32768}, {'M': 2, 'K': 0x7fffffff}):
        assert call(args(**over)) == -1, over
    # the sim, map and beam rules of f110_step
    bad = nat.F110Sim(); ctypes.pointer(bad)[0] = sim; bad.integrator = 3
    assert call(args(), s=bad) == -4
    bad = nat.F110Sim(); ctypes.pointer(bad)[0] = sim; bad.state = None
    assert call(args(), s=bad) == -1
    assert call(args(), m=None) == -1
    nomap = nat.F110Map(); ctypes.pointer(nomap)[0] = mp; nomap.dt = None
    assert call(args(), m=nomap) == -2                         # no table: F110_ERR_NO_MAP, after the argument checks
    assert call(args(H=0), m=nomap) == -1
    nb = nat.F110Beams(); ctypes.pointer(nb)[0] = bm; nb.num_beams = 1
    assert call(args(), b=nb) == -1
    # setups the short path cannot take
    for name, edit in (('side_max unknown', lambda s, m, b: setattr(b, 'side_max', 0.0)),
                       ('side_max >= max_range', lambda s, m, b: setattr(b, 'side_max', 30.0)),
                       ('dt_min_positive <= eps', lambda s, m, b: setattr(m, 'dt_min_positive', 0.0)),
                       ('no doubled LUT', lambda s, m, b: setattr(m, 'sincos2', None)),
                       ('no march record', lambda s, m, b: setattr(s, 'march_rec', None)),
                       ('no march queue', lambda s, m, b: setattr(s, 'march_ipa', 0)),
                       ('fov >= 2 pi', lambda s, m, b: setattr(b, 'fov', 6.3))):
        s2, m2, b2 = nat.F110Sim(), nat.F110Map(), nat.F110Beams()
        ctypes.pointer(s2)[0], ctypes.pointer(m2)[0], ctypes.pointer(b2)[0] = sim, mp, bm
        edit(s2, m2, b2)
        assert call(args(), s=s2, m=m2, b=b2) == -1, name


def test_predict_kernel_resource_budget():
    """k_predict: one instance per map kind (cells, metres, rot), the state in registers for all H steps: at most 160 registers
    (three 128-thread blocks per SM), a small call stack (the out-of-line march_generic / replay / trig slow paths) and no
    local memory, i.e. no spills."""
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack), rest) for fn, reg, stack, rest in
             re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)([^\n]*)', out)}
    pred = [k for k in usage if 'k_predict' in k]
    assert len(pred) == 3, pred
    for k in pred:
        reg, stack, rest = usage[k]
        assert reg <= 160 and stack <= 64, (k, usage[k])
        assert re.search(r'LOCAL:0\b', rest), (k, rest)


# ------------------------------------------------------------------ the clearance rule
def oracle_dt_lookup(m, x, y):
    """oracle/f110_oracle.c dt_lookup, literally: xy_2_rc (laser_models.py:55-86) with dt[-1,-1] off the map."""
    tx, ty = x - m.orig_x, y - m.orig_y
    xr = tx * m.orig_c + ty * m.orig_s
    yr = -tx * m.orig_s + ty * m.orig_c
    H, W = m.dt.shape
    r, c = H - 1, W - 1
    if not (xr < 0 or xr >= W * m.resolution or yr < 0 or yr >= H * m.resolution):
        cc, rr = int(xr / m.resolution), int(yr / m.resolution)
        if cc < W and rr < H:
            c, r = cc, rr
    return m.dt[r, c]


def kernel_clearance(m, x, y):
    """What k_predict writes: fp32(d0 * d0_scale), d0 the first lookup k_dynamics takes -- on a power-of-two resolution with an
    unrotated origin the cell-unit table (dt / res, exact) at cell_index(x / res, y / res) (floor through the magic add, two
    unsigned bounds tests), times res; else the metre table through xy_2_rc (rotated when the origin is)."""
    H, W = m.dt.shape
    if m.fast_path:
        inv = 1.0 / m.resolution
        c = np.floor(x * inv - m.orig_x * inv)
        r = np.floor(y * inv - m.orig_y * inv)
        cells = m.dt * inv
        d0 = cells[int(r), int(c)] if (0 <= c < W and 0 <= r < H) else cells[-1, -1]
        return np.float32(d0 * m.resolution)
    tx, ty = x - m.orig_x, y - m.orig_y
    if not (m.orig_c == 1.0 and m.orig_s == 0.0):
        xr = tx * m.orig_c + ty * m.orig_s
        ty = -tx * m.orig_s + ty * m.orig_c
        tx = xr
    d0 = m.dt[-1, -1]
    if not (tx < 0 or tx >= W * m.resolution or ty < 0 or ty >= H * m.resolution):
        c, r = int(tx / m.resolution), int(ty / m.resolution)
        if c < W and r < H:
            d0 = m.dt[r, c]
    return np.float32(d0)


def _poses(m, rng, n):
    """Poses on the map, on and one ulp either side of cell edges, and off every side of it."""
    H, W = m.dt.shape
    res = m.resolution
    u = rng.uniform(-0.1, 1.1, (n, 2)) * np.array([W * res, H * res])
    edge = np.stack([rng.integers(0, W + 1, n) * res, rng.integers(0, H + 1, n) * res], 1)
    edge = np.concatenate([edge, np.nextafter(edge, np.inf), np.nextafter(edge, -np.inf)])
    local = np.concatenate([u, edge])
    x = m.orig_x + local[:, 0] * m.orig_c - local[:, 1] * m.orig_s
    y = m.orig_y + local[:, 0] * m.orig_s + local[:, 1] * m.orig_c
    return x, y


@pytest.mark.parametrize('name', list(BUNDLED) + ['berlin_rotated'])
def test_clearance_rule_against_the_oracle_lookup(name):
    from f1tenth_gym_b200 import maps
    base = name.replace('_rotated', '')
    path = maps.resolve_map_path(base)
    ext = '.pgm' if os.path.exists(os.path.splitext(path)[0] + '.pgm') else '.png'
    h = maps.load_map(path, ext)
    if name.endswith('_rotated'):
        h = maps.HostMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.35))
    rng = np.random.default_rng(len(name))
    x, y = _poses(h, rng, 3000)
    got = np.array([kernel_clearance(h, a, b) for a, b in zip(x, y)])
    want = np.array([np.float32(oracle_dt_lookup(h, a, b)) for a, b in zip(x, y)])
    assert np.array_equal(got, want), (name, int(np.sum(got != want)))
    assert np.unique(want).size > 10                  # not vacuous: the poses see many distances, walls and off-map included
