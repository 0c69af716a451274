"""Host-side checks of f110_tick_repeat (no GPU).

  * The bound the short path rests on, against the oracle: wherever the first distance-table lookup at the scan pose exceeds the
    iTTC pre-test threshold of the agent's speed (and max_range does), the oracle's check_ttc on the oracle's scan does not
    fire; and it does fire for some of the other poses.  Poses come from random-action rollouts of the oracle on example_map
    and berlin, 1 and 2 agents, lidar_dist 0 and 0.275; the share of poses that would be marched is printed per workload.
  * The select rule of k_ttc_select as a numpy model, one ulp either side of the threshold, at v = 0, v < 0, off the map and NaN.
  * Argument rejection before anything is enqueued, the ctypes mirror of f110_repeat, and the register / stack budget of the
    new kernels.
"""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'f110_b200.h')
TTC_THRESH = 0.005
MAX_RANGE = 30.0


def threshold(v, side_max):
    """k_dynamics' per-agent iTTC pre-test threshold (csrc/f110_b200.cu)."""
    v = np.asarray(v, dtype=np.float64)
    return np.where(v != 0.0, (side_max + TTC_THRESH * 1.000001 * np.abs(v)) * (1.0 + 1e-9), -np.inf)


def listed(d0_m, thr, max_range=MAX_RANGE, absurd=False):
    """k_ttc_select: an agent is skipped only when `d0 > thr and max_range > thr` is true."""
    with np.errstate(invalid='ignore'):
        clear = (np.asarray(d0_m) > thr) & (max_range > np.asarray(thr))
    return np.asarray(absurd) | ~clear


def first_lookup(omap, x, y):
    """dt at the scan pose as xy_2_rc reads it (laser_models.py:55-104) on an unrotated map; dt[-1,-1] off the map."""
    H, W = omap.dt.shape
    tx, ty = x - omap.orig_x, y - omap.orig_y
    if tx < 0 or tx >= W * omap.resolution or ty < 0 or ty >= H * omap.resolution:
        return omap.dt[-1, -1]
    c, r = int(tx / omap.resolution), int(ty / omap.resolution)
    return omap.dt[r, c] if (c < W and r < H) else omap.dt[-1, -1]


@pytest.mark.parametrize('lidar_dist', [0.0, 0.275])
@pytest.mark.parametrize('A', [1, 2])
@pytest.mark.parametrize('name', ['example_map', 'berlin'])
def test_the_bound_against_the_oracle(name, A, lidar_dist):
    import oracle
    from f1tenth_gym_b200 import maps
    om = oracle.OracleMap.from_yaml(maps.resolve_map_path(name), '.png')
    _, cosines, sides = oracle.beam_tables(1080, 4.7, maps.DEFAULT_PARAMS)
    side_max = float(sides.max())
    rng = np.random.default_rng(A * 10 + int(lidar_dist * 100))
    free = np.argwhere((om.dt > 0.3) & (om.dt < 0.8))
    n, ticks = 6, 60
    sims = [oracle.OracleSim(om, num_agents=A, lidar_dist=lidar_dist) for _ in range(n)]

    def start():
        r, c = free[rng.integers(free.shape[0])]
        p0 = np.array([c * om.resolution + om.orig_x, r * om.resolution + om.orig_y, rng.uniform(0, 2 * np.pi)])
        return np.stack([p0 + np.array([0.45, 0.1, 0.3]) * i for i in range(A)])
    for s in sims:
        s.env_restart(start())
    total = marched = fired = fired_listed = 0
    for t in range(ticks):
        for s in sims:
            s.step(np.stack([rng.uniform(-0.4189, 0.4189, A), rng.uniform(0, 8, A)], axis=1))
            for i in range(A):
                x, y, v, yaw = s.state[i, 0], s.state[i, 1], s.state[i, 3], s.state[i, 4]
                # (after a hit the oracle has zeroed v and the yaw: the pose still counts, with the probe speeds)
                sx, sy = x + lidar_dist * np.cos(yaw), y + lidar_dist * np.sin(yaw)
                d0 = first_lookup(om, sx, sy)
                scan = oracle.get_scan(om, np.array([sx, sy, yaw]))
                for vv in (v, 8.0, -3.0):      # the rollout's speed and two probe speeds on the same pose
                    hit = bool(oracle.check_ttc(scan, vv, cosines, sides, TTC_THRESH))
                    m = bool(listed(d0, threshold(vv, side_max)))
                    total += 1
                    marched += m
                    fired += hit
                    fired_listed += hit and m
                    assert m or not hit, (name, t, sx, sy, vv, d0)
            if s.collisions[0]:
                s.env_restart(start())
    print('%s A=%d lidar_dist=%g: listed %.3f of %d pose-speeds, %d fired' % (name, A, lidar_dist, marched / total, total, fired))
    assert fired > 0 and fired == fired_listed          # not vacuous: the check fires, and only among the listed
    assert marched < total                              # and the rule does skip poses


def test_select_rule_guard_band():
    side_max = 0.2937
    v = 3.0
    thr = float(threshold(v, side_max))
    up, down = np.nextafter(thr, np.inf), np.nextafter(thr, -np.inf)
    assert not listed(up, thr) and listed(thr, thr) and listed(down, thr)       # skipped only strictly above
    assert not listed(0.0, threshold(0.0, side_max))                             # v == 0: thr = -inf, never marched
    assert float(threshold(-3.0, side_max)) == thr                                # v < 0: |v|
    assert listed(0.0, thr) and not listed(5.0, thr)                              # off the map: d0 = dt[-1,-1], whatever it holds
    assert listed(np.nan, thr) and listed(5.0, np.nan)                            # a NaN on either side lists the agent
    assert listed(5.0, thr, absurd=True)                                          # absurd coordinates are always marched
    assert listed(50.0, 31.0)                                                     # thr at or beyond max_range: marched
    # cell-unit tables: d0 in cells times a power-of-two resolution is exact, so the rule sees the metre value
    assert (np.float64(7.0) * 0.0625) / 0.0625 == 7.0


def test_tick_repeat_rejects_bad_arguments_before_any_launch():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    sim, mp, bm, rep = nat.F110Sim(), nat.F110Map(), nat.F110Beams(), nat.F110Repeat()
    args = (ctypes.byref(sim), ctypes.byref(mp), None, ctypes.byref(bm), None)
    assert L.f110_tick_repeat(None, None, None, None, None, 2, None, 1, None, 0, 0, 0, None) == -1
    assert L.f110_tick_repeat(*args, 2, ctypes.byref(rep), 0, None, 0, 0, 0, None) == -1       # an empty sim
    # a sim that passes check_sim, so that the repeat arguments themselves are reached
    buf = (ctypes.c_double * 64)()
    p = ctypes.addressof(buf)
    sim.num_envs = sim.num_agents = 1
    sim.integrator = 1
    for f in ('params', 'state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'scans', 'wall_flag', 'collisions',
              'collision_idx'):
        setattr(sim, f, p)
    rep.list, rep.list_count = p, p
    for repeat in (0, -1, 65):
        assert L.f110_tick_repeat(*args, repeat, ctypes.byref(rep), 0, None, 0, 0, 0, None) == -1
    assert L.f110_tick_repeat(*args, 2, None, 0, None, 0, 0, 0, None) == -1                       # no f110_repeat
    assert L.f110_tick_repeat(*args, 2, ctypes.byref(nat.F110Repeat()), 0, None, 0, 0, 0, None) == -1   # no scratch
    rep.done_any = p
    assert L.f110_tick_repeat(*args, 2, ctypes.byref(rep), 0, None, 0, 0, 0, None) == -1        # done_any without env_level
    rep.done_any = None
    for first, count in ((-1, 1), (0, 0), (2, 1), (1, 2)):
        assert L.f110_tick_repeat_ticks(*args, 2, first, count, ctypes.byref(rep), 0, None, 0, 0, 0, None) == -1
    assert L.f110_tick_repeat(*args, 2, ctypes.byref(rep), 0, None, 0, 0, 0, None) == -2        # valid so far: no map is set
    assert L.f110_track_progress_sum(None, None, None, None, 1, None) == -1


def test_repeat_struct_matches_c_layout(tmp_path):
    from f1tenth_gym_b200 import _native as nat
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){',
             'printf("size %zu\\n", sizeof(f110_repeat));']
    for f, _ in nat.F110Repeat._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(f110_repeat, %s));' % (f, f))
    lines.append('printf("max %d\\n", F110_MAX_REPEAT); return 0;}')
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out['size']) == ctypes.sizeof(nat.F110Repeat)
    for f, _ in nat.F110Repeat._fields_:
        assert int(out[f]) == getattr(nat.F110Repeat, f).offset, f
    assert int(out['max']) == nat.MAX_REPEAT


def test_repeat_kernel_resource_budget():
    """k_march_ttc keeps 64 registers (four 256-thread blocks per SM) and next to no stack; the scan-free tail stays within the
    stack the auto-reset's pose staging needs (DESIGN.md 3.8)."""
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    march = [k for k in usage if 'k_march_ttc' in k]
    assert len(march) == 6, march                       # cells / metres / rot x plain / counting
    for k in march:
        assert usage[k][0] <= 64 and usage[k][1] <= 16, (k, usage[k])
    tail = [k for k in usage if 'k_tail_noscan' in k]
    assert len(tail) == 1 and usage[tail[0]][0] <= 96 and usage[tail[0]][1] <= 1024, (tail, usage.get(tail[0] if tail else ''))
    sel = [k for k in usage if 'k_ttc_select' in k]
    assert len(sel) == 1 and usage[sel[0]][0] <= 32 and usage[sel[0]][1] == 0
