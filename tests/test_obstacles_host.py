"""Host-side checks of the static box obstacles (no GPU).

  * The ctypes mirror of f110_obstacles against the header's layout, the exported entry points and the ABI version.
  * The numpy restatement of the respawn draw: deterministic, its count and clearance rules on hand-built cases.
  * obstacle_candidates: every box inside the lateral band of its centerline segment, deterministic in the seed.
  * Argument rejection: the entry points that reach the obstacle checks without a map, and Simulator / F110Env validation
    where it runs before any device work.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'f110_b200.h')


def test_obstacles_struct_matches_c_layout(tmp_path):
    from f1tenth_gym_b200 import _native as nat
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){',
             'printf("size %zu\\n", sizeof(f110_obstacles));']
    for f, _ in nat.F110Obstacles._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(f110_obstacles, %s));' % (f, f))
    lines.append('printf("max %d\\n", F110_MAX_OBSTACLES); printf("abi %d\\n", F110_ABI_VERSION); return 0;}')
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out['size']) == ctypes.sizeof(nat.F110Obstacles)
    for f, _ in nat.F110Obstacles._fields_:
        assert int(out[f]) == getattr(nat.F110Obstacles, f).offset, f
    assert int(out['max']) == nat.MAX_OBSTACLES == 16
    assert int(out['abi']) == nat.ABI_VERSION == 6


def test_obstacle_symbols_exported():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    for name in ('f110_step_obst', 'f110_tick_obst', 'f110_tick_repeat_ticks_obst', 'f110_autoreset_obst',
                 'f110_obstacles_respawn'):
        assert name in nat.SIGNATURES and hasattr(L, name), name
    assert L.f110_abi_version() == 6


# ----------------------------------------------------------------------------- the respawn draw
def test_respawn_draw_deterministic_and_keyed():
    from f1tenth_gym_b200.obstacles import respawn_draw
    rng = np.random.default_rng(0)
    cand = np.column_stack([rng.uniform(-50, 50, (40, 2)), rng.uniform(-3, 3, 40), np.full(40, 0.58), np.full(40, 0.31)])
    xy = np.array([[1000.0, 1000.0]])
    a = respawn_draw(cand, xy, 8, (2, 6), 1.0, 7, 11, 3)
    b = respawn_draw(cand, xy, 8, (2, 6), 1.0, 7, 11, 3)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    # every slot holds a candidate row; another tick, env or seed draws another layout
    assert all(any(np.array_equal(r, c) for c in cand) for r in a[0])
    others = [respawn_draw(cand, xy, 8, (2, 6), 1.0, s, t, e)[0] for s, t, e in ((8, 11, 3), (7, 12, 3), (7, 11, 4))]
    assert all(not np.array_equal(a[0], o) for o in others)


def test_respawn_draw_count_rule():
    from f1tenth_gym_b200.obstacles import respawn_draw
    cand = np.array([[0.0, 0.0, 0.0, 0.58, 0.31]])
    far = np.array([[500.0, 500.0]])
    seen = set()
    for t in range(300):
        _, act = respawn_draw(cand, far, 6, (1, 4), 1.0, 3, t, 0)
        c = int(act.sum())
        assert 1 <= c <= 4 and act[:c].all() and not act[c:].any()     # slots k < c are active, the rest not
        seen.add(c)
    assert seen == {1, 2, 3, 4}
    for t in range(20):
        assert respawn_draw(cand, far, 3, (3, 3), 1.0, 3, t, 1)[1].tolist() == [1, 1, 1]
        assert not respawn_draw(cand, far, 3, (0, 0), 1.0, 3, t, 1)[1].any()


def test_respawn_draw_clearance_rule():
    from f1tenth_gym_b200.obstacles import respawn_draw
    cand = np.array([[2.0, 0.0, 0.0, 0.58, 0.31]])
    for r, want in ((1.9, 1), (2.0, 1), (2.1, 0)):
        # an agent exactly `clearance` away keeps the box; closer, the slot stays inactive (no retry)
        _, act = respawn_draw(cand, np.array([[0.0, 0.0]]), 2, (2, 2), r, 1, 5, 0)
        assert act.tolist() == [want, want], r
    # any agent of the env counts
    _, act = respawn_draw(cand, np.array([[100.0, 0.0], [2.5, 0.0]]), 1, (1, 1), 1.0, 1, 5, 0)
    assert act.tolist() == [0]


# ----------------------------------------------------------------------------- candidates along a centerline
def test_obstacle_candidates_lateral_band():
    from f1tenth_gym_b200 import maps, obstacle_candidates
    wp = maps.load_waypoints()[:, :2]
    lo, hi = -0.8, 0.5
    boxes = obstacle_candidates(wp, 500, lateral=(lo, hi), size=(0.6, 0.3), yaw_jitter=0.2, seed=4)
    assert boxes.shape == (500, 5) and np.isfinite(boxes).all()
    assert np.array_equal(boxes, obstacle_candidates(wp, 500, lateral=(lo, hi), size=(0.6, 0.3), yaw_jitter=0.2, seed=4))
    assert not np.array_equal(boxes, obstacle_candidates(wp, 500, lateral=(lo, hi), size=(0.6, 0.3), yaw_jitter=0.2, seed=5))
    assert (boxes[:, 3] == 0.6).all() and (boxes[:, 4] == 0.3).all()
    p = wp if not np.array_equal(wp[0], wp[-1]) else wp[:-1]
    d = np.roll(p, -1, axis=0) - p
    for x, y, yaw, _, _ in boxes:
        # some segment has the box's foot point inside it and the signed offset (left of travel) inside the band
        rel = np.array([x, y]) - p
        l2 = (d ** 2).sum(1)
        t = (rel * d).sum(1) / l2
        off = (d[:, 0] * rel[:, 1] - d[:, 1] * rel[:, 0]) / np.sqrt(l2)
        ok = (t >= -1e-9) & (t <= 1 + 1e-9) & (off >= lo - 1e-9) & (off <= hi + 1e-9)
        assert ok.any(), (x, y)
        h = np.arctan2(d[ok, 1], d[ok, 0])
        assert (np.abs((yaw - h + np.pi) % (2 * np.pi) - np.pi) <= 0.2 + 1e-9).any()


def test_obstacle_candidates_rejects():
    from f1tenth_gym_b200 import obstacle_candidates
    sq = np.array([[0.0, 0.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1.0]])
    for kw in (dict(count=0), dict(lateral=(1.0, -1.0)), dict(size=(0.0, 0.3)), dict(size=(0.5, np.nan)),
               dict(yaw_jitter=-1.0)):
        args = dict(count=3)
        args.update(kw)
        with pytest.raises(ValueError):
            obstacle_candidates(sq, **args)
    for bad in (sq[:2], np.array([[0.0, 0.0], [0.0, 0.0], [1.0, 1.0]]), np.zeros(4)):
        with pytest.raises(ValueError):
            obstacle_candidates(bad, 3)


# ----------------------------------------------------------------------------- the C checks before any launch
def _valid_sim(nat):
    sim = nat.F110Sim()
    buf = (ctypes.c_double * 64)()
    p = ctypes.addressof(buf)
    sim.num_envs, sim.num_agents, sim.integrator = 2, 1, 1
    for f in ('params', 'state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'scans', 'wall_flag', 'collisions',
              'collision_idx'):
        setattr(sim, f, p)
    return sim, buf, p


def obstacle_struct_cases(nat, p, offs):
    """(name, f110_obstacles) for every struct the header says is rejected."""
    def mk(**kw):
        o = nat.F110Obstacles(4, p, p, None, p, None, 8, 0, 1, 2, 0.5, 1)
        for k, v in kw.items():
            setattr(o, k, v)
        return o
    return [('K=0', mk(per_env=0)), ('K=17', mk(per_env=17)), ('no boxes', mk(boxes=None)), ('no active', mk(active=None)),
            ('count_min > count_max', mk(count_min=3, count_max=2)), ('count_max > K', mk(count_max=5)),
            ('count_min < 0', mk(count_min=-1)), ('negative clearance', mk(clearance=-0.1)),
            ('NaN clearance', mk(clearance=float('nan'))), ('inf clearance', mk(clearance=float('inf'))),
            ('no candidate rows', mk(num_candidates=0)),
            ('offsets not ending at C', mk(cand_offsets=offs, num_cand_tables=1)),
            ('zero tables', mk(cand_offsets=offs, num_cand_tables=0))]


def test_obstacle_entry_points_reject_bad_structs():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    sim, buf, p = _valid_sim(nat)
    offs_buf = (ctypes.c_int32 * 3)(0, 3, 9)
    offs = ctypes.addressof(offs_buf)
    sim.env_layer = p
    for name, o in obstacle_struct_cases(nat, p, offs):
        assert L.f110_obstacles_respawn(ctypes.byref(sim), ctypes.byref(o), None, 0, None) == -1, name
        assert L.f110_autoreset_obst(ctypes.byref(sim), p, 4, 1, 0, 0, ctypes.byref(o), None) == -1, name
    o = nat.F110Obstacles(4, p, p, None, None, None, 0, 0, 0, 0, 0.0, 0)
    assert L.f110_obstacles_respawn(ctypes.byref(sim), ctypes.byref(o), None, 0, None) == -1       # no candidates
    assert L.f110_obstacles_respawn(ctypes.byref(sim), None, None, 0, None) == -1
    # per-layer tables need env_layer
    sim.env_layer = None
    o = nat.F110Obstacles(4, p, p, None, p, offs, 9, 2, 0, 1, 0.0, 0)
    assert L.f110_obstacles_respawn(ctypes.byref(sim), ctypes.byref(o), None, 0, None) == -1
    # more than 32 agents per env
    sim.num_agents = 33
    o = nat.F110Obstacles(4, p, p, None, p, None, 9, 0, 0, 1, 0.0, 0)
    assert L.f110_obstacles_respawn(ctypes.byref(sim), ctypes.byref(o), None, 0, None) == -1
    # the tick checks the map first, like the call without obstacles: an empty map is F110_ERR_NO_MAP either way
    assert L.f110_tick_obst(None, None, None, None, None, 0, None, 0, 0, 0, ctypes.byref(o), None) == -1


def test_env_obstacle_settings_rejected_before_device_work():
    from f1tenth_gym_b200 import F110Env
    cand = np.zeros((3, 5))
    with pytest.raises(ValueError):
        F110Env(map='example_map', obstacles={'candidates': cand})                 # single-env mode
    for bad in ({'count': (1, 2)}, {'candidates': cand, 'size': 1}, {'candidates': cand, 'count': (2, 1)},
                {'candidates': cand, 'count': (0, 17)}, {'candidates': cand, 'count': (0, 0)},
                {'candidates': cand, 'count': 'x'}, {'candidates': cand, 'clearance': -1.0},
                {'candidates': cand, 'clearance': np.nan}, [cand]):
        with pytest.raises(ValueError):
            F110Env(map='example_map', num_envs=2, obstacles=bad)


def test_render_palette_has_an_obstacle_colour():
    from f1tenth_gym_b200.env import RENDER_PALETTE
    assert tuple(RENDER_PALETTE[5]) not in {tuple(RENDER_PALETTE[c]) for c in (0, 1, 2, 3, 4)}

