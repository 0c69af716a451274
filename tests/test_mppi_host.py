"""Host-side checks of the scored rollout and the MPPI planner (C ABI include/f110_mppi.h, csrc/predict.cuh, csrc/mppi.cuh; no GPU).

  * The ctypes mirrors of f110_cost and f110_mppi against the header, the exports, and the ABI version (still 6).
  * Every refusal of f110_predict_scored, f110_mppi_sample and f110_mppi_update returns its code before anything is enqueued.
    The scored rollout checks its cost and track before the map, so each refusal has a positive control: the same call with a
    valid cost and no distance table reaches the map check (F110_ERR_NO_MAP).
  * Registers, stack and spills of k_scored_rollout (one instance per map kind), k_scored_acquire and the two MPPI kernels.
  * The numpy cost model (the tracker of test_progress_host.TrackerModel, then the cost sum in the kernel's order) on hand-worked
    cases: a straight run, a hairpin where the window keeps the tracker on its branch, a re-acquire, a lap wrap, NaN propagation.
  * The numpy update model: NaN and infinite costs get weight 0, no finite cost keeps and shifts the nominal, and a temperature
    small enough leaves only the argmin a weight.
  * Every ValueError of Simulator.predict(cost=) and MPPIPlanner, raised before any device work.
tests/test_gpu_mppi.py compares the kernels with these models.
"""
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from test_predict_host import _lean_setup
from test_progress_host import NONE, TrackerModel, hairpin, project_model, records, window_search

CPU = torch.device('cpu')
HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, '..', 'include', 'f110_mppi.h')
NAN = float('nan')


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


# ----------------------------------------------------------------------------- the models
def cost_model(recs, tables, src_pose, states, clr, actions, prev, wall, w, back, fwd, reacquire_dist, events=None):
    """cost (S,) of S samples: tables (S,) table ids; src_pose (S, 3) the source agent's (x, y, yaw); states (S, H, 7) the state
    after each step; clr (S, H) the fp64 clearance; actions (S, H, 2); prev (S, 2) or None; wall (S,) wall_step; w the weights.
    The tracker is TrackerModel: one acquiring update at the source pose, then one tracking update per step.  events: a dict that
    receives per-sample counts of 'reacquire' (a tracking update that left the window) and 'wrap' (a delta unwrapped by a lap)."""
    S, H = states.shape[:2]
    tm = TrackerModel(recs, S, back, fwd, reacquire_dist)
    st = np.full((7, S), np.nan)
    st[0], st[1], st[4] = src_pose[:, 0], src_pose[:, 1], src_pose[:, 2]
    tables = np.asarray(tables, np.int64)
    tm.update(st, np.zeros(S, np.int64), tables)
    lost = tm.seg < 0
    n = np.array([recs[t].shape[0] if 0 <= t < len(recs) else 1 for t in tables])
    L = np.array([tm.lengths[t] if 0 <= t < len(recs) else np.nan for t in tables])
    ev = {'reacquire': np.zeros(S, np.int64), 'wrap': np.zeros(S, np.int64)}
    c = np.zeros(S)
    with np.errstate(invalid='ignore', over='ignore'):
        for h in range(H):
            seg_before, s_before = tm.seg.copy(), tm.s.copy()
            for tb, rec in enumerate(recs):           # a re-acquire: the window's best distance is above reacquire_dist
                sel = np.nonzero(~lost & (tables == tb) & np.isfinite(states[:, h, [0, 1, 4]]).all(axis=1))[0]
                if sel.size:
                    k, _, dist = window_search(rec, states[sel, h, 0], states[sel, h, 1], (seg_before[sel] - back) % n[sel],
                                               min(back + fwd + 1, rec.shape[0]))
                    ev['reacquire'][sel] += (k == NONE) | ~(dist <= reacquire_dist)
            tm.update(np.ascontiguousarray(states[:, h].T), np.ones(S, np.int64), tables)
            lost |= tm.seg < 0
            ok = ~lost
            ev['wrap'] += ok & (np.abs(tm.s - s_before) > L * 0.5)
            up = (actions[:, h - 1] if h > 0 else (prev if prev is not None else actions[:, 0]))
            gap = w['clear_min'] - clr[:, h]
            pen = np.where(gap > 0.0, gap, 0.0)
            ds, dv = actions[:, h, 0] - up[:, 0], actions[:, h, 1] - up[:, 1]
            c = c + w['w_lat'] * (tm.d * tm.d)
            c = c + w['w_head'] * (tm.e * tm.e)
            c = c + w['w_clear'] * (pen * pen)
            c = c + w['w_dsteer'] * (ds * ds)
            c = c + w['w_dspeed'] * (dv * dv)
        c = c - w['w_prog'] * tm.progress
        c = np.where(wall >= 0, c + w['w_wall'], c)
    c[lost] = np.nan
    if events is not None:
        events.update(ev)
    return c


def update_model(A, c, nominal, lam, bounds):
    """f110_mppi_update on (M, K, H, 2) actions and (M, K) costs -> (U (M, H, 2), new nominal, weights, argmin, no_finite)."""
    fin = np.isfinite(c)
    any_ = fin.any(axis=1)
    beta = np.where(any_, np.min(np.where(fin, c, np.inf), axis=1), 0.0)
    with np.errstate(invalid='ignore', over='ignore'):
        w = np.where(fin, np.exp(-(c - beta[:, None]) / lam), 0.0)
    U = np.einsum('mk,mkhc->mhc', w, A) / np.maximum(w.sum(axis=1), 1e-300)[:, None, None]
    lo, hi = np.array([bounds[0], bounds[2]]), np.array([bounds[1], bounds[3]])
    U = np.where(any_[:, None, None], U, np.clip(nominal, lo, hi))
    nom = np.concatenate([U[:, 1:], U[:, -1:]], axis=1)
    argmin = np.where(any_, np.argmin(np.where(fin, c, np.inf), axis=1), -1)
    return U, nom, w, argmin, ~any_


W1 = {'w_lat': 1.0, 'w_head': 0.5, 'w_clear': 4.0, 'clear_min': 0.5, 'w_dsteer': 2.0, 'w_dspeed': 0.25, 'w_prog': 3.0,
      'w_wall': 100.0}


def straight_case():
    """One sample on the hairpin's lower straight: from (0.5, 0.25) it moves 1 m per step in x at lateral offset 0.25 m and
    yaw 0.5, with clearance 0.25 m: every term is exact in binary."""
    H = 3
    st = np.zeros((1, H, 7))
    for h in range(H):
        st[0, h, 0], st[0, h, 1], st[0, h, 4] = 1.5 + h, 0.25, 0.5
    act = np.array([[[0.1, 2.0], [0.3, 2.5], [0.3, 2.0]]])
    return st, act


def test_cost_model_straight(f110):
    rec = records(f110, hairpin())
    st, act = straight_case()
    clr = np.full((1, 3), 0.25)
    c = cost_model([rec], [0], np.array([[0.5, 0.25, 0.5]]), st, clr, act, None, np.array([-1]), W1, 2, 4, 5.0)
    # per step: lat 0.0625, head 0.125, clear 4 * 0.0625 = 0.25; rates: step 1 2 * 0.04 + 0.25 * 0.25, step 2 0.25 * 0.25
    rates = 2.0 * (0.2 ** 2) + 0.25 * 0.25 + 0.25 * 0.25
    want = 3 * (0.0625 + 0.125 + 0.25) + rates - 3.0 * 3.0
    assert abs(c[0] - want) < 1e-12, (c[0], want)
    # prev_action gives step 0 its rate terms; a wall hit adds w_wall
    c2 = cost_model([rec], [0], np.array([[0.5, 0.25, 0.5]]), st, clr, act, np.array([[0.0, 2.0]]), np.array([1]), W1, 2, 4, 5.0)
    assert abs(c2[0] - (want + 2.0 * 0.01 + 100.0)) < 1e-12


def test_cost_model_hairpin_window_reacquire_and_nan(f110):
    """The hairpin of test_progress_host: drifting to 0.6 m off the lower straight keeps the tracker there (d = +0.6) where
    the global projection would take the upper branch (0.4 m); a teleport beyond reacquire_dist re-acquires; NaN states and an
    unacquired source give NaN costs."""
    rec = records(f110, hairpin())
    w = dict(W1, w_head=0.0, w_clear=0.0, w_dsteer=0.0, w_dspeed=0.0, w_prog=1.0)
    st = np.zeros((4, 2, 7))
    st[:, 0, 0], st[:, 0, 1] = 3.5, 0.6
    st[:, 1, 0], st[:, 1, 1] = 4.5, 0.6
    st[1, 1, 0], st[1, 1, 1] = 8.0, -20.0          # a teleport: the window misses, the global projection finds segment 7
    st[2, 1, 0] = np.nan
    src = np.array([[2.5, 0.0, 0.0]] * 3 + [[np.nan, 0.0, 0.0]])
    act = np.zeros((4, 2, 2))
    ev = {}
    c = cost_model([rec], [0] * 4, src, st, np.ones((4, 2)), act, None, np.full(4, -1), w, 2, 4, 5.0, ev)
    assert project_model([rec], [[3.5, 0.6, 0.0]])[0, 0] == 17             # global: the upper branch
    assert abs(c[0] - (0.36 + 0.36 - 2.0)) < 1e-12                          # progress 1 + 1, d = 0.6 both steps
    glob = project_model([rec], [[8.0, -20.0, 0.0]])[0]
    assert abs(c[1] - (0.36 + glob[2] ** 2 - (1.0 + 4.5))) < 1e-9
    assert ev['reacquire'].tolist() == [0, 1, 0, 0]
    assert np.isnan(c[2]) and np.isnan(c[3])


def test_cost_model_lap_wrap(f110):
    """Crossing the start of the lap: s jumps from near L to near 0, the delta is unwrapped to the short way round."""
    tab = hairpin()
    rec = records(f110, tab)
    L = rec[-1, 5] + rec[-1, 6]
    st = np.zeros((1, 2, 7))
    st[0, 0, 0], st[0, 0, 1] = 0.0, 0.25       # on the closing segment (x = 0, from y = 1 down to y = 0), 0.25 before the end
    st[0, 1, 0], st[0, 1, 1] = 0.5, 0.0        # 0.5 m into the lap
    w = dict(W1, w_lat=0.0, w_head=0.0, w_clear=0.0, w_dsteer=0.0, w_dspeed=0.0, w_prog=1.0)
    ev = {}
    c = cost_model([rec], [0], np.array([[0.0, 0.5, -np.pi / 2]]), st, np.ones((1, 2)), np.zeros((1, 2, 2)), None,
                   np.array([-1]), w, 2, 4, 5.0, ev)
    assert abs(c[0] + 1.0) < 1e-12, c               # 0.25 + 0.25 + 0.5 m of progress
    assert ev['wrap'][0] == 1 and L == 22.0


def test_update_model_cases():
    rng = np.random.default_rng(1)
    M, K, H = 4, 6, 3
    A = rng.uniform(-1, 1, (M, K, H, 2))
    nominal = rng.uniform(-2, 2, (M, H, 2))
    c = rng.uniform(0, 5, (M, K))
    c[0, [1, 3]] = [np.nan, np.inf]
    c[1, :] = np.nan                                   # no finite sample
    c[2, 4] = -np.inf
    bounds = (-0.5, 0.5, -1.0, 1.0)
    U, nom, w, am, nf = update_model(A, c, nominal, 1.0, bounds)
    assert w[0, 1] == 0.0 and w[0, 3] == 0.0 and w[2, 4] == 0.0
    assert (w[1] == 0).all() and am[1] == -1 and nf.tolist() == [False, True, False, False]
    assert np.array_equal(U[1], np.clip(nominal[1], [-0.5, -1.0], [0.5, 1.0]))
    assert np.array_equal(nom[:, :-1], U[:, 1:]) and np.array_equal(nom[:, -1], U[:, -1])
    assert all(w[m, am[m]] == 1.0 for m in (0, 2, 3))
    # a small temperature leaves the argmin alone: U is its sample
    U2, _, w2, am2, _ = update_model(A, c, nominal, 1e-9, bounds)
    for m in (0, 2, 3):
        assert (w2[m] > 0).sum() == 1 and np.array_equal(U2[m], A[m, am2[m]])


# ----------------------------------------------------------------------------- C ABI
def test_structs_match_c_layout(tmp_path):
    from f1tenth_gym_b200 import _native as nat
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){']
    for name, cls in (('f110_cost', nat.F110Cost), ('f110_mppi', nat.F110Mppi)):
        lines.append('printf("%s.size %%zu\\n", sizeof(%s));' % (name, name))
        for f, _ in cls._fields_:
            cf = 'lambda' if f == 'lambda_' else f
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (name, f, name, cf))
    lines.append('printf("maxk %d\\nmaxh %d\\n", F110_MPPI_MAX_K, F110_MPPI_MAX_H);')
    lines.append('printf("abi %d\\n", F110_ABI_VERSION); return 0;}')
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    for name, cls in (('f110_cost', nat.F110Cost), ('f110_mppi', nat.F110Mppi)):
        assert int(out[name + '.size']) == ctypes.sizeof(cls)
        for f, _ in cls._fields_:
            assert int(out['%s.%s' % (name, f)]) == getattr(cls, f).offset, (name, f)
    assert int(out['maxk']) == nat.MPPI_MAX_K and int(out['maxh']) == nat.MPPI_MAX_H
    assert int(out['abi']) == nat.ABI_VERSION == 6


def test_entry_points_exported():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    declared = set(re.findall(r'^\S[^(;]*?\b(f110_\w+)\s*\(', open(HEADER).read(), re.M))
    assert declared == set(nat.MPPI_SIGNATURES) == {'f110_predict_scored', 'f110_mppi_sample', 'f110_mppi_update'}
    for name in declared:
        assert hasattr(L, name)


def _cost(**over):
    from f1tenth_gym_b200 import _native as nat
    c = nat.F110Cost()
    for k, v in W1.items():
        setattr(c, k, v)
    c.back, c.fwd, c.reacquire_dist = 8, 56, 5.0
    buf = (ctypes.c_double * 8)()
    c.cost = c.seg0 = c.s0 = ctypes.addressof(buf)
    c._keep = buf
    for k, v in over.items():
        setattr(c, k, v)
    return c


def test_predict_scored_rejects_before_any_launch():
    """Each bad field gives F110_ERR_INVALID; the same call with the field valid and no distance table gives F110_ERR_NO_MAP,
    so the refusal came from that field.  Nothing here can launch: the map has no table or the call is refused."""
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    buf = (ctypes.c_double * 64)()
    p = ctypes.addressof(buf)
    sim, mp, bm = _lean_setup(buf)
    nomap = nat.F110Map(); ctypes.pointer(nomap)[0] = mp; nomap.dt = None
    track = nat.F110Track(1, 3, p, p)
    args = nat.F110PredictArgs(p, p, 2, 3, 5, p, p, None, None)

    def call(c, t=track, m=nomap, a=args):
        return L.f110_predict_scored(ctypes.byref(sim), ctypes.byref(m), None, ctypes.byref(bm),
                                     ctypes.byref(t) if t is not None else None, ctypes.byref(a),
                                     ctypes.byref(c) if c is not None else None, None)

    assert call(_cost()) == -2                               # the positive control: everything up to the map is accepted
    assert call(None) == -1 and call(_cost(), t=None) == -1
    bad_tracks = [nat.F110Track(2, 3, p, p), nat.F110Track(0, 3, p, p), nat.F110Track(1, 2, p, p), nat.F110Track(1, 3, None, p),
                  nat.F110Track(1, 3, p, None)]
    for t in bad_tracks:
        assert call(_cost(), t=t) == -1, (t.num_tables, t.min_segments)
    stack = nat.F110Map(); ctypes.pointer(stack)[0] = nomap; stack.num_layers = 2
    assert call(_cost(), t=nat.F110Track(2, 3, p, p), m=stack) == -2     # two tables on a two-layer stack
    assert call(_cost(), t=track, m=stack) == -1
    for over in ({'cost': None}, {'seg0': None}, {'s0': None}, {'back': -1}, {'fwd': -1}, {'back': 1000, 'fwd': 24},
                 {'reacquire_dist': 0.0}, {'reacquire_dist': -1.0}, {'reacquire_dist': NAN}, {'reacquire_dist': math.inf},
                 {'clear_min': NAN}, {'clear_min': math.inf}) + tuple(
                {k: v} for k in ('w_lat', 'w_head', 'w_clear', 'w_dsteer', 'w_dspeed', 'w_prog', 'w_wall')
                for v in (-1.0, NAN, math.inf)):
        assert call(_cost(**over)) == -1, over
    assert call(_cost(clear_min=-3.0, back=0, fwd=0, w_prog=0.0)) == -2
    # f110_predict's own refusals come first
    assert call(_cost(), a=nat.F110PredictArgs(p, p, 2, 3, 0, p, p, None, None)) == -1


def _mppi(p, **over):
    from f1tenth_gym_b200 import _native as nat
    g = nat.F110Mppi(2, 8, 5, p, p, p, p, 0.2, 1.0, -0.4, 0.4, -1.0, 8.0, 1.0, 7)
    for k, v in over.items():
        setattr(g, k, v)
    return g


def test_mppi_calls_reject_before_any_launch():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    buf = (ctypes.c_double * 64)()
    p = ctypes.addressof(buf)
    sim, _, _ = _lean_setup(buf)
    bad = [{'M': 0}, {'K': 1}, {'K': 4097}, {'H': 0}, {'H': 1001}, {'M': 1 << 20, 'K': 4096, 'H': 1000},
           {'agent_ids': None}, {'nominal': None}, {'iteration': None}, {'no_finite': None},
           {'sigma_steer': -0.1}, {'sigma_speed': NAN}, {'steer_lo': 0.5}, {'speed_hi': math.inf}, {'speed_lo': NAN},
           {'lambda_': 0.0}, {'lambda_': -1.0}, {'lambda_': math.inf}]
    for over in bad:
        g = _mppi(p, **over)
        assert L.f110_mppi_sample(ctypes.byref(sim), ctypes.byref(g), None, p, None) == -1, over
        assert L.f110_mppi_update(ctypes.byref(g), p, p, p, 8, None, None, None) == -1, over
    g = _mppi(p)
    assert L.f110_mppi_sample(None, ctypes.byref(g), None, p, None) == -1
    assert L.f110_mppi_sample(ctypes.byref(sim), ctypes.byref(g), None, None, None) == -1
    nocnt = nat.F110Sim(); ctypes.pointer(nocnt)[0] = sim; nocnt.steer_cnt = None
    assert L.f110_mppi_sample(ctypes.byref(nocnt), ctypes.byref(g), None, p, None) == -1
    ep = nat.F110Episodes(); ep.terminated = p                     # truncated missing
    assert L.f110_mppi_sample(ctypes.byref(sim), ctypes.byref(g), ctypes.byref(ep), p, None) == -1
    assert L.f110_mppi_sample(ctypes.byref(sim), None, None, p, None) == -1
    for a, c, o, rows in ((None, p, p, 8), (p, None, p, 8), (p, p, None, 8), (p, p, p, 0)):
        assert L.f110_mppi_update(ctypes.byref(g), a, c, o, rows, None, None, None) == -1
    assert L.f110_mppi_update(None, p, p, p, 8, None, None, None) == -1


def test_kernel_resource_budget():
    """k_scored_rollout holds k_predict's rollout plus the tracker and cost (at most 168 registers: three 128-thread blocks per
    SM); the acquire and MPPI kernels are small.  No local memory anywhere (no spills); the stack only for the rollout's
    out-of-line slow paths."""
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack), rest) for fn, reg, stack, rest in
             re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)([^\n]*)', out)}
    scored = [k for k in usage if 'k_scored_rollout' in k]
    assert len(scored) == 3, scored
    for k in scored:
        reg, stack, rest = usage[k]
        assert reg <= 168 and stack <= 64, (k, usage[k])
        assert re.search(r'LOCAL:0\b', rest), (k, rest)
    for name, regs in (('k_scored_acquire', 64), ('k_mppi_sample', 64), ('k_mppi_update', 64)):
        ks = [k for k in usage if name in k]
        assert len(ks) == 1, (name, ks)
        reg, stack, rest = usage[ks[0]]
        assert reg <= regs and stack == 0 and re.search(r'LOCAL:0\b', rest), (name, usage[ks[0]])


# ----------------------------------------------------------------------------- Python ValueErrors
@pytest.fixture
def sim(f110):
    dm = f110.DeviceMap.from_yaml(f110.maps.resolve_map_path('example_map'), '.png', CPU)
    s = f110.Simulator(f110.maps.DEFAULT_PARAMS, 2, 1, num_envs=3, device=CPU)
    s.set_device_map(dm)
    return s


def test_predict_cost_value_errors(f110, sim):
    act = np.zeros((2, 3, 4, 2))
    with pytest.raises(ValueError, match='centerlines'):
        sim.predict(act, agent_ids=[0, 1], cost={})
    sim.set_centerlines(f110.maps.load_waypoints()[:, :2])
    for cost in ({'w_foo': 1.0}, {'w_lat': -1.0}, {'w_prog': NAN}, {'w_wall': math.inf}, {'clear_min': NAN},
                 {'w_head': 'x'}, [1.0]):
        with pytest.raises(ValueError):
            sim.predict(act, agent_ids=[0, 1], cost=cost)
    for prev in (np.zeros((3, 2)), np.zeros((2,))):
        with pytest.raises(ValueError):
            sim.predict(act, agent_ids=[0, 1], cost={}, prev_action=prev)
    with pytest.raises(ValueError):
        sim.predict(act, agent_ids=[0, 1], prev_action=np.zeros((2, 2)))   # prev_action without a cost


def test_mppi_planner_value_errors(f110, sim):
    with pytest.raises(ValueError, match='centerlines'):
        f110.MPPIPlanner(sim, [0], 10, 16)
    sim.set_centerlines(f110.maps.load_waypoints()[:, :2])
    ok = dict(agent_ids=[0, 2, 4], horizon=10, samples=16)
    f110.MPPIPlanner(sim, **ok)                                   # the positive control
    for over in ({'agent_ids': []}, {'agent_ids': [0, 6]}, {'agent_ids': [-1]}, {'agent_ids': [0, 0]}, {'agent_ids': [0.5]},
                 {'agent_ids': [[0, 1]]}, {'horizon': 0}, {'horizon': 1001}, {'horizon': 2.5}, {'samples': 1},
                 {'samples': 4097}, {'noise_std': (0.1,)}, {'noise_std': (-0.1, 1.0)}, {'noise_std': (NAN, 1.0)},
                 {'noise_std': 0.3}, {'temperature': 0.0}, {'temperature': NAN}, {'weights': {'w_lat': -1}},
                 {'weights': {'nope': 1}}, {'bounds': (0.4, -0.4, 0, 8)}, {'bounds': (0, 1, 0)},
                 {'bounds': (0, 1, 0, NAN)}):
        with pytest.raises(ValueError):
            f110.MPPIPlanner(sim, **dict(ok, **over))
    p = f110.MPPIPlanner(sim, **ok)
    assert p.bounds == (f110.maps.DEFAULT_PARAMS['s_min'], f110.maps.DEFAULT_PARAMS['s_max'],
                        f110.maps.DEFAULT_PARAMS['v_min'], f110.maps.DEFAULT_PARAMS['v_max'])
    assert p.nominal.shape == (3, 10, 2)
    with pytest.raises(ValueError):
        p.plan_into(torch.zeros((6, 2), dtype=torch.float64))       # not on the device
    with pytest.raises(ValueError):
        p.reset(np.zeros(2, bool))
    p.reset(np.array([True, False, False]))
