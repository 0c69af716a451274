"""Centerline progress on the CPU: the two exports and their header declarations, the ctypes layout of f110_track and
f110_progress, every argument f110_track_project / f110_track_progress refuse before anything is enqueued, the Python-side
ValueErrors, the drop of a repeated end point, the register and stack budget of the two kernels (DESIGN.md §3.7), and a numpy
model of the projection and of the tracker (csrc/progress.cuh).

The model's projection equals the reference's nearest_point_on_trajectory (tests/golden/kat_progress.npz) bit for bit in
seg, t and dist, and disagrees with it when the tie rule is changed.  tests/test_gpu_progress.py compares both kernels with
this model.
"""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

CPU = torch.device('cpu')
INVALID = -1
HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, '..', 'include', 'f110_b200.h')
GOLDEN = os.path.join(HERE, 'golden', 'kat_progress.npz')
TWO_PI, PI = 2 * np.pi, np.pi
NONE = np.iinfo(np.int64).max


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


def golden():
    g = np.load(GOLDEN)
    return g, int(g['num_tables'])


# ----------------------------------------------------------------------------- the model
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a
    h = c - (c - a)
    return h, a - h


def fma(a, b, c):
    """Correctly rounded a * b + c, elementwise (fp64 arrays of moderate magnitude: no overflow or underflow in the steps).
    Exact product by Dekker's split, exact sum with c, the low parts added with round-to-odd, then one rounding (Boldo and
    Melquiond, 'Emulation of FMA and correctly rounded sums: proved algorithms using rounding to odd', 2008)."""
    with np.errstate(invalid='ignore', over='ignore'):
        uh = a * b
        ah, al = _split(a)
        bh, bl = _split(b)
        ul = ((ah * bh - uh) + ah * bl + al * bh) + al * bl
        th, tl = _two_sum(c, uh)
        s, e = _two_sum(tl, ul)
        even = (s.view(np.int64) & 1) == 0
        s = np.where((e != 0) & even, np.nextafter(s, np.copysign(np.inf, e)), s)
        r = th + s
    return np.where(np.isfinite(r), r, a * b + c)


def test_fma_emulation_is_exact():
    from fractions import Fraction
    rng = np.random.default_rng(3)
    a, b, c = (rng.normal(0, 1, 4000) * 10.0 ** rng.integers(-3, 4, 4000) for _ in range(3))
    c[:1000] = -a[:1000] * b[:1000]                                      # heavy cancellation
    got = fma(a, b, c)
    for k in range(a.size):
        assert got[k] == float(Fraction(a[k]) * Fraction(b[k]) + Fraction(c[k])), k


def window_search(rec, px, py, base, W, tie='first'):
    """First minimum of dist over window positions k = 0 .. W-1, segment (base + k) mod n, for P poses at once.
    px, py, base: (P,); W int.  Returns (k (P,) int64, NONE where every dist is NaN or inf; t; dist), in the kernel's
    operation order.  tie='last' (a deliberate mutation) takes the last minimum instead."""
    n = rec.shape[0]
    idx = (base[:, None] + np.arange(W)[None, :]) % n
    x, y, dx, dy, l2 = (rec[idx, c] for c in range(5))
    with np.errstate(invalid='ignore', over='ignore'):
        dot = fma(py[:, None] - y, dy, (px[:, None] - x) * dx)          # the reference's np.dot (BLAS ddot)
        t = dot / l2
        t = np.where(t < 0.0, 0.0, t)
        t = np.where(t > 1.0, 1.0, t)
        qx, qy = x + t * dx, y + t * dy
        ex, ey = px[:, None] - qx, py[:, None] - qy
        d = np.sqrt(ex * ex + ey * ey)
        valid = d < np.inf
    dd = np.where(valid, d, np.inf)
    k = np.argmin(dd, axis=1) if tie == 'first' else W - 1 - np.argmin(dd[:, ::-1], axis=1)
    rows = np.arange(px.shape[0])
    k = np.where(valid.any(axis=1), k, NONE)
    kk = np.where(k == NONE, 0, k)
    return k, t[rows, kk], d[rows, kk]


def outputs(rec, seg, t, px, py, yaw):
    """(t, dist, s, d, e) of poses on segments seg at t, in the kernel's operation order."""
    x, y, dx, dy = rec[seg, 0], rec[seg, 1], rec[seg, 2], rec[seg, 3]
    with np.errstate(invalid='ignore', over='ignore'):
        qx, qy = x + t * dx, y + t * dy
        ex, ey = px - qx, py - qy
        dist = np.sqrt(ex * ex + ey * ey)
        s = rec[seg, 5] + t * rec[seg, 6]
        d = np.where(dx * ey - dy * ex >= 0.0, dist, -dist)
        e = yaw - rec[seg, 7]
        e = e - TWO_PI * np.floor((e + PI) / TWO_PI)
    return t, dist, s, d, e


def project_model(recs, poses, table_ids=None, tie='first'):
    """(M, 5) = (seg, t, d, s, e) of f110_track_project; recs: list of (n, 8) records."""
    poses = np.asarray(poses, dtype=np.float64)
    M = poses.shape[0]
    ids = np.zeros(M, np.int64) if table_ids is None else np.asarray(table_ids, np.int64)
    out = np.full((M, 5), np.nan)
    fin = np.isfinite(poses).all(axis=1)
    for tb, rec in enumerate(recs):
        sel = np.nonzero(fin & (ids == tb))[0]
        if not sel.size:
            continue
        px, py, yaw = poses[sel, 0], poses[sel, 1], poses[sel, 2]
        k, t, _ = window_search(rec, px, py, np.zeros(sel.size, np.int64), rec.shape[0], tie)
        ok = k != NONE
        sel, k, t, px, py, yaw = sel[ok], k[ok], t[ok], px[ok], py[ok], yaw[ok]
        t, _, s, d, e = outputs(rec, k, t, px, py, yaw)
        out[sel] = np.stack([k.astype(np.float64), t, d, s, e], axis=1)
    return out


class TrackerModel(object):
    """The per-agent state of f110_track_progress and one update."""

    def __init__(self, recs, NA, back=8, fwd=56, reacquire_dist=5.0):
        self.recs, self.back, self.fwd, self.r = recs, back, fwd, reacquire_dist
        self.lengths = [rec[-1, 5] + rec[-1, 6] for rec in recs]
        self.seg = np.full(NA, -1, np.int64)
        self.s, self.d, self.e, self.progress, self.delta = (np.zeros(NA) for _ in range(5))

    def update(self, state, steer_cnt, table_of_agent):
        """state (7, NA); steer_cnt (NA,); table_of_agent (NA,) table ids."""
        px, py, yaw = state[0], state[1], state[4]
        NA = px.shape[0]
        nan = np.full(NA, np.nan)
        ok = np.isfinite(px) & np.isfinite(py) & np.isfinite(yaw) & (table_of_agent >= 0) & \
            (table_of_agent < len(self.recs))
        bad = ~ok
        self.seg[bad] = -1
        for arr in (self.s, self.d, self.e, self.progress, self.delta):
            arr[bad] = nan[bad]
        for tb, rec in enumerate(self.recs):
            n = rec.shape[0]
            sel = np.nonzero(ok & (table_of_agent == tb))[0]
            if not sel.size:
                continue
            sg = self.seg[sel]
            acquire = (sg < 0) | (sg >= n) | (steer_cnt[sel] == 0)
            seg = np.full(sel.size, NONE)
            t = np.zeros(sel.size)
            tr = np.nonzero(~acquire)[0]
            if tr.size:
                base = (sg[tr] - self.back) % n
                k, tt, dist = window_search(rec, px[sel[tr]], py[sel[tr]], base, min(self.back + self.fwd + 1, n))
                good = (k != NONE) & (dist <= self.r)
                seg[tr[good]] = (base[good] + k[good]) % n
                t[tr[good]] = tt[good]
            glob = np.nonzero(seg == NONE)[0]
            if glob.size:
                k, tt, _ = window_search(rec, px[sel[glob]], py[sel[glob]], np.zeros(glob.size, np.int64), n)
                seg[glob], t[glob] = k, tt
            lost = seg == NONE
            if lost.any():
                ls = sel[lost]
                self.seg[ls] = -1
                for arr in (self.s, self.d, self.e, self.progress, self.delta):
                    arr[ls] = np.nan
            keep = ~lost
            sl, seg, t, acq = sel[keep], seg[keep], t[keep], acquire[keep]
            _, _, s, d, e = outputs(rec, seg, t, px[sl], py[sl], yaw[sl])
            L = self.lengths[tb]
            delta = s - self.s[sl]
            delta = np.where(delta > L * 0.5, delta - L, np.where(delta < -(L * 0.5), delta + L, delta))
            delta = np.where(acq, 0.0, delta)
            prog = np.where(acq, 0.0, self.progress[sl] + delta)
            self.seg[sl] = seg
            self.s[sl], self.d[sl], self.e[sl], self.progress[sl], self.delta[sl] = s, d, e, prog, delta


def records(f110, table):
    return f110.simulator.centerline_segments(table)[0]


# ----------------------------------------------------------------------------- model vs the reference
def test_model_equals_reference_golden(f110):
    g, T = golden()
    for tb in range(T):
        rec = records(f110, g['table_%d' % tb])
        assert rec.shape[0] == g['table_%d' % tb].shape[0] - 1          # the repeated end point is dropped
        poses = g['poses_%d' % tb]
        ref = g['seg_%d' % tb].shape[0]
        out = project_model([rec], poses)
        assert np.array_equal(out[:ref, 0].astype(np.int64), g['seg_%d' % tb]), tb
        assert np.array_equal(out[:ref, 1], g['t_%d' % tb]), tb
        assert np.array_equal(np.abs(out[:ref, 2]), g['dist_%d' % tb]), tb
        assert np.isnan(out[ref:]).all(), tb                             # non-finite poses: NaN rows
        assert ((out[:ref, 3] >= 0) & (out[:ref, 3] <= rec[-1, 5] + rec[-1, 6])).all()
        assert ((out[:ref, 4] >= -np.pi) & (out[:ref, 4] < np.pi)).all()


def test_golden_covers_ties_clamps_and_closing_segment(f110):
    g, T = golden()
    for tb in range(T):
        n = g['table_%d' % tb].shape[0] - 1
        seg, t = g['seg_%d' % tb], g['t_%d' % tb]
        assert (t == 0).any() and (t == 1).any() and ((t > 0) & (t < 1)).any()
        assert (seg == n - 1).sum() >= 50
        assert g['poses_%d' % tb].shape[0] >= 2000
        # ties: poses whose best distance is reached by more than one segment
        rec = records(f110, g['table_%d' % tb])
        poses = g['poses_%d' % tb][:seg.shape[0]]
        first = project_model([rec], poses)
        last = project_model([rec], poses, tie='last')
        assert (first[:, 0] != last[:, 0]).sum() >= 100, tb


def test_reference_dot_is_fused(f110):
    """The reference's np.dot fuses its second product: with two separate roundings the t values differ."""
    g, _ = golden()
    rec = records(f110, g['table_0'])
    ref = g['seg_0'].shape[0]
    P = g['poses_0'][:ref]
    k = g['seg_0']
    x, y, dx, dy, l2 = (rec[k, c] for c in range(5))
    t = np.clip(((P[:, 0] - x) * dx + (P[:, 1] - y) * dy) / l2, 0.0, 1.0)
    assert (t != g['t_0']).sum() > 100
    t = np.clip(fma(P[:, 1] - y, dy, (P[:, 0] - x) * dx) / l2, 0.0, 1.0)
    assert np.array_equal(t, g['t_0'])


def test_model_disagrees_with_last_minimum_tie_rule(f110):
    g, _ = golden()
    rec = records(f110, g['table_0'])
    ref = g['seg_0'].shape[0]
    out = project_model([rec], g['poses_0'], tie='last')
    assert not np.array_equal(out[:ref, 0].astype(np.int64), g['seg_0'])


def test_model_window_order_matters(f110):
    """On a window that wraps past segment 0, window order and index order pick different segments at a tie: the vertex
    point 0 is at distance 0 from segments n-1 (t = 1) and 0 (t = 0)."""
    g, _ = golden()
    rec = records(f110, g['table_0'])
    n = rec.shape[0]
    px, py = np.array([rec[0, 0]]), np.array([rec[0, 1]])
    k, t, d = window_search(rec, px, py, np.array([n - 3]), 8)
    assert (n - 3 + k[0]) % n == n - 1 and t[0] == 1.0 and d[0] == 0.0
    k, t, _ = window_search(rec, px, py, np.array([0]), n)
    assert k[0] == 0 and t[0] == 0.0


def test_tracker_model_windows_and_reacquire(f110):
    """A hairpin: two parallel straights 1 m apart.  A tracked agent on the lower straight that drifts to 0.6 m stays on it
    (the window does not reach the upper one), where the global projection jumps; a teleport beyond reacquire_dist
    re-acquires and keeps the progress."""
    tab = hairpin()
    rec = records(f110, tab)
    m = TrackerModel([rec], 1, back=2, fwd=4)
    st = np.zeros((7, 1))
    st[0, 0], st[1, 0] = 2.5, 0.0
    m.update(st, np.array([0]), np.array([0]))
    assert m.seg[0] == 2 and m.progress[0] == 0.0 and m.s[0] == 2.5
    st[0, 0], st[1, 0] = 3.5, 0.6
    m.update(st, np.array([1]), np.array([0]))
    assert m.seg[0] == 3 and m.progress[0] == 1.0 and abs(m.d[0] - 0.6) < 1e-12
    glob = project_model([rec], [[3.5, 0.6, 0.0]])
    assert glob[0, 0] == 17 and abs(glob[0, 2] - 0.4) < 1e-12                # the global projection jumps to the other branch
    st[0, 0], st[1, 0] = 8.0, -20.0                                          # teleport
    m.update(st, np.array([2]), np.array([0]))
    assert m.seg[0] == project_model([rec], [[8.0, -20.0, 0.0]])[0, 0] == 7
    assert m.delta[0] == 4.5 and m.progress[0] == 5.5
    m.update(st, np.array([0]), np.array([0]))                              # a reset: acquired afresh
    assert m.progress[0] == 0.0 and m.delta[0] == 0.0


def hairpin(length=10.0, gap=1.0, step=1.0):
    """A closed hairpin: the straight y = 0 from x = 0 to `length`, the straight y = gap back, in `step` m segments."""
    xs = np.arange(0.0, length + step / 2, step)
    lower = np.stack([xs, np.zeros_like(xs)], axis=1)
    upper = np.stack([xs[::-1], np.full_like(xs, gap)], axis=1)
    return np.concatenate([lower, upper])


# ----------------------------------------------------------------------------- host rules
def test_drop_of_repeated_end_point(f110):
    tab = hairpin()
    a, La = f110.simulator.centerline_segments(tab)
    b, Lb = f110.simulator.centerline_segments(np.vstack([tab, tab[0]]))
    assert np.array_equal(a, b) and La == Lb
    assert a.shape == (tab.shape[0], 8)
    assert La == np.cumsum(np.sqrt(np.diff(np.vstack([tab, tab[0]]), axis=0) ** 2 @ np.ones(2)))[-1]
    assert La == a[-1, 5] + a[-1, 6]                                          # what the kernel derives


def test_centerline_value_errors(f110):
    bad = [np.zeros((2, 2)) + [[0, 0], [1, 0]], np.array([[0, 0], [1, 0], [0, 0]]),      # < 3 points (after the drop)
           np.array([[0, 0], [1, 0], [1, np.nan]]), np.array([[0, 0], [1, 0], [np.inf, 1]]),
           np.array([[0, 0], [1, 0], [1, 0], [0, 1]]),                                 # zero-length segment
           np.zeros((4, 3)), np.zeros(4)]
    for tab in bad:
        with pytest.raises(ValueError):
            f110.simulator.centerline_segments(tab)


@pytest.fixture
def sim(f110):
    return f110.Simulator(f110.maps.DEFAULT_PARAMS, 2, 1, num_envs=3, device=CPU)


def test_simulator_value_errors(f110, sim):
    tab = hairpin()
    for kw in (dict(window=(0, 1024)), dict(window=(-1, 4)), dict(window=(4, -1)), dict(window=8),
               dict(reacquire_dist=0.0), dict(reacquire_dist=-1.0), dict(reacquire_dist=math.nan),
               dict(reacquire_dist=math.inf)):
        with pytest.raises(ValueError):
            sim.set_centerlines(tab, **kw)
    with pytest.raises(ValueError):                    # two tables for a simulator without a stacked map
        sim.set_centerlines([tab, tab])
    sim.set_centerlines(tab, window=(0, 0))
    sim.set_centerlines(tab, window=(1000, 23))
    assert sim.centerlines.num_tables == 1 and (sim.track_seg == -1).all()
    sim.set_centerlines(None)
    assert sim.centerlines is None and sim.track_seg is None
    with pytest.raises(ValueError):
        sim.update_progress()
    with pytest.raises(ValueError):
        sim.project_centerline([[0.0, 0.0, 0.0]])


def test_env_value_errors(f110):
    with pytest.raises(ValueError):
        f110.F110Env(map='vegas', device=CPU, reward='progress')
    with pytest.raises(ValueError):
        f110.F110Env(map='vegas', device=CPU, reward='speed')


def test_refused_update_map_changes_nothing(f110):
    """update_map without a centerline is refused with reward='progress' before any setting changes."""
    tab = np.loadtxt(os.path.join(HERE, '..', 'f1tenth_gym_b200', 'maps', 'example_waypoints.csv'), delimiter=';',
                     skiprows=3)[:, 1:3]
    env = f110.F110Env(map='example_map', num_envs=2, device=CPU, centerline=tab, reward='progress')
    tables = env.sim.centerlines
    with pytest.raises(ValueError):
        env.update_map(env.map_path, '.png', env_map_ids=[0, 0], mixed_resolution=True, rotated_origins=True)
    assert env.env_map_ids is None and not env.mixed_resolution and not env.rotated_origins
    assert env.centerline is tab and env.sim.centerlines is tables


# ----------------------------------------------------------------------------- the C ABI
def test_exports_and_header(f110):
    L = f110._native.lib()
    assert L.f110_abi_version() == 6 == f110._native.ABI_VERSION
    for name in ('f110_track_project', 'f110_track_progress'):
        assert name in f110._native.SIGNATURES and hasattr(L, name)
    with open(HEADER) as fh:
        hdr = fh.read()
    assert re.search(r'int f110_track_project\(const f110_track \*track, const double \*poses, const int32_t \*table_ids, '
                     r'int32_t M, double \*out,\s+void \*stream\);', hdr)
    assert re.search(r'int f110_track_progress\(const f110_sim \*sim, const f110_track \*track, f110_progress \*progress, '
                     r'void \*stream\);', hdr)
    assert 'waypoint_follow.py:16-47' in hdr
    assert '#define F110_ABI_VERSION 6' in hdr


def test_ctypes_layout_matches_header(f110, tmp_path):
    nat = f110._native
    structs = {'f110_track': nat.F110Track, 'f110_progress': nat.F110Progress}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){']
    for cname, st in structs.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for f, _ in st._fields_:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
    lines.append('return 0;}')
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    for cname, st in structs.items():
        assert int(out[cname]) == C.sizeof(st), cname
        for f, _ in st._fields_:
            assert int(out['%s.%s' % (cname, f)]) == getattr(st, f).offset, (cname, f)


def copy(struct):
    return type(struct).from_buffer_copy(struct)


def test_refusals(f110, sim):
    """Every refusal returns F110_ERR_INVALID from the host, before a launch (there is no GPU here: a launch would fail with
    F110_ERR_CUDA instead)."""
    L = f110._native.lib()
    sim.set_centerlines(hairpin())
    tc, pc = sim.centerlines.c, sim._progress_c
    poses = torch.zeros((4, 3), dtype=torch.float64)
    out = torch.zeros((4, 5), dtype=torch.float64)
    ids = torch.zeros(4, dtype=torch.int32)
    P, O, I = poses.data_ptr(), out.data_ptr(), ids.data_ptr()

    def project(t, p=P, i=None, M=4, o=O):
        return L.f110_track_project(None if t is None else C.byref(t), p, i, M, o, None)
    assert project(None) == INVALID
    assert project(tc, p=None) == INVALID
    assert project(tc, o=None) == INVALID
    for M in (0, -1):
        assert project(tc, M=M) == INVALID
    for field, val in (('num_tables', 0), ('min_segments', 2), ('min_segments', 0), ('table_start', None),
                       ('segments', None)):
        t = copy(tc); setattr(t, field, val)
        assert project(t) == INVALID, field
        assert project(t, i=I) == INVALID, field
    t = copy(tc); t.num_tables = 2
    assert project(t) == INVALID                       # table_ids NULL with more than one table

    def progress(s=sim.c, t=tc, p=pc):
        return L.f110_track_progress(None if s is None else C.byref(s), None if t is None else C.byref(t),
                                     None if p is None else C.byref(p), None)
    assert progress(s=None) == INVALID
    assert progress(t=None) == INVALID
    assert progress(p=None) == INVALID
    for field in ('state', 'steer_cnt'):
        s = copy(sim.c); setattr(s, field, None)
        assert progress(s=s) == INVALID, field
    for field, val in (('num_envs', 0), ('num_agents', 0), ('num_envs', -3)):
        s = copy(sim.c); setattr(s, field, val)
        assert progress(s=s) == INVALID, field
    for field, val in (('num_tables', 0), ('min_segments', 2), ('table_start', None), ('segments', None)):
        t = copy(tc); setattr(t, field, val)
        assert progress(t=t) == INVALID, field
    for field in ('seg', 's', 'd', 'heading_error', 'progress', 'delta'):
        p = copy(pc); setattr(p, field, None)
        assert progress(p=p) == INVALID, field
    for back, fwd in ((-1, 4), (4, -1), (1024, 0), (0, 1024), (600, 600)):
        p = copy(pc); p.back, p.fwd = back, fwd
        assert progress(p=p) == INVALID, (back, fwd)
    for r in (0.0, -1.0, math.nan, math.inf, -math.inf):
        p = copy(pc); p.reacquire_dist = r
        assert progress(p=p) == INVALID, r


# ----------------------------------------------------------------------------- resource budget
# kernel -> (registers, stack bytes), DESIGN.md §3.7
PROGRESS_BUDGET = {'_ZN4f11015k_track_projectEPKdPKiiS1_S3_iPd': (56, 0),
                   '_ZN4f11016k_track_progressENS_6TrackKE': (56, 16)}


def test_progress_kernel_resource_budget():
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    for name, budget in PROGRESS_BUDGET.items():
        assert usage.get(name) == budget, (name, usage.get(name))
