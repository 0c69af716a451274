"""Generate tests/golden/kat_progress.npz from the UNMODIFIED reference: examples/waypoint_follow.py:16-47
nearest_point_on_trajectory (numba), imported the way make_golden.kat_planner imports the planner.

Run in the build container only (needs the reference tree):   python tests/golden/make_golden_progress.py

The committed fixture was made with numba 0.65.0, numpy 2.3.5 and scipy 1.18.1 on an Intel Xeon (x86-64 with FMA).  The
reference's np.dot of two 2-vectors goes through numba to BLAS ddot, here scipy's bundled OpenBLAS 0.3.31.dev (SkylakeX
kernels), which fuses the second product into the sum: dot = fma(py - y, dy, (px - x) * dx).  The device kernel and the model
of tests/test_progress_host.py do the same, and test_reference_dot_is_fused pins it.  Another BLAS, or a CPU without FMA,
could round those dot products differently and so change t (and rarely the segment) in the last bit: regenerate with the
same stack, or check that test first.

Tables (each stored closed, as the reference takes it: the last row repeats the first)
  table0   examples/example_waypoints.csv columns x, y as shipped (its last row already repeats its first)
  table1-3 trackgen.random_tracks(5, 3) waypoints in metres, closed with vstack(T, T[0])
Poses per table (2400 finite + 8 non-finite; yaw uniform in [-2pi, 2pi])
  exactly on every other vertex; on the closing segment; outside corners, where the projections on the two segments that
  meet there clamp to the shared vertex (t = 1 and t = 0: a tie the first minimum decides); near the line (|offset| < 1 m);
  far off the track (up to 200 m away); and non-finite coordinates.
Fixture arrays per table k: tables_k (n+1, 2), poses_k (M, 3), seg_k, t_k, dist_k (the reference's min_dist_segment, t and
dist for the finite poses; a non-finite pose has no reference row: the projection defines NaN for it, see DESIGN §3.7).
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, '..', '..')
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402


def reference_nearest():
    ref_import.load()
    for name in ('gym', 'pyglet', 'pyglet.gl'):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules['pyglet.gl'].GL_POINTS = 0
    sys.modules['pyglet'].gl = sys.modules['pyglet.gl']
    ex = os.path.join(ref_import.REF_ROOT, 'examples')
    if ex not in sys.path:
        sys.path.insert(0, ex)
    import waypoint_follow as wf
    return wf.nearest_point_on_trajectory


def tables():
    wp = np.loadtxt(os.path.join(ref_import.REF_ROOT, 'examples', 'example_waypoints.csv'), delimiter=';', skiprows=3)
    out = [np.ascontiguousarray(wp[:, 1:3])]
    from f1tenth_gym_b200 import trackgen
    for t in trackgen.random_tracks(5, 3):
        T = np.ascontiguousarray(t.waypoints)
        out.append(np.vstack([T, T[0]]))
    return out


def poses_for(C, rng):
    """C: the closed table (n+1, 2)."""
    T = C[:-1]
    n = T.shape[0]
    d = np.roll(T, -1, axis=0) - T
    u = d / np.sqrt((d * d).sum(axis=1))[:, None]
    P = []
    P.append(T[::2])                                                    # on vertices
    w = rng.random(100)
    P.append(T[n - 1] + w[:, None] * (T[0] - T[n - 1]))                 # on the closing segment
    # outside corners: along the outward bisector of the two unit normals, at least as far out as both clamps
    k = rng.integers(0, n, 600)
    uin, uout = u[(k - 1) % n], u[k]
    b = uout - uin
    nb = np.sqrt((b * b).sum(axis=1))
    ok = nb > 1e-9
    b[ok] /= nb[ok, None]
    b[~ok] = 0.0
    P.append(T[k] - b * rng.uniform(0.01, 3.0, 600)[:, None])
    k = rng.integers(0, n, 700)
    nrm = np.stack([-u[k, 1], u[k, 0]], axis=1)
    P.append(T[k] + d[k] * rng.random(700)[:, None] + nrm * rng.uniform(-1, 1, 700)[:, None])      # near the line
    lo, hi = T.min(axis=0) - 200, T.max(axis=0) + 200
    m = 2400 - sum(p.shape[0] for p in P)
    P.append(rng.uniform(lo, hi, (m, 2)))                                # far off the track
    xy = np.concatenate(P)
    return np.concatenate([xy, rng.uniform(-2 * np.pi, 2 * np.pi, (xy.shape[0], 1))], axis=1)


def main():
    nearest = reference_nearest()
    rng = np.random.default_rng(2026)
    arrays = {}
    bad = np.array([[np.nan, 0, 0], [0, np.nan, 0], [0, 0, np.nan], [np.inf, 0, 0], [0, -np.inf, 0], [0, 0, np.inf],
                    [np.nan, np.nan, np.nan], [1e308 * 10, 0, 0]])
    for ti, C in enumerate(tables()):
        poses = poses_for(C, rng)
        seg, t, dist = (np.empty(poses.shape[0]) for _ in range(3))
        for m, p in enumerate(poses):
            _, dist[m], t[m], seg[m] = nearest(np.ascontiguousarray(p[:2]), C)
        arrays['table_%d' % ti] = C
        arrays['poses_%d' % ti] = np.concatenate([poses, bad])
        arrays['seg_%d' % ti] = seg.astype(np.int32)
        arrays['t_%d' % ti] = t
        arrays['dist_%d' % ti] = dist
        print('table %d: %d points, %d poses, t==0: %d, t==1: %d' % (ti, C.shape[0] - 1, poses.shape[0], int((t == 0).sum()),
                                                                     int((t == 1).sum())))
    path = os.path.join(HERE, 'kat_progress.npz')
    np.savez_compressed(path, num_tables=len(tables()), **arrays)
    print('kat_progress.npz %8.1f KB' % (os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
