"""Static box obstacles on the host side: candidate boxes along a centerline, and the respawn draw restated in numpy.

A box row is (x, y, yaw, length, width) in metres and radians, the layout of f110_obstacles.boxes (include/f110_b200.h).
"""
import numpy as np

M64 = (1 << 64) - 1
_C_TICK, _C_ENV, _C_SLOT, _C_COUNT = 0xA0761D6478BD642F, 0xE7037ED1A0B428DB, 0x8EBC6AF09C88C6E3, 0x589965CC75374CC3


def obstacle_candidates(centerline, count, lateral=(-0.5, 0.5), size=(0.58, 0.31), yaw_jitter=0.0, seed=0):
    """`count` candidate boxes (count, 5) along a closed centerline ((n, 2+) table of x, y, the one set_centerlines takes; a last
    row equal to the first is dropped): a point uniform in arc length, moved sideways by an offset uniform in `lateral`
    (positive = left of the direction of travel), heading along its segment plus a yaw uniform in [-yaw_jitter, yaw_jitter],
    size = (length, width).  numpy only and deterministic in `seed`."""
    p = np.asarray(centerline, dtype=np.float64)
    if p.ndim != 2 or p.shape[1] < 2:
        raise ValueError('centerline must be an (n, 2) table of x, y')
    p = p[:, :2]
    if p.shape[0] > 1 and np.array_equal(p[0], p[-1]):
        p = p[:-1]
    if p.shape[0] < 3 or not np.isfinite(p).all():
        raise ValueError('centerline needs at least 3 finite points')
    count = int(count)
    lo, hi = (float(v) for v in lateral)
    length, width = (float(v) for v in size)
    if count < 1 or not (np.isfinite(lo) and np.isfinite(hi) and lo <= hi):
        raise ValueError('count must be >= 1 and lateral a finite (lo, hi) with lo <= hi')
    if not (np.isfinite(length) and np.isfinite(width) and length > 0 and width > 0):
        raise ValueError('size must be a finite (length, width) > 0')
    if not (np.isfinite(yaw_jitter) and yaw_jitter >= 0):
        raise ValueError('yaw_jitter must be finite and >= 0')
    d = np.roll(p, -1, axis=0) - p
    seg = np.hypot(d[:, 0], d[:, 1])
    if not (seg > 0).all():
        raise ValueError('centerline has a zero-length segment')
    cum = np.concatenate([[0.0], np.cumsum(seg)])
    rng = np.random.default_rng(seed)
    s = rng.uniform(0.0, cum[-1], count)
    off = rng.uniform(lo, hi, count)
    jit = rng.uniform(-yaw_jitter, yaw_jitter, count)
    i = np.clip(np.searchsorted(cum, s, side='right') - 1, 0, p.shape[0] - 1)
    t = (s - cum[i]) / seg[i]
    h = np.arctan2(d[i, 1], d[i, 0])
    x = p[i, 0] + t * d[i, 0] - off * np.sin(h)
    y = p[i, 1] + t * d[i, 1] + off * np.cos(h)
    return np.stack([x, y, h + jit, np.full(count, length), np.full(count, width)], axis=1)


def _mix64(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def _unit(h):
    return float(h >> 11) * (1.0 / 9007199254740992.0)


def respawn_draw(candidates, agent_xy, K, count, clearance, seed, tick, env):
    """The device's respawn of one env (obst_respawn_one, csrc/obstacles.cuh), restated: candidates (C, 5) = the env's own table,
    agent_xy (A, 2) the agents' new positions -> (boxes (K, 5), active (K,) uint8), bit for bit."""
    cand = np.asarray(candidates, dtype=np.float64).reshape(-1, 5)
    C = cand.shape[0]
    lo, hi = (int(v) for v in count)
    base = (int(seed) + _C_TICK * (int(tick) + 1) + _C_ENV * (int(env) + 1)) & M64
    span = hi - lo + 1
    c = lo + min(int(_unit(_mix64((base + _C_COUNT) & M64)) * span), span - 1)
    clr2 = float(clearance) * float(clearance)
    xy = np.asarray(agent_xy, dtype=np.float64).reshape(-1, 2)
    boxes = np.empty((K, 5))
    active = np.zeros(K, np.uint8)
    for k in range(K):
        j = min(int(_unit(_mix64((base + _C_SLOT * (k + 1)) & M64)) * C), C - 1)
        boxes[k] = cand[j]
        on = k < c
        for ax, ay in xy:
            dx, dy = cand[j, 0] - ax, cand[j, 1] - ay
            if dx * dx + dy * dy < clr2:
                on = False
        active[k] = 1 if on else 0
    return boxes, active
