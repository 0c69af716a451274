"""Per-episode parameter draws on the host side: the validation of a draw and the draw itself restated in numpy.

A draw (C ABI f110_param_draw, include/f110_param_draw.h) says, for each agent slot, which keys of the 18-key parameter vector
(maps.PARAM_KEYS order) are redrawn when an env starts a new episode, and from which range [lo, hi].  Keys of one group share
their uniform number; with per_env every slot of an env shares its draws.
"""
import numpy as np

from .maps import PARAM_KEYS

M64 = (1 << 64) - 1
DRAWABLE = 16                                   # keys 0..15; width and length (16, 17) are not drawable
C_TICK, C_ENV, C_SLOT, C_GROUP = 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x27D4EB2F165667C5, 0x85EBCA77C2B2AE63
_U_MAX = float((1 << 53) - 1) * (1.0 / 9007199254740992.0)      # the largest u of the draw

# the sign conditions under which a car at rest stays at rest under the action (0, 0) whatever the drawn values (DESIGN §3.13)
_SIGN = {}
for _k in ('mu', 'C_Sf', 'C_Sr', 'lf', 'lr', 'm', 'I', 'v_switch', 'a_max', 'v_max'):
    _SIGN[_k] = ('> 0', lambda v: v > 0)
_SIGN['h'] = ('>= 0', lambda v: v >= 0)
for _k in ('s_min', 'sv_min'):
    _SIGN[_k] = ('<= 0', lambda v: v <= 0)
for _k in ('s_max', 'sv_max'):
    _SIGN[_k] = ('>= 0', lambda v: v >= 0)
_SIGN['v_min'] = ('< 0', lambda v: v < 0)


def _mix64(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def parse(ranges, groups, per_env, seed, num_agents):
    """Validate a draw -> dict(lo (A, 18), hi (A, 18), keys (A,) bit masks, group (18,) int32, per_env, seed).  ranges: a
    {key: (lo, hi)} dict for every slot, or a list of num_agents such dicts ({} = the slot is never drawn); groups: None or a
    list of lists of keys that share their draw.  ValueError for an unknown or undrawable key, a range that is not a finite
    lo <= hi, a group that names a key twice or an undrawable key, and a range whose values could break the sign conditions
    (_SIGN).  Host only: nothing touches a device."""
    A = int(num_agents)
    if isinstance(ranges, dict):
        per_slot = [ranges] * A
    elif isinstance(ranges, (list, tuple)) and all(isinstance(r, dict) for r in ranges):
        per_slot = list(ranges)
        if len(per_slot) != A:
            raise ValueError('param_draw ranges as a list needs one dict per agent slot (%d), got %d' % (A, len(per_slot)))
    else:
        raise ValueError('param_draw ranges must be a {key: (lo, hi)} dict or a list of one per agent slot, got %r' % (ranges,))
    if A > 32:
        raise ValueError('param_draw covers at most 32 agent slots, this simulator has %d' % A)
    lo = np.zeros((A, 18))
    hi = np.zeros((A, 18))
    keys = np.zeros(A, dtype=np.uint32)
    for i, r in enumerate(per_slot):
        for k, v in r.items():
            q = _drawable_index(k, 'param_draw ranges')
            try:
                a, b = (float(x) for x in v)
            except (TypeError, ValueError):
                raise ValueError('param_draw range of %r must be (lo, hi), got %r' % (k, v))
            if not (np.isfinite(a) and np.isfinite(b) and a <= b):
                raise ValueError('param_draw range of %r must be finite with lo <= hi, got %r' % (k, v))
            # u -> lo + u * (hi - lo) is non-decreasing in u, so its values lie between those at u = 0 and at the largest u
            for x in (a, a + _U_MAX * (b - a)):
                if k in _SIGN and not _SIGN[k][1](x):
                    raise ValueError('param_draw range of %r must keep %s %s, got %r' % (k, k, _SIGN[k][0], v))
            lo[i, q], hi[i, q] = a, b
            keys[i] |= np.uint32(1 << q)
    group = np.arange(18, dtype=np.int32)
    seen = set()
    for g in ([] if groups is None else groups):
        if isinstance(g, str) or not hasattr(g, '__iter__'):
            raise ValueError('param_draw groups must be a list of lists of keys, got %r' % (groups,))
        idx = [_drawable_index(k, 'param_draw groups') for k in g]
        if not idx or seen & set(idx) or len(set(idx)) != len(idx):
            raise ValueError('param_draw groups must be non-empty and name each key at most once, got %r' % (groups,))
        seen |= set(idx)
        group[idx] = min(idx)
    return {'lo': lo, 'hi': hi, 'keys': keys, 'group': group, 'per_env': bool(per_env), 'seed': int(seed) & M64}


def _drawable_index(k, who):
    if k not in PARAM_KEYS:
        raise ValueError('%s: unknown parameter key %r' % (who, k))
    q = PARAM_KEYS.index(k)
    if q >= DRAWABLE:
        raise ValueError('%s: %r is not drawable (the opponent ray-cast and the collision body would disagree)' % (who, k))
    return q


def check_table(table, draw):
    """ValueError unless the undrawn values of every slot that has a drawn key keep the sign conditions in every env.
    table: (N, A, 18) host array."""
    t = np.asarray(table, dtype=np.float64)
    for i, m in enumerate(draw['keys']):
        if not m:
            continue
        for k, (text, ok) in _SIGN.items():
            q = PARAM_KEYS.index(k)
            if not (int(m) >> q) & 1 and not np.all(ok(t[:, i, q])):
                raise ValueError('param_draw: slot %d keeps its table value of %r, which must be %s in every env' % (i, k, text))


def draw_env(rows, draw, tick, env):
    """The device's draw (k_param_draw) of env `env` at tick counter `tick`, restated bit for bit: rows (A, 18) = the env's old
    rows -> a drawn copy."""
    out = np.array(rows, dtype=np.float64, copy=True)
    for i in range(out.shape[0]):
        m = int(draw['keys'][i])
        s = 0 if draw['per_env'] else i
        base = (draw['seed'] + C_TICK * (int(tick) + 1) + C_ENV * (int(env) + 1) + C_SLOT * (s + 1)) & M64
        for q in range(DRAWABLE):
            if (m >> q) & 1:
                h = _mix64((base + C_GROUP * (int(draw['group'][q]) + 1)) & M64)
                u = float(h >> 11) * (1.0 / 9007199254740992.0)
                lo, hi = draw['lo'][i, q], draw['hi'][i, q]
                out[i, q] = lo + u * (hi - lo)
    return out


def draw_rows(table, draw, tick, envs):
    """A copy of table (N, A, 18) whose rows of the envs in `envs` are drawn at tick counter `tick` (draw_env)."""
    out = np.array(table, dtype=np.float64, copy=True)
    for e in envs:
        out[e] = draw_env(out[e], draw, tick, e)
    return out
