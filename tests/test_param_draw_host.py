"""Host-side checks of per-episode parameter draws (C ABI f110_param_draw, include/f110_param_draw.h; no GPU).

  * The ctypes mirror of f110_param_draw against the header's offsetof, and the draw constants against the header; the
    header's entry points against PARAM_DRAW_SIGNATURES, and their export.
  * Every rejection of the three entry points returns F110_ERR_INVALID before anything is enqueued.  Only rejected calls are
    made: every other argument is valid, so a missing check would reach the launch and fail here with F110_ERR_CUDA.
  * The register and stack budget of k_param_draw.
  * Every ValueError of the validator set_param_draw and F110Env(param_draw=...) run (param_draw.parse / check_table), raised
    before any device work, and the restated draw's groups, slots and per_env.
"""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, '..', 'include', 'f110_param_draw.h')


def test_param_draw_struct_matches_c_layout(tmp_path):
    from f1tenth_gym_b200 import _native as nat
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){',
             'printf("size %zu\\n", sizeof(f110_param_draw));']
    for f, _ in nat.F110ParamDraw._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(f110_param_draw, %s));' % (f, f))
    for j in range(1, 5):
        lines.append('printf("C%d %%llu\\n", (unsigned long long)F110_PARAM_DRAW_C%d);' % (j, j))
    lines.append('printf("keys %d\\n", F110_PARAM_DRAW_KEYS);')
    lines.append('printf("abi %d\\n", F110_ABI_VERSION); return 0;}')
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out['size']) == ctypes.sizeof(nat.F110ParamDraw)
    for f, _ in nat.F110ParamDraw._fields_:
        assert int(out[f]) == getattr(nat.F110ParamDraw, f).offset, f
    from f1tenth_gym_b200 import param_draw as pd
    assert tuple(int(out['C%d' % j]) for j in range(1, 5)) == nat.PARAM_DRAW_C == (pd.C_TICK, pd.C_ENV, pd.C_SLOT, pd.C_GROUP)
    assert all(c & 1 for c in nat.PARAM_DRAW_C)
    assert int(out['keys']) == nat.PARAM_DRAW_KEYS == pd.DRAWABLE == 16
    assert int(out['abi']) == 6


def test_param_draw_entry_points_exported():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    declared = set(re.findall(r'^\S[^(;]*?\b(f110_\w+)\s*\(', open(HEADER).read(), re.M))
    assert declared == set(nat.PARAM_DRAW_SIGNATURES) == {'f110_params_draw', 'f110_params_draw_autoreset',
                                                          'f110_params_draw_episodes'}
    for name in declared:
        assert hasattr(L, name), name


@pytest.mark.parametrize('A', [1, 2, 32])
def test_param_draw_rejects_before_any_launch(A):
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    buf = (ctypes.c_double * 64)()
    p = ctypes.addressof(buf)

    def sim(**over):
        s = nat.F110Sim()
        s.num_envs, s.num_agents, s.integrator, s.params_per_env = 2, A, 1, 1
        for f in ('params', 'state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'scans', 'wall_flag', 'collisions',
                  'collision_idx', 'tick_counter'):
            setattr(s, f, p)
        for k, v in over.items():
            setattr(s, k, v)
        return s

    def draw(keys=None, group=None, **over):
        d = nat.F110ParamDraw()
        d.lo = d.hi = p
        for i in range(A):
            d.keys[i] = 1
        for q in range(18):
            d.group[q] = q
        for i, v in (keys or {}).items():
            d.keys[i] = v
        for q, v in (group or {}).items():
            d.group[q] = v
        for k, v in over.items():
            setattr(d, k, v)
        return d

    def ep(**over):
        e = nat.F110Episodes(0, *([p] * 12), None)
        for k, v in over.items():
            setattr(e, k, v)
        return e

    def calls(s=None, d=None, e=None):
        s = sim() if s is None else s
        d = draw() if d is None else d
        e = ep() if e is None else e
        sr = None if s is False else ctypes.byref(s)
        dr = None if d is False else ctypes.byref(d)
        return (L.f110_params_draw(sr, dr, p, None), L.f110_params_draw_autoreset(sr, dr, None),
                L.f110_params_draw_episodes(sr, dr, None if e is False else ctypes.byref(e), None))

    bad = (-1, -1, -1)
    assert calls(s=False) == bad
    assert calls(d=False) == bad
    assert calls(d=draw(lo=None)) == bad
    assert calls(d=draw(hi=None)) == bad
    assert calls(s=sim(params_per_env=0)) == bad
    assert calls(s=sim(num_agents=33)) == bad
    assert calls(s=sim(tick_counter=None)) == bad
    assert calls(s=sim(params=None)) == bad
    assert calls(s=sim(num_envs=0)) == bad
    assert calls(s=sim(num_agents=0)) == bad
    for bit in (16, 17, 31):
        assert calls(d=draw(keys={A - 1: 1 << bit})) == bad, bit
    for g in (-1, 18, 1 << 30):
        assert calls(d=draw(group={17: g})) == bad, g
        assert calls(d=draw(group={0: g})) == bad, g
    # rule 2 reads collisions at the ego slot, rule 3 the episode flags: only the rule that reads them is called (the others
    # would accept these arguments and launch)
    for s in (sim(collisions=None), sim(ego_idx=A), sim(ego_idx=-1)):
        assert L.f110_params_draw_autoreset(ctypes.byref(s), ctypes.byref(draw()), None) == -1
    for e in (None, ep(terminated=None), ep(truncated=None)):
        assert L.f110_params_draw_episodes(ctypes.byref(sim()), ctypes.byref(draw()), None if e is None else ctypes.byref(e),
                                           None) == -1
    del buf


# registers and stack of the sm_90a build (cuobjdump -res-usage)
DRAW_BUDGET = {'_ZN4f11012k_param_drawENS_10ParamDrawKE': (40, 0)}


def test_param_draw_kernel_resource_budget():
    """The draw runs after every tick that can restart an env: few registers and no stack (its by-value key masks are read
    from the parameter bank, not copied to the stack)."""
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    for name, (reg, stack) in DRAW_BUDGET.items():
        assert name in usage, name
        assert usage[name][0] <= reg and usage[name][1] <= stack, (name, usage[name])


BAD_RANGES = [
    ({'mu': (1.0, 0.5)}, 'lo <= hi'),
    ({'mu': (0.5, float('inf'))}, 'finite'),
    ({'mu': (float('nan'), 1.0)}, 'finite'),
    ({'mu': 1.0}, r'\(lo, hi\)'),
    ({'mu': (1.0, 2.0, 3.0)}, r'\(lo, hi\)'),
    ({'bogus': (1.0, 2.0)}, 'unknown'),
    ({'width': (0.2, 0.3)}, 'not drawable'),
    ({'length': (0.5, 0.6)}, 'not drawable'),
    ({'mu': (0.0, 1.0)}, 'mu > 0'),
    ({'m': (-1.0, 1.0)}, 'm > 0'),
    ({'v_max': (0.0, 0.0)}, 'v_max > 0'),
    ({'h': (-0.01, 0.1)}, 'h >= 0'),
    ({'s_min': (-0.4, 0.1)}, 's_min <= 0'),
    ({'sv_min': (-3.0, 1e-9)}, 'sv_min <= 0'),
    ({'s_max': (-0.1, 0.4)}, 's_max >= 0'),
    ({'v_min': (-5.0, 1.0)}, 'v_min < 0'),
    ({'v_min': (0.0, 0.0)}, 'v_min < 0'),
]


@pytest.mark.parametrize('ranges,msg', BAD_RANGES)
def test_param_draw_validator_rejects_ranges(ranges, msg):
    from f1tenth_gym_b200 import F110Env
    from f1tenth_gym_b200 import param_draw as pd
    with pytest.raises(ValueError, match=msg):
        pd.parse(ranges, None, False, 0, 2)
    with pytest.raises(ValueError, match=msg):
        pd.parse([{}, ranges], None, False, 0, 2)
    with pytest.raises(ValueError, match=msg):
        F110Env(map='example_map', num_envs=4, param_draw={'ranges': ranges})


def test_param_draw_validator_rejects_the_rest():
    from f1tenth_gym_b200 import F110Env, maps
    from f1tenth_gym_b200 import param_draw as pd
    ok = {'mu': (0.5, 1.5), 'm': (3.0, 4.0), 'I': (0.04, 0.05)}
    d = pd.parse(ok, [['m', 'I']], True, 7, 2)            # the positive control
    assert d['group'][6] == d['group'][7] == 6 and list(d['keys']) == [(1 << 0) | (1 << 6) | (1 << 7)] * 2
    assert sorted(pd.parse([{}, ok], None, False, 0, 2)['keys']) == [0, d['keys'][0]]
    for groups in ([['m', 'm']], [['m', 'I'], ['I']], [[]], [['width']], [['bogus']], ['mI'], [3]):
        with pytest.raises(ValueError):
            pd.parse(ok, groups, False, 0, 2)
    for ranges in ([ok], [ok, ok, ok], None, 'mu', [ok, None]):
        with pytest.raises(ValueError):
            pd.parse(ranges, None, False, 0, 2)
    # hi = 0 is never drawn: u < 1, and lo + u (hi - lo) stays below 0 at the largest u
    pd.parse({'v_min': (-5.0, 0.0)}, None, False, 0, 2)
    with pytest.raises(ValueError, match='32'):
        pd.parse({}, None, False, 0, 33)
    # the undrawn values of a drawn slot must keep the sign conditions; a slot without drawn keys is not checked
    table = np.tile(maps.params_vector(maps.DEFAULT_PARAMS), (3, 2, 1))
    pd.check_table(table, d)
    bad = table.copy()
    bad[1, 0, maps.PARAM_KEYS.index('sv_max')] = -1.0
    with pytest.raises(ValueError, match='sv_max'):
        pd.check_table(bad, d)
    bad[1, 0, maps.PARAM_KEYS.index('sv_max')] = 3.2
    bad[2, 1, maps.PARAM_KEYS.index('v_min')] = 0.0
    with pytest.raises(ValueError, match='v_min'):
        pd.check_table(bad, d)
    pd.check_table(bad, pd.parse([ok, {}], None, False, 0, 2))
    bad[2, 1, maps.PARAM_KEYS.index('mu')] = 0.0            # drawn in slot 1: its table value does not matter
    pd.check_table(table, d)
    # F110Env: the dict, the mode, and the undrawn values of its params
    for cfg in ({'ranges': ok, 'bogus': 1}, {'groups': [['m', 'I']]}, {'ranges': None}, 'mu', {'ranges': ok, 'seed': 'x'},
                {'ranges': ok, 'groups': [['width']]}):
        with pytest.raises(ValueError):
            F110Env(map='example_map', num_envs=4, param_draw=cfg)
    with pytest.raises(ValueError, match='batched'):
        F110Env(map='example_map', param_draw={'ranges': ok})
    params = dict(maps.DEFAULT_PARAMS, a_max=0.0)
    with pytest.raises(ValueError, match='a_max'):
        F110Env(map='example_map', num_envs=4, params=params, param_draw={'ranges': ok})


def test_restated_draw_groups_slots_and_per_env():
    """The numpy restatement: keys of one group move together, slots draw apart unless per_env, undrawn keys stay."""
    from f1tenth_gym_b200 import maps
    from f1tenth_gym_b200 import param_draw as pd
    ranges = {'mu': (0.5, 1.5), 'm': (3.0, 5.0), 'I': (0.03, 0.06), 'C_Sf': (4.0, 5.0)}
    table = np.tile(maps.params_vector(maps.DEFAULT_PARAMS), (6, 2, 1))
    K = maps.PARAM_KEYS
    d = pd.parse(ranges, [['m', 'I']], False, 3, 2)
    out = pd.draw_rows(table, d, 41, [1, 4])
    assert np.array_equal(out[[0, 2, 3, 5]], table[[0, 2, 3, 5]])
    frac = lambda e, i, k: (out[e, i, K.index(k)] - ranges[k][0]) / (ranges[k][1] - ranges[k][0])
    for e in (1, 4):
        for i in (0, 1):
            assert abs(frac(e, i, 'm') - frac(e, i, 'I')) < 1e-12
            assert frac(e, i, 'm') != frac(e, i, 'mu')
            for k in ranges:
                assert ranges[k][0] <= out[e, i, K.index(k)] <= ranges[k][1]
        assert out[e, 0, K.index('mu')] != out[e, 1, K.index('mu')]
        undrawn = [q for q in range(18) if K[q] not in ranges]
        assert np.array_equal(out[e][:, undrawn], table[e][:, undrawn])
    assert out[1, 0, 0] != out[4, 0, 0]
    assert not np.array_equal(pd.draw_rows(table, d, 42, [1])[1], out[1])
    shared = pd.draw_rows(table, pd.parse(ranges, None, True, 3, 2), 41, [1])
    assert np.array_equal(shared[1, 0], shared[1, 1])
