"""Host-side checks of episode mode (C ABI f110_episodes, include/f110_episodes.h; no GPU).

  * The ctypes mirror of f110_episodes against the header's offsetof, and the exported entry point.
  * Every rejection of f110_tick_episodes returns F110_ERR_INVALID before anything is enqueued: a sim that passes check_sim, no
    map (so a call that gets past the episode checks returns F110_ERR_NO_MAP instead, the positive control).
  * The register and stack budget of the kernels only an episode tick launches.
  * F110Env(autoreset=...) refuses single-env mode, action_repeat > 1 and a bad dict before any device work.
"""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, '..', 'include', 'f110_episodes.h')


def test_episodes_struct_matches_c_layout(tmp_path):
    from f1tenth_gym_b200 import _native as nat
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){',
             'printf("size %zu\\n", sizeof(f110_episodes));']
    for f, _ in nat.F110Episodes._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(f110_episodes, %s));' % (f, f))
    lines.append('printf("abi %d\\n", F110_ABI_VERSION); return 0;}')
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out['size']) == ctypes.sizeof(nat.F110Episodes)
    for f, _ in nat.F110Episodes._fields_:
        assert int(out[f]) == getattr(nat.F110Episodes, f).offset, f
    assert int(out['abi']) == 6


def test_episodes_entry_point_exported():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    assert 'f110_tick_episodes' in nat.EPISODE_SIGNATURES and hasattr(L, 'f110_tick_episodes')
    assert L.f110_abi_version() == 6
    declared = set(re.findall(r'^\S[^(;]*?\b(f110_\w+)\s*\(', open(HEADER).read(), re.M))
    assert declared == set(nat.EPISODE_SIGNATURES) == {'f110_tick_episodes'}


def _sim(nat, A):
    sim = nat.F110Sim()
    buf = (ctypes.c_double * 64)()
    p = ctypes.addressof(buf)
    sim.num_envs, sim.num_agents = 1, A
    sim.integrator = 1
    for f in ('params', 'state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'scans', 'wall_flag', 'collisions',
              'collision_idx', 'current_time', 'lap_times', 'lap_counts', 'toggle_list', 'near_starts', 'start_xs', 'start_ys',
              'start_thetas', 'start_rot', 'done'):
        setattr(sim, f, p)
    return sim, buf, p


@pytest.mark.parametrize('A', [1, 2, 32, 33])
def test_episodes_rejects_before_any_launch(A):
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    sim, buf, p = _sim(nat, A)
    mp, bm = nat.F110Map(), nat.F110Beams()

    def ep(**over):
        e = nat.F110Episodes(0, *([p] * 12), None)
        for k, v in over.items():
            setattr(e, k, v)
        return e

    def call(e, start=p, num_start=4, lidar=None):
        return L.f110_tick_episodes(ctypes.byref(sim), ctypes.byref(mp), None, ctypes.byref(bm), p, start, num_start, 23, 1, None,
                                    None if lidar is None else ctypes.byref(lidar), None if e is None else ctypes.byref(e), None)

    if A <= 32:
        assert call(ep()) == -2                                   # positive controls: past every episode check to the missing map
        assert call(ep(max_ticks=200, track_seg=p)) == -2
    else:
        assert call(ep()) == -1                                   # more than 32 agents per env
    assert call(None) == -1
    assert call(ep(max_ticks=-1)) == -1
    assert call(ep(), start=None, num_start=0) == -1
    assert call(ep(), num_start=0) == -1
    for f, _ in nat.F110Episodes._fields_:
        if f not in ('max_ticks', 'track_seg'):
            assert call(ep(**{f: None})) == -1, f
    if 1 < A < 32:
        assert call(ep(), lidar=nat.F110Lidar(1 << A, p, p, None)) == -1     # what f110_tick_lidar rejects
    del buf


# registers and stack of the sm_90a build (cuobjdump -res-usage); k_episode_end's stack is the start-pose staging of the auto-reset
EPISODE_BUDGET = {'k_episode_end': (64, 1024), 'k_episode_dyn': (136, 40), 'k_restart_march': (80, 0), 'k_episode_cast': (128, 40),
                  'k_episode_tail': (112, 256), 'k_episode_obstacles': (127, 176)}


def test_episodes_kernel_resource_budget():
    """The restart march keeps at least three 256-thread blocks per SM and no stack; the others stay within the budgets of the
    kernels they copy."""
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    for name, (reg, stack) in EPISODE_BUDGET.items():
        found = [k for k in usage if name in k]
        assert found, name
        for k in found:
            assert usage[k][0] <= reg and usage[k][1] <= stack, (k, usage[k])
    assert len([k for k in usage if 'k_restart_march' in k]) == 6


def test_env_autoreset_rejected_before_device_work():
    from f1tenth_gym_b200 import F110Env
    table = [[0.0, 0.0, 0.0]]
    with pytest.raises(ValueError):
        F110Env(map='example_map', autoreset={'poses': table})                          # single env
    with pytest.raises(ValueError):
        F110Env(map='example_map', num_envs=4, action_repeat=2, autoreset={'poses': table})
    for bad in ({}, {'poses': table, 'bogus': 1}, {'poses': table, 'max_episode_steps': -1}, {'poses': [[0.0, 0.0]]},
                {'poses': table, 'max_episode_steps': 1.5}, [table]):
        with pytest.raises(ValueError):
            F110Env(map='example_map', num_envs=4, autoreset=bad)
