"""Host-side checks of episodes under a held action (C ABI f110_episode_repeat, include/f110_episode_repeat.h; no GPU).

  * The ctypes mirror of f110_episode_repeat against the header's offsetof; the header's entry points against
    EPISODE_REPEAT_SIGNATURES, and their export.
  * Every rejection of f110_tick_repeat_episodes(_ticks) returns F110_ERR_INVALID before anything is enqueued: a sim that passes
    check_sim, no map (so a call that gets past every other check returns F110_ERR_NO_MAP instead, the positive control).
  * The register and stack budget of the two kernels only this call launches.
  * F110Env(autoreset={..., 'action_repeat': K}) refuses a bad K, single-env mode and a top-level action_repeat before any
    device work.
"""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, '..', 'include', 'f110_episode_repeat.h')


def test_episode_repeat_struct_matches_c_layout(tmp_path):
    from f1tenth_gym_b200 import _native as nat
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){',
             'printf("size %zu\\n", sizeof(f110_episode_repeat));']
    for f, _ in nat.F110EpisodeRepeat._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(f110_episode_repeat, %s));' % (f, f))
    lines.append('printf("abi %d\\n", F110_ABI_VERSION); return 0;}')
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out['size']) == ctypes.sizeof(nat.F110EpisodeRepeat)
    for f, _ in nat.F110EpisodeRepeat._fields_:
        assert int(out[f]) == getattr(nat.F110EpisodeRepeat, f).offset, f
    assert int(out['abi']) == 6


def test_episode_repeat_entry_points_exported():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    declared = set(re.findall(r'^\S[^(;]*?\b(f110_\w+)\s*\(', open(HEADER).read(), re.M))
    assert declared == set(nat.EPISODE_REPEAT_SIGNATURES) == {'f110_tick_repeat_episodes', 'f110_tick_repeat_episodes_ticks'}
    for name in declared:
        assert hasattr(L, name), name
    assert L.f110_abi_version() == 6


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
def test_episode_repeat_rejects_before_any_launch(A):
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    sim, buf, p = _sim(nat, A)
    mp, bm = nat.F110Map(), nat.F110Beams()

    def ep(**over):
        e = nat.F110Episodes(0, *([p] * 12), None)
        for k, v in over.items():
            setattr(e, k, v)
        return e

    def er(**over):
        e = nat.F110EpisodeRepeat(*([p] * 6), None)
        for k, v in over.items():
            setattr(e, k, v)
        return e

    def rep(**over):
        r = nat.F110Repeat(p, p, p, p, None)
        for k, v in over.items():
            setattr(r, k, v)
        return r

    def calls(e=None, x=None, r=None, K=4, start=p, num_start=4, lidar=None, first=0, count=None):
        e = ep() if e is None else e
        x = er() if x is None else x
        r = rep() if r is None else r
        args = (start, num_start, 23, 1, None, None if lidar is None else ctypes.byref(lidar),
                None if e is False else ctypes.byref(e), None if x is False else ctypes.byref(x), None)
        whole = L.f110_tick_repeat_episodes(ctypes.byref(sim), ctypes.byref(mp), None, ctypes.byref(bm), p, K,
                                            None if r is False else ctypes.byref(r), *args)
        part = L.f110_tick_repeat_episodes_ticks(ctypes.byref(sim), ctypes.byref(mp), None, ctypes.byref(bm), p, K, first,
                                                 K - first if count is None else count, None if r is False else ctypes.byref(r),
                                                 *args)
        return whole, part

    if A <= 32:
        # positive controls: past every check to the missing map
        assert calls() == (-2, -2)
        assert calls(K=1) == (-2, -2)
        assert calls(e=ep(max_ticks=7, track_seg=p), x=er(track_delta_sum=p), r=rep(done_any=None, done_tick=None)) == (-2, -2)
        assert calls(first=2, count=2) == (-2, -2)
    else:
        assert calls() == (-1, -1)                                 # more than 32 agents per env
    # f110_tick_repeat's rejections
    for K in (0, -1, 65):
        assert calls(K=K, count=1) == (-1, -1), K
    assert calls(first=3, count=2)[1] == -1
    assert calls(first=-1, count=1)[1] == -1
    assert calls(count=0)[1] == -1
    assert calls(r=False) == (-1, -1)
    assert calls(r=rep(list=None)) == (-1, -1)
    assert calls(r=rep(list_count=None)) == (-1, -1)
    # f110_tick_episodes' rejections
    assert calls(e=False) == (-1, -1)
    assert calls(e=ep(max_ticks=-1)) == (-1, -1)
    assert calls(start=None, num_start=0) == (-1, -1)
    assert calls(num_start=0) == (-1, -1)
    for f, _ in nat.F110Episodes._fields_:
        if f not in ('max_ticks', 'track_seg'):
            assert calls(e=ep(**{f: None})) == (-1, -1), f
    # the new buffers
    assert calls(x=False) == (-1, -1)
    for f, _ in nat.F110EpisodeRepeat._fields_:
        if f != 'track_delta_sum':
            assert calls(x=er(**{f: None})) == (-1, -1), f
    if 1 < A < 32:
        assert calls(lidar=nat.F110Lidar(1 << A, p, p, None)) == (-1, -1)     # what f110_tick_lidar rejects
        assert calls(lidar=nat.F110Lidar(1, None, p, None)) == (-1, -1)
    del buf


# registers and stack of the sm_90a build (cuobjdump -res-usage); k_episode_restart's stack is the start-pose staging of the
# auto-reset, as k_episode_end's
REPEAT_BUDGET = {'_ZN4f11015k_episode_latchE8f110_simNS_6LatchKE': (40, 0),
                 '_ZN4f11017k_episode_restartE8f110_simNS_13AutoResetArgsENS_6LatchKENS_8ObstDrawEPiPdPjS6_': (64, 1024)}


def test_episode_repeat_kernel_resource_budget():
    """The latch runs after every tick: few registers, no stack.  The restart stays within k_episode_end's budget."""
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    for name, (reg, stack) in REPEAT_BUDGET.items():
        assert name in usage, name
        assert usage[name][0] <= reg and usage[name][1] <= stack, (name, usage[name])


def test_env_episode_repeat_rejected_before_device_work():
    from f1tenth_gym_b200 import F110Env
    table = [[0.0, 0.0, 0.0]]
    for K in (0, -1, 65, 1.5, True, None):
        with pytest.raises(ValueError):
            F110Env(map='example_map', num_envs=4, autoreset={'poses': table, 'action_repeat': K})
    with pytest.raises(ValueError):
        F110Env(map='example_map', autoreset={'poses': table, 'action_repeat': 4})             # single env
    with pytest.raises(ValueError, match='action_repeat'):
        F110Env(map='example_map', num_envs=4, action_repeat=2, autoreset={'poses': table})
    with pytest.raises(ValueError, match='action_repeat'):
        F110Env(map='example_map', num_envs=4, action_repeat=2, autoreset={'poses': table, 'action_repeat': 2})
    with pytest.raises(ValueError):
        F110Env(map='example_map', num_envs=4, autoreset={'poses': table, 'action_repeat': 2, 'bogus': 1})
