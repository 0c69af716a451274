"""Host-side checks of the lidar mask (C ABI f110_lidar, no GPU).

  * The ctypes mirror of f110_lidar against the header's offsetof, F110_LIDAR_ALL and the three exported entry points.
  * Every rejection of the three _lidar entry points returns F110_ERR_INVALID before anything is enqueued: a sim that passes
    check_sim, no map (so a call that gets past the mask checks returns F110_ERR_NO_MAP instead, the positive control).
  * The register and stack budget of the kernels only a masked tick launches.
  * F110Env(lidar=...) in single-env mode is refused before any device work.
"""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, '..', 'include', 'f110_b200.h')


def test_lidar_struct_matches_c_layout(tmp_path):
    from f1tenth_gym_b200 import _native as nat
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){',
             'printf("size %zu\\n", sizeof(f110_lidar));']
    for f, _ in nat.F110Lidar._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(f110_lidar, %s));' % (f, f))
    lines.append('printf("all %u\\n", F110_LIDAR_ALL); printf("abi %d\\n", F110_ABI_VERSION); return 0;}')
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out['size']) == ctypes.sizeof(nat.F110Lidar)
    for f, _ in nat.F110Lidar._fields_:
        assert int(out[f]) == getattr(nat.F110Lidar, f).offset, f
    assert int(out['all']) == nat.LIDAR_ALL
    assert int(out['abi']) == 6


def test_lidar_entry_points_exported():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    for name in ('f110_step_lidar', 'f110_tick_lidar', 'f110_tick_repeat_ticks_lidar'):
        assert name in nat.SIGNATURES and hasattr(L, name), name
    assert L.f110_abi_version() == 6
    header = open(HEADER).read()
    declared = set(re.findall(r'^\S[^(;]*?\b(f110_\w+)\s*\(', header, re.M))
    assert len(declared) == 49, sorted(declared)
    assert declared <= set(nat.SIGNATURES) | set(nat.DEBUG_SIGNATURES), declared - set(nat.SIGNATURES)


def _sim_that_passes_check_sim(nat, A):
    sim = nat.F110Sim()
    buf = (ctypes.c_double * 64)()
    p = ctypes.addressof(buf)
    sim.num_envs, sim.num_agents = 1, A
    sim.integrator = 1
    for f in ('params', 'state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'scans', 'wall_flag', 'collisions',
              'collision_idx'):
        setattr(sim, f, p)
    return sim, buf, p


@pytest.mark.parametrize('A', [1, 2, 5, 32, 33])
def test_lidar_rejects_bad_masks_before_any_launch(A):
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()
    sim, buf, p = _sim_that_passes_check_sim(nat, A)
    mp, bm, rep = nat.F110Map(), nat.F110Beams(), nat.F110Repeat()
    rep.list, rep.list_count = p, p
    base = (ctypes.byref(sim), ctypes.byref(mp), None, ctypes.byref(bm), p)

    def calls(lidar):
        ref = None if lidar is None else ctypes.byref(lidar)
        return (L.f110_step_lidar(*base, None, ref, None),
                L.f110_tick_lidar(*base, 0, None, 0, 0, 0, None, ref, None),
                L.f110_tick_repeat_ticks_lidar(*base, 2, 0, 2, ctypes.byref(rep), 0, None, 0, 0, 0, None, ref, None))

    # positive controls: no mask, the ALL mask, and a valid mask get past the mask checks to the missing map
    assert calls(None) == (-2, -2, -2)
    assert calls(nat.F110Lidar(nat.LIDAR_ALL, None, None, None)) == (-2, -2, -2)
    if A <= 32:
        assert calls(nat.F110Lidar(1, p, p, None)) == (-2, -2, -2)
        assert calls(nat.F110Lidar(0, p, p, p)) == (-2, -2, -2)                  # no slot has a lidar
    bad = [nat.F110Lidar(0, None, p, None), nat.F110Lidar(0, p, None, None)]     # scratch missing, on either path
    if A < 32:
        bad.append(nat.F110Lidar(1 << A, p, p, None))                            # a bit at or above A
        bad.append(nat.F110Lidar(0x80000000, p, p, None))
    if A > 32:
        bad.append(nat.F110Lidar(1, p, p, None))                                 # any mask but ALL with A > 32
    for lidar in bad:
        assert calls(lidar) == (-1, -1, -1), (A, lidar.mask, lidar.list, lidar.list_count)
    assert L.f110_step_lidar(None, None, None, None, None, None, None, None) == -1
    del buf


# resources of the kernels only a tick with a lidar mask launches, as the build reports them (cuobjdump -res-usage)
LIDAR_BUDGET = {
    '_ZN4f11013k_lidar_orderE8f110_simNS_10LidarOrderE': (40, 0),
    '_ZN4f11012k_lidar_castE8f110_simNS_8BeamViewENS_10LidarOrderEd': (120, 40),
    '_ZN4f11011k_obstaclesILb1ELb1EEEv8f110_simNS_8BeamViewENS_5ObstKEd': (127, 176),
}


def test_lidar_kernel_resource_budget():
    """k_lidar_order keeps build_march_order's budget (no stack); k_lidar_cast and the masked k_obstacles stay at the registers
    and stack of the build they were measured with; k_ttc_select with its slot filter stays at <= 32 registers and no stack."""
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    for name, (reg, stack) in LIDAR_BUDGET.items():
        assert name in usage, name
        assert usage[name][0] <= reg and usage[name][1] <= stack, (name, usage[name])
    sel = [k for k in usage if 'k_ttc_select' in k]
    assert len(sel) == 1 and usage[sel[0]][0] <= 32 and usage[sel[0]][1] == 0


def test_env_lidar_single_env_rejected_before_device_work():
    from f1tenth_gym_b200 import F110Env
    with pytest.raises(ValueError):
        F110Env(map='example_map', lidar=[True, False])
