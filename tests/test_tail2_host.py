"""k_tail2 without a GPU: the register, stack and shared-memory budget of the built kernel, and the bound on the beam intervals
that its task record holds."""
import importlib.util
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, 'f1tenth_gym_b200', 'csrc', 'f110_b200.cu')


def study():
    spec = importlib.util.spec_from_file_location('tail_cast_study', os.path.join(ROOT, 'tools', 'tail_cast_study.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_tail2_kernel_resource_budget():
    """k_tail2 keeps the budget it was measured with: 80 registers (three 256-thread or six 128-thread blocks per SM), no more
    stack than the GJK arrays need, and under 6 KB of static shared memory (the per-ego poses and the per-rank offsets)."""
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    lib_path = os.path.join(os.path.dirname(os.path.abspath(nat.__file__)), 'libf110_b200.so')
    out = subprocess.run([tool, '-res-usage', lib_path], capture_output=True, text=True).stdout
    usage = {fn: (int(r), int(st), int(sh)) for fn, r, st, sh in
             re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)', out)}
    name = '_ZN4f1107k_tail2E8f110_simNS_8BeamViewEiNS_13AutoResetArgsEdi'
    assert name in usage, name
    reg, stack, shared = usage[name]
    assert reg <= 80, reg
    assert stack <= 1056, stack
    assert shared <= 6144, shared


def test_tail2_record_constants_match_the_study():
    src = open(SRC).read()
    assert re.search(r'#define F110_TAIL2_IVALS (\d+)', src).group(1) == str(study().IVALS)
    # the record stays 120 bytes (launch record: smem = envs per block * A (A - 1) * 120)
    body = re.search(r'struct Tail2Task \{(.*?)\};', src, re.S).group(1)
    assert 'double phi, cone;' in body and 'double v[8];' in body and 'int iv[2 * F110_TAIL2_IVALS];' in body
    assert 'int pad[2];' in body


@pytest.mark.parametrize('B', [270, 1080, 2160])
def test_tail2_interval_count_bound(B):
    """Over fov <= 2 pi and cone <= pi / 2 + 0.05 (the window rule makes cone <= asin(0.8) + 0.05) a wide window needs at most
    F110_TAIL2_IVALS intervals, disjoint and ascending, inside [lo, hi]: the fall-back to [lo, hi] is never taken there."""
    m = study()
    worst = 0
    for fov in np.linspace(0.5, 2 * math.pi, 14):
        inc = fov / (B - 1)
        for cone in np.linspace(0.0, math.pi / 2 + 0.05, 12):
            for d in np.linspace(-math.pi, math.pi, 73):
                for lo, hi in ((0, B - 1), (0, B // 2), (B // 3, B - 1)):
                    if hi - lo < 96:
                        continue
                    iv, whole = m.task_intervals(lo, hi, d, 0.0, cone, fov, inc, ivals=99)
                    assert not whole
                    worst = max(worst, len(iv))
                    prev = lo - 1
                    for i0, i1 in iv:
                        assert prev < i0 <= i1 <= hi
                        prev = i1
    assert worst <= m.IVALS, worst


def test_tail2_interval_overflow_falls_back_to_the_whole_window():
    """A window that would need more intervals than the record holds (here a field of view of 4 pi) is stored as [lo, hi]."""
    m = study()
    B, fov = 2160, 4 * math.pi
    iv, whole = m.task_intervals(0, B - 1, 0.3, 0.0, 0.5, fov, fov / (B - 1))
    assert whole and iv == [(0, B - 1)]
    iv, whole = m.task_intervals(0, B - 1, 0.3, 0.0, 0.5, fov, fov / (B - 1), ivals=99)
    assert not whole and len(iv) > m.IVALS
