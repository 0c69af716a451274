"""f110_scan_layers (ABI v6) on the CPU: the export and the ABI version, every argument combination it must refuse before
anything is enqueued, and the register and stack budget of its kernel k_scan_lean (DESIGN.md §3.5).

Nothing here launches a kernel: the maps are built in host memory, and their pointers are only passed to calls that must
reject them first.
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

from test_multimap_host import MAPS, TRACKS

CPU = torch.device('cpu')
INVALID, NO_MAP = -1, -2


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def maps(f110):
    load = lambda n, e: f110.DeviceMap.from_yaml(os.path.join(MAPS, n + '.yaml'), e, CPU)  # noqa: E731
    em, berlin, vegas = load('example_map', '.png'), load(*TRACKS[0]), load(*TRACKS[1])
    h = berlin.host
    rot = f110.DeviceMap(f110.maps.HostMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.35)), CPU)
    return {'single': berlin, 'cells': em, 'rot_single': rot,
            'same_size': f110.DeviceMap.stack([em, em]),
            'canvas': f110.DeviceMap.stack([berlin, vegas]),
            'mixres': f110.DeviceMap.stack([berlin, em], mixed_resolution=True),
            'rot': f110.DeviceMap.stack([rot, vegas], rotated_origins=True)}


@pytest.fixture(scope='module')
def beams(f110):
    return f110.DeviceBeams(1080, 4.7, f110.maps.DEFAULT_PARAMS, CPU)


def call(f110, mc, bc, M=4, poses=True, ids=True, out=True):
    """f110_scan_layers with host buffers standing in for device ones (never dereferenced when the call is refused)."""
    p = np.zeros((max(M, 1), 3))
    lid = np.zeros(max(M, 1), np.int32)
    o = np.zeros(8, np.float32)
    addr = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
    return f110._native.lib().f110_scan_layers(C.byref(mc), C.byref(bc), addr(p) if poses else None,
                                                addr(lid) if ids else None, M, addr(o) if out else None, None, None, None)


def copy(st):
    return type(st).from_buffer_copy(st)


def test_export_and_abi_version(f110):
    L = f110._native.lib()
    assert L.f110_abi_version() == 6 == f110._native.ABI_VERSION
    assert 'f110_scan_layers' in f110._native.SIGNATURES
    assert hasattr(L, 'f110_scan_layers')
    with open(os.path.join(os.path.dirname(__file__), '..', 'include', 'f110_b200.h')) as f:
        hdr = f.read()
    assert re.search(r'int f110_scan_layers\(const f110_map \*map, const f110_beams \*beams, const double \*poses, '
                     r'const int32_t \*layer_ids, int32_t M,', hdr)
    assert '#define F110_ABI_VERSION 6' in hdr


def test_no_map(f110, beams):
    assert call(f110, f110.simulator.empty_map_struct(), beams.c) == NO_MAP


def test_table_rules(f110, maps, beams):
    """The tick's rules: layer_res needs layer_geom and no fast_path; layer_rot needs both tables and no fast_path."""
    cases = []
    m = copy(maps['mixres'].c); m.layer_geom = None; cases.append(('layer_res without layer_geom', m))
    m = copy(maps['mixres'].c); m.fast_path = 1; cases.append(('layer_res with fast_path', m))
    m = copy(maps['mixres'].c); m.layer_res_min = 0.0; cases.append(('layer_res_min 0', m))
    m = copy(maps['single'].c); m.layer_res = maps['mixres'].c.layer_res; cases.append(('layer_res on one map', m))
    m = copy(maps['rot'].c); m.layer_res = None; cases.append(('layer_rot without layer_res', m))
    m = copy(maps['rot'].c); m.layer_geom = None; cases.append(('layer_rot without layer_geom', m))
    m = copy(maps['rot'].c); m.fast_path = 1; cases.append(('layer_rot with fast_path', m))
    m = copy(maps['rot_single'].c); m.layer_rot = maps['rot'].c.layer_rot; cases.append(('layer_rot on one map', m))
    m = copy(maps['same_size'].c); m.orig_c, m.orig_s = math.cos(0.3), math.sin(0.3)
    cases.append(('rotated same-size stack', m))
    for name, mc in cases:
        assert call(f110, mc, beams.c) == INVALID, name


def test_layer_ids_null_on_a_stack(f110, maps, beams):
    for k in ('same_size', 'canvas', 'mixres', 'rot'):
        assert maps[k].c.num_layers == 2
        assert call(f110, maps[k].c, beams.c, ids=False) == INVALID, k


def test_lean_preconditions(f110, maps, beams):
    for k in ('single', 'cells', 'rot_single', 'canvas', 'rot'):
        m = copy(maps[k].c); m.sincos2 = None
        assert call(f110, m, beams.c) == INVALID, (k, 'sincos2')
        m = copy(maps[k].c); m.dt_min_positive = m.eps
        assert call(f110, m, beams.c) == INVALID, (k, 'dt_min_positive')
        m = copy(maps[k].c); m.dt_min_positive = 0.0
        assert call(f110, m, beams.c) == INVALID, (k, 'dt_min_positive unknown')
        for fov in (2 * math.pi, 7.0):
            b = copy(beams.c); b.fov = fov
            assert call(f110, maps[k].c, b) == INVALID, (k, fov)


def test_sizes_and_pointers(f110, maps, beams):
    mc = maps['canvas'].c
    B = beams.num_beams
    big = (1 << 32) // B + 1                       # the smallest M with M * B >= 2^32
    assert big * B >= 1 << 32 and (big - 1) * B < 1 << 32
    assert call(f110, mc, beams.c, M=big) == INVALID
    assert call(f110, mc, beams.c, M=0x7fffffff) == INVALID
    assert call(f110, mc, beams.c, M=0) == INVALID
    assert call(f110, mc, beams.c, M=-3) == INVALID
    assert call(f110, mc, beams.c, poses=False) == INVALID
    assert call(f110, mc, beams.c, out=False) == INVALID
    b = copy(beams.c); b.num_beams = 1
    assert call(f110, mc, b) == INVALID


# ----------------------------------------------------------------------------- resource budget
# k_scan_lean<UNITS, COUNT> -> (registers, stack bytes), DESIGN.md §3.5; UNITS 0 = cells, 1 = metres, 2 = rot
SCAN_BUDGET = {(u, c): (60, 8) for u in (0, 1, 2) for c in (0, 1)}


def test_scan_kernel_resource_budget():
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    for (units, count), want in SCAN_BUDGET.items():
        name = '_ZN4f11011k_scan_leanILi%dELb%dEEEvNS_9ScanLeanKE' % (units, count)
        assert usage.get(name) == want, (name, usage.get(name))
