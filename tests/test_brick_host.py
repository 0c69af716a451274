"""The 4 x 4-cell brick table of the ray march (f110_march_tables.dt_cells_brick, DESIGN.md §3.2), on the CPU.

  * the host model of f110_map_brick (maps.brick_table) read through the kernel's index expression (maps.brick_index, the
    form of csrc/march_lean.cuh brick_index) gives the padded row-major table's value at every cell of every cell-unit map,
    the padding row and column included, and at every clamped off-map coordinate; synthetic maps cover every width and
    height modulo 4;
  * the brick table is built for single cell-unit maps only: CPU maps and stacks carry none, and the f110_map struct of a
    DeviceMap is what it was;
  * the register and stack budget of the brick kernels (DESIGN.md §3.2, codegen caveat).
"""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
CPU = torch.device('cpu')


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


def cell_unit_tables(f110):
    """(name, dt / res) of every bundled map on the cell-unit path, and random tables of every height and width mod 4."""
    out = []
    for name in ('berlin', 'example_map', 'levine', 'skirk', 'stata_basement', 'vegas'):
        ext = '.pgm' if name == 'levine' else '.png'
        h = f110.maps.load_map(os.path.join(MAPS, name + '.yaml'), ext)
        if h.fast_path:
            out.append((name, h.dt / h.resolution))
    assert [n for n, _ in out] == ['example_map']
    rng = np.random.default_rng(7)
    for H in (1, 2, 3, 4, 5, 6, 7, 8):
        for W in (1, 2, 3, 4, 5, 6, 7, 8, 37):
            out.append(('random %dx%d' % (H, W), np.sqrt(rng.integers(0, 4000, (H, W)).astype(np.float64))))
    return out


def check_table(f110, cells):
    H, W = cells.shape
    pad = f110.maps.pad_table(cells)
    brick = f110.maps.brick_table(pad)
    assert brick.dtype == np.float64 and brick.size == (-(-(H + 1) // 4) * 4) * (-(-(W + 1) // 4) * 4)
    r, c = np.meshgrid(np.arange(H + 1), np.arange(W + 1), indexing='ij')
    idx = f110.maps.brick_index(r, c, W)
    assert idx.min() >= 0 and idx.max() < brick.size
    assert np.unique(idx).size == idx.size                 # one element per cell
    # bit for bit: the padded table, its extra row and column included
    assert np.array_equal(brick[idx].view(np.int64), pad.view(np.int64))
    # what the kernel reads for an off-map coordinate: min(r, H), min(c, W) on the unsigned cell coordinates
    big = np.array([-(1 << 31), -7, -1, H, H + 1, H + 5, (1 << 31) - 1], dtype=np.int64)
    rr = np.minimum(big.astype(np.uint32), H).astype(np.int64)
    cc = np.minimum(np.concatenate([big, [W, W + 3]]).astype(np.uint32), W).astype(np.int64)
    for r0 in rr:
        for c0 in cc:
            v = brick[f110.maps.brick_index(r0, c0, W)]
            assert v == pad[r0, c0]
            if r0 == H or c0 == W:
                assert v == cells[-1, -1]
    # the cells that round the table up to whole bricks hold dt[-1,-1] too
    rest = np.ones(brick.size, bool)
    rest[idx.ravel()] = False
    assert np.all(brick[rest] == cells[-1, -1])


def test_brick_index_reads_the_padded_table(f110):
    for name, cells in cell_unit_tables(f110):
        check_table(f110, cells)


def test_brick_table_only_for_single_device_maps(f110):
    h = f110.maps.load_map(os.path.join(MAPS, 'example_map.yaml'), '.png')
    m = f110.DeviceMap(h, CPU)
    # no device table on the host; the f110_map struct is unchanged and the tick's table struct is empty
    assert m.dt_cells_brick is None and not m.march_tables.dt_cells_brick
    assert [f for f, _ in f110._native.F110Map._fields_][-1] == 'layer_rot'
    st = f110.DeviceMap.stack([m, f110.DeviceMap(h, CPU)])
    assert st.dt_cells_brick is None and not st.march_tables.dt_cells_brick


def test_brick_entry_points_are_declared_and_bound(f110):
    header = open(os.path.join(os.path.dirname(__file__), '..', 'include', 'f110_b200.h')).read()
    for name in ('f110_step_ex', 'f110_step_profile_ex', 'f110_tick_ex', 'f110_step_host_async_ex', 'f110_map_brick',
                 'f110_map_brick_elems'):
        assert re.search(r'\b%s\(' % name, header), name
        assert name in f110._native.SIGNATURES, name
    assert '#define F110_ABI_VERSION 6' in header
    L = f110._native.lib()
    # no table on a map without the padded cell-unit table
    assert L.f110_map_brick_elems(f110.simulator.empty_map_struct()) == 0
    assert L.f110_map_brick(f110.simulator.empty_map_struct(), None, None) == -1


def test_brick_kernel_resource_budget():
    """k_march_lean_brick at the launches step_impl picks: 32 registers (64 warps per SM) and at most 24 bytes of stack, the
    budget of k_march_lean (test_host_logic.test_march_kernel_resource_budget)."""
    import shutil
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    lib_path = os.path.join(os.path.dirname(os.path.abspath(nat.__file__)), 'libf110_b200.so')
    out = subprocess.run([tool, '-res-usage', lib_path], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    # k_march_lean_brick<NOISE, COUNT=0, 512 threads, 4 blocks/SM, DYN, IPT, RING>
    names = ['_ZN4f11018k_march_lean_brickILb%dELb0ELi512ELi4ELb1ELi%dELi2EEEvNS_5LeanKENS_10MarchQueueE' % (noise, ipt)
             for noise in (0, 1) for ipt in (4, 2, 0)]
    names.append('_ZN4f11018k_march_lean_brickILb0ELb0ELi512ELi4ELb0ELi1ELi0EEEvNS_5LeanKENS_10MarchQueueE')
    for name in names:
        assert name in usage, name
        reg, stack = usage[name]
        assert reg <= 32, (name, reg)
        assert stack <= 24, (name, stack)
