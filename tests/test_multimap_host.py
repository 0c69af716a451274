"""Canvas stacks of maps that differ in size and origin (DeviceMap.stack -> f110_map.layer_geom), on the CPU.

  * the canvas build: each layer's table in the low corner of its slice, that layer's dt[-1,-1] everywhere else (also in the
    extra row and column of the cell-unit padded table), the layer_geom rows, today's struct for a same-shape stack, and the
    ValueError cases;
  * a numpy restatement of k_march_lean_het's lookup (csrc/march_het.cuh) on the canvas -- cell units and metres -- against
    the oracle's per-layer xy_2_rc / distance_transform (oracle/f110_oracle.c dt_lookup) at >= 1e5 coordinates per layer,
    boundary builders of tests/boundary_inputs.py included; with the canvas x_max in place of the layer's it must disagree;
  * the register and stack budget of the new kernel (DESIGN.md §3.2).
"""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import boundary_inputs as bi

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
CPU = torch.device('cpu')
TRACKS = [('berlin', '.png'), ('vegas', '.png'), ('skirk', '.png'), ('levine', '.pgm')]


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def tracks(f110):
    return [f110.DeviceMap.from_yaml(os.path.join(MAPS, n + '.yaml'), e, CPU) for n, e in TRACKS]


def synthetic(f110, H, W, res, origin, seed):
    """A layer of random distances (every cell differs from its neighbours and from dt[-1,-1])."""
    rng = np.random.default_rng(seed)
    dt = res * np.sqrt(rng.integers(1, 4000, (H, W)).astype(np.float64))
    return f110.DeviceMap(f110.maps.HostMap(dt, res, origin), CPU)


def cropped(f110, dmap, r0, c0, H, W):
    """A crop of a cell-unit map with its origin moved so that the crop stays where it was, EDT recomputed from the crop
    (as a map of that size loaded from an image would be)."""
    from scipy.ndimage import distance_transform_edt as edt
    h = dmap.host
    free = (h.dt[r0:r0 + H, c0:c0 + W] > 0).astype(np.float64) * 255.
    return f110.DeviceMap(f110.maps.HostMap(h.resolution * edt(free), h.resolution,
                                            (h.orig_x + c0 * h.resolution, h.orig_y + r0 * h.resolution, 0.0)), CPU)


# ----------------------------------------------------------------------------- canvas build
def test_canvas_build_of_the_four_tracks(f110, tracks):
    st = f110.DeviceMap.stack(tracks)
    hs = [m.host for m in tracks]
    Hc, Wc = max(h.height for h in hs), max(h.width for h in hs)
    assert (st.c.height, st.c.width, st.c.num_layers) == (Hc, Wc, 4)
    assert tuple(st.dt.shape) == (4, Hc, Wc) and st.dt_cells is None and st.dt_cells_pad is None
    dt = st.dt.numpy()
    for l, h in enumerate(hs):
        assert np.array_equal(dt[l, :h.height, :h.width], h.dt)
        pad = np.ones((Hc, Wc), bool)
        pad[:h.height, :h.width] = False
        assert np.all(dt[l][pad] == h.dt[-1, -1])
        assert dt[l, -1, -1] == h.dt[-1, -1]
        assert list(st.layer_geom_host[l]) == [h.orig_x, h.orig_y, h.width * h.resolution, h.height * h.resolution,
                                               h.width, h.height]
    assert st.c.layer_geom == st.layer_geom.data_ptr() and np.array_equal(st.layer_geom.numpy(), st.layer_geom_host)
    assert st.c.layer_orig_max == max(max(abs(h.orig_x), abs(h.orig_y)) for h in hs)
    assert st.c.dt == st.dt.data_ptr() and not st.c.dt_codes and not st.c.dt_codes_pad
    assert st.c.dt_min_positive == min(m.c.dt_min_positive for m in tracks)


def test_canvas_build_cell_units(f110):
    em = f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', CPU)
    layers = [em, cropped(f110, em, 100, 300, 900, 1100), cropped(f110, em, 450, 40, 1150, 700)]
    st = f110.DeviceMap.stack(layers)
    Hc, Wc = 1600, 1600
    assert (st.c.height, st.c.width, st.c.fast_path) == (Hc, Wc, 1)
    pad, cells = st.dt_cells_pad.numpy(), st.dt_cells.numpy()
    assert pad.shape == (3, Hc + 1, Wc + 1) and cells.shape == (3, Hc, Wc)
    for l, m in enumerate(layers):
        h = m.host
        c = h.dt / h.resolution
        assert np.array_equal(pad[l, :h.height, :h.width], c) and np.array_equal(cells[l, :h.height, :h.width], c)
        mask = np.ones((Hc + 1, Wc + 1), bool)
        mask[:h.height, :h.width] = False
        assert np.all(pad[l][mask] == c[-1, -1])


def test_same_shape_stack_keeps_todays_struct(f110, tracks):
    b = tracks[0]
    flipped = f110.DeviceMap(f110.maps.HostMap(np.ascontiguousarray(b.host.dt[::-1, ::-1]), 0.05,
                                               (b.host.orig_x, b.host.orig_y, 0.0)), CPU)
    st = f110.DeviceMap.stack([b, flipped])
    assert not st.c.layer_geom and st.c.layer_orig_max == 0.0 and not hasattr(st, 'layer_geom_host')
    assert (st.c.height, st.c.width, st.c.num_layers) == (b.host.height, b.host.width, 2)
    assert tuple(st.dt.shape) == (2, b.host.height, b.host.width)
    ref = type(b.c).from_buffer_copy(b.c)
    for f, _ in ref._fields_:
        if f not in ('dt', 'dt_cells', 'dt_cells_pad', 'dt_codes', 'dt_lut', 'dt_codes_pad', 'num_layers', 'dt_min_positive'):
            assert getattr(st.c, f) == getattr(ref, f), f


def test_stack_rejects_what_the_canvas_cannot_hold(f110, tracks):
    em = f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', CPU)
    stata = f110.DeviceMap.from_yaml(os.path.join(MAPS, 'stata_basement.yaml'), '.png', CPU)
    with pytest.raises(ValueError):
        f110.DeviceMap.stack([tracks[0], em])
    with pytest.raises(ValueError):
        f110.DeviceMap.stack([tracks[0], stata])
    h = tracks[2].host
    rot = f110.DeviceMap(f110.maps.HostMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.2)), CPU)
    with pytest.raises(ValueError):
        f110.DeviceMap.stack([tracks[0], rot])


# ----------------------------------------------------------------------------- host model of the lookup
def oracle_lookup(h, x, y):
    """oracle/f110_oracle.c dt_lookup (reference xy_2_rc + distance_transform, unrotated), vectorised."""
    tx, ty = x - h.orig_x, y - h.orig_y
    inb = ~((tx < 0) | (tx >= h.width * h.resolution) | (ty < 0) | (ty >= h.height * h.resolution))
    with np.errstate(invalid='ignore'):
        cc = np.where(inb, tx / h.resolution, 0).astype(np.int64)
        rr = np.where(inb, ty / h.resolution, 0).astype(np.int64)
    ok = inb & (cc < h.width) & (rr < h.height)
    return np.where(ok, h.dt[np.where(ok, rr, 0), np.where(ok, cc, 0)], h.dt[-1, -1])


def u32(v):
    """(unsigned) of the int32 the kernel takes from the low word of the magic add."""
    return np.asarray(v, dtype=np.int64) & 0xFFFFFFFF


def het_lookup_metres(canvas, geom, Hc, Wc, res, x, y, x_max=None):
    """k_march_lean_het, metre loop: tx = X - orig_l; c = floor(RN(tx / res)) (the FMA-corrected quotient equals the IEEE
    division: test_boundary_inputs); idx = r * Wc + c unless c >= Wc, r >= Hc, tx >= x_max_l or ty >= y_max_l (-> last)."""
    tx, ty = x - geom[0], y - geom[1]
    c, r = u32(np.floor(tx / res)), u32(np.floor(ty / res))
    xm = geom[2] if x_max is None else x_max
    off = (c >= Wc) | (r >= Hc) | (tx >= xm) | (ty >= geom[3])
    idx = np.where(off, Hc * Wc - 1, r * Wc + np.where(off, 0, c))
    return canvas.reshape(-1)[idx]


def het_lookup_cells(pad, geom, Hc, Wc, res, x, y):
    """k_march_lean_het, cell loop (k_dynamics' first lookup is the same index on the unpadded canvas): X = x / res,
    c = floor(X - orig_x / res), value = pad[min(r, Hc)][min(c, Wc)] (unsigned min)."""
    inv = 1.0 / res
    c = u32(np.floor(x * inv - geom[0] * inv))
    r = u32(np.floor(y * inv - geom[1] * inv))
    return pad[np.minimum(r, Hc), np.minimum(c, Wc)] * res


def probe_points(h, rng, n):
    """>= n coordinates around one layer: uniform over (and well beyond) the map, the 8-ulp cell-edge builder on both axes,
    the far-edge builder just below / at W*res and H*res, negative and far-off coordinates."""
    res = h.resolution
    W, H = h.width * res, h.height * res
    xs = [rng.uniform(-0.2 * W, 1.2 * W, n), rng.uniform(-1e4, 1e4, 200)]
    ys = [rng.uniform(-0.2 * H, 1.2 * H, n), rng.uniform(-1e4, 1e4, 200)]
    t, _ = bi.cell_boundary_points(res, max(2, min(h.width, h.height)), 2000, rng)
    xs.append(t); ys.append(rng.permutation(t))
    for Lc, other in ((h.width, H), (h.height, W)):
        e = np.concatenate([bi.far_edge_points(Lc, res)[0], [Lc * res, math.nextafter(Lc * res, 1e9), -0.0,
                                                             math.nextafter(0.0, -1.0)]])
        o = rng.uniform(0, other, e.size)
        if Lc == h.width:
            xs.append(e); ys.append(o)
        else:
            xs.append(o); ys.append(e)
    x, y = np.concatenate(xs), np.concatenate(ys)
    return x + h.orig_x, y + h.orig_y


def lowered_width(res, lo=100, hi=3000):
    """A width whose fp64 extent fl(W * res) divides back below W: a coordinate there passes `floor(RN(t / res)) < W` yet fails
    `t < fl(W * res)`, so only the layer's own x_max gives the reference's answer."""
    return next(W for W in range(lo, hi) if math.floor((W * res) / res) < W)


def test_het_lookup_model_metres(f110, tracks):
    res = 0.05
    affected = bi.far_edge_sizes(res, 100, 3000)[0]
    low = lowered_width(res)
    layers = list(tracks) + [synthetic(f110, 420, affected, res, (-3.3, 2.1, 0.0), 1),
                             # origin 0: the edge coordinates survive `x - orig` unrounded
                             synthetic(f110, 300, low, res, (0.0, 0.0, 0.0), 2)]
    st = f110.DeviceMap.stack(layers)
    Hc, Wc = st.c.height, st.c.width
    canvas = st.dt.numpy()
    rng = np.random.default_rng(5)
    told_apart = 0
    for l, m in enumerate(layers):
        h = m.host
        x, y = probe_points(h, rng, 100000)
        assert x.size >= 100000
        want = oracle_lookup(h, x, y)
        got = het_lookup_metres(canvas[l], st.layer_geom_host[l], Hc, Wc, res, x, y)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (l, x[bad[:3]] - h.orig_x, y[bad[:3]] - h.orig_y)
        canvas_xmax = het_lookup_metres(canvas[l], st.layer_geom_host[l], Hc, Wc, res, x, y, x_max=Wc * res)
        told_apart += int((canvas_xmax != want).sum())
    assert told_apart > 0


def test_het_lookup_model_cells(f110):
    em = f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', CPU)
    layers = [em, cropped(f110, em, 100, 300, 900, 1100), cropped(f110, em, 450, 40, 1150, 700)]
    st = f110.DeviceMap.stack(layers)
    Hc, Wc = st.c.height, st.c.width
    pad = st.dt_cells_pad.numpy()
    rng = np.random.default_rng(6)
    for l, m in enumerate(layers):
        h = m.host
        x, y = probe_points(h, rng, 100000)
        want = oracle_lookup(h, x, y)
        got = het_lookup_cells(pad[l], st.layer_geom_host[l], Hc, Wc, h.resolution, x, y)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (l, x[bad[:3]], y[bad[:3]])


# ----------------------------------------------------------------------------- resource budget
# k_march_lean_het<NOISE, COUNT, CELLS, PT, MINB> -> (registers, stack bytes), DESIGN.md §3.2
HET_BUDGET = {(0, 0, 1): (32, 80), (1, 0, 1): (32, 80), (0, 1, 1): (32, 88),
              (0, 0, 0): (32, 88), (1, 0, 0): (32, 96), (0, 1, 0): (32, 96)}


def test_het_kernel_resource_budget():
    import shutil
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    lib_path = os.path.join(os.path.dirname(os.path.abspath(nat.__file__)), 'libf110_b200.so')
    out = subprocess.run([tool, '-res-usage', lib_path], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    b = lambda v: 'Lb1E' if v else 'Lb0E'  # noqa: E731
    for (noise, count, cells), want in HET_BUDGET.items():
        for pt, minb in ((512, 4), (1024, 2)):
            name = '_ZN4f11016k_march_lean_hetI%s%s%sLi%dELi%dEEEvNS_5LeanKENS_10LayerGeomKENS_10MarchQueueE' % (
                b(noise), b(count), b(cells), pt, minb)
            assert usage.get(name) == want, (name, usage.get(name))
