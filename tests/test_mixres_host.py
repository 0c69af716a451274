"""Canvas stacks of maps that also differ in resolution (DeviceMap.stack(maps, mixed_resolution=True) -> f110_map.layer_res),
on the CPU.

  * the canvas build of the six bundled maps: the metre canvas only, layer_res rows (res_l, 1 / res_l) and their host
    copies, x_max / y_max at each layer's own resolution; one shared resolution gives today's stack field for field;
    rotated origins still raise ValueError;
  * the numpy restatement of k_march_lean_het's metre lookup (test_multimap_host.het_lookup_metres), with the layer's own
    res_l, against the oracle's per-layer lookup at >= 1e5 coordinates per layer; with another layer's resolution it must
    disagree;
  * the register and stack budget of k_march_lean_het_res (DESIGN.md §3.2).
"""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import boundary_inputs as bi
from test_multimap_host import MAPS, TRACKS, het_lookup_metres, oracle_lookup, probe_points, synthetic

CPU = torch.device('cpu')
SIX = TRACKS + [('stata_basement', '.png'), ('example_map', '.png')]


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def six(f110):
    return [f110.DeviceMap.from_yaml(os.path.join(MAPS, n + '.yaml'), e, CPU) for n, e in SIX]


# ----------------------------------------------------------------------------- canvas build
def test_canvas_build_of_the_six_bundled_maps(f110, six):
    with pytest.raises(ValueError):
        f110.DeviceMap.stack(six)                                   # still opt-in
    st = f110.DeviceMap.stack(six, mixed_resolution=True)
    hs = [m.host for m in six]
    assert sorted({h.resolution for h in hs}) == [0.05, 0.0504, 0.0625]
    Hc, Wc = max(h.height for h in hs), max(h.width for h in hs)
    assert (st.c.height, st.c.width, st.c.num_layers, st.c.fast_path) == (Hc, Wc, 6, 0)
    assert tuple(st.dt.shape) == (6, Hc, Wc)
    assert st.dt_cells is None and st.dt_cells_pad is None and st.dt_codes is None and st.dt_lut is None
    assert not st.c.dt_cells and not st.c.dt_cells_pad and not st.c.dt_codes and not st.c.dt_codes_pad and not st.c.dt_lut
    assert st.c.codes_pitch == 0
    dt = st.dt.numpy()
    for l, h in enumerate(hs):
        assert np.array_equal(dt[l, :h.height, :h.width], h.dt)
        pad = np.ones((Hc, Wc), bool)
        pad[:h.height, :h.width] = False
        assert np.all(dt[l][pad] == h.dt[-1, -1])
        assert dt[l, -1, -1] == h.dt[-1, -1]
        assert list(st.layer_geom_host[l]) == [h.orig_x, h.orig_y, h.width * h.resolution, h.height * h.resolution,
                                               h.width, h.height]
        assert list(st.layer_res_host[l]) == [h.resolution, 1.0 / h.resolution]
    assert st.c.layer_res == st.layer_res.data_ptr() and np.array_equal(st.layer_res.numpy(), st.layer_res_host)
    assert (st.c.layer_res_min, st.c.layer_res_max) == (0.05, 0.0625)
    assert st.c.layer_geom == st.layer_geom.data_ptr() and np.array_equal(st.layer_geom.numpy(), st.layer_geom_host)
    assert st.c.layer_orig_max == max(max(abs(h.orig_x), abs(h.orig_y)) for h in hs)
    assert st.c.dt == st.dt.data_ptr()
    assert st.c.dt_min_positive == min(m.c.dt_min_positive for m in six)
    assert st.c.resolution == hs[0].resolution


def _same_struct(a, b):
    """Every f110_map field equal, the device pointers through the tables they point at."""
    tables = ('dt', 'dt_cells', 'dt_cells_pad', 'layer_geom', 'layer_res')
    for f, _ in type(a.c)._fields_:
        if f in tables:
            assert bool(getattr(a.c, f)) == bool(getattr(b.c, f)), f
        elif f not in ('sines', 'cosines', 'sincos', 'sincos2'):
            assert getattr(a.c, f) == getattr(b.c, f), f
    for t in tables + ('dt_codes', 'dt_lut', 'dt_codes_pad'):
        x, y = getattr(a, t, None), getattr(b, t, None)
        assert (x is None) == (y is None), t
        if x is not None:
            assert torch.equal(x, y), t
    for t in ('layer_geom_host', 'layer_res_host'):
        assert hasattr(a, t) == hasattr(b, t), t
        if hasattr(a, t):
            assert np.array_equal(getattr(a, t), getattr(b, t)), t


def test_one_resolution_ignores_the_flag(f110, six):
    tracks = six[:4]
    _same_struct(f110.DeviceMap.stack(tracks, mixed_resolution=True), f110.DeviceMap.stack(tracks))
    # same shape too (the layered [L][H][W] stack), and cell units
    em = six[5]
    _same_struct(f110.DeviceMap.stack([em, em], mixed_resolution=True), f110.DeviceMap.stack([em, em]))
    assert not f110.DeviceMap.stack(tracks, mixed_resolution=True).c.layer_res


def test_rotated_layers_still_raise(f110, six):
    h = six[4].host
    rot = f110.DeviceMap(f110.maps.HostMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.2)), CPU)
    for flag in (False, True):
        with pytest.raises(ValueError):
            f110.DeviceMap.stack([six[0], rot], mixed_resolution=flag)
        with pytest.raises(ValueError):
            f110.DeviceMap.stack([six[5], rot], mixed_resolution=flag)


# ----------------------------------------------------------------------------- host model of the lookup
def test_het_res_lookup_model(f110, six):
    """floor(tx / res_l) on the canvas with each layer's own extent: equal to the oracle on every layer (six bundled maps, a
    0.0504 m layer of a far-edge-affected width, a 0.0625 m layer of a generated track's size); with another layer's
    resolution in place of res_l it disagrees."""
    affected = bi.far_edge_sizes(0.0504, 100, 3000)[0]
    layers = list(six) + [synthetic(f110, 420, affected, 0.0504, (-3.3, 2.1, 0.0), 3),
                          synthetic(f110, 1600, 1600, 0.0625, (-40.0, -50.0, 0.0), 4)]
    st = f110.DeviceMap.stack(layers, mixed_resolution=True)
    Hc, Wc = st.c.height, st.c.width
    canvas = st.dt.numpy()
    rng = np.random.default_rng(7)
    told_apart = 0
    for l, m in enumerate(layers):
        h = m.host
        res_l = st.layer_res_host[l, 0]
        x, y = probe_points(h, rng, 100000)
        assert x.size >= 100000
        want = oracle_lookup(h, x, y)
        got = het_lookup_metres(canvas[l], st.layer_geom_host[l], Hc, Wc, res_l, x, y)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (l, x[bad[:3]] - h.orig_x, y[bad[:3]] - h.orig_y)
        other = next(r for r in st.layer_res_host[:, 0] if r != res_l)
        wrong = het_lookup_metres(canvas[l], st.layer_geom_host[l], Hc, Wc, other, x, y)
        told_apart += int((wrong != want).sum())
        if res_l != st.c.resolution:
            told_apart += int((het_lookup_metres(canvas[l], st.layer_geom_host[l], Hc, Wc, st.c.resolution, x, y) != want).sum())
    assert told_apart > 0


# ----------------------------------------------------------------------------- resource budget
# k_march_lean_het_res<NOISE, COUNT, PT, MINB> -> (registers, stack bytes), DESIGN.md §3.2
HET_RES_BUDGET = {(0, 0): (32, 96), (1, 0): (32, 112), (0, 1): (32, 96)}


def test_het_res_kernel_resource_budget():
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
    for (noise, count), want in HET_RES_BUDGET.items():
        for pt, minb in ((512, 4), (1024, 2)):
            name = '_ZN4f11020k_march_lean_het_resI%s%sLi%dELi%dEEEvNS_5LeanKENS_10LayerGeomKEPKdNS_10MarchQueueE' % (
                b(noise), b(count), pt, minb)
            assert usage.get(name) == want, (name, usage.get(name))
