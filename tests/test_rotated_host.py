"""Maps whose yaml origin has a yaw (HostMap(dt, res, (ox, oy, yaw))): the canvas stack DeviceMap.stack(maps,
rotated_origins=True) -> f110_map.layer_rot, and the lookup of k_march_lean_rot (csrc/march_rot.cuh), on the CPU.

  * the canvas build of rotated berlin, vegas, rotated example_map and a rotated generated track: the metre canvas, layer_res
    for every layer, layer_rot rows (orig_c, orig_s) as HostMap computed them and their pointers; without a rotated layer the
    flag changes nothing; the ValueError cases, the same-geometry rotated stack without the flag included;
  * a numpy restatement of the new kernel's lookup (rotation without FMA, the FMA-corrected quotient, canvas clamps, the
    layer's own extent) against the oracle's xy_2_rc / distance_transform (oracle/f110_oracle.c dt_lookup, read through
    orc_get_scan with eps and max_range out of reach, so that every beam returns the first lookup) at >= 1e5 points per
    layer, with builders for the rotated frame: x_rot or y_rot within 8 ulps of a cell edge, just below W*res or H*res, tiny
    negative or -0.0; every builder is checked to land in its band.  Without the rotation, or with another layer's (c, s),
    the model disagrees;
  * the register and stack budget of k_march_lean_rot (DESIGN.md §3.2).
"""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import boundary_inputs as bi
from test_mixres_host import _same_struct
from test_multimap_host import MAPS, TRACKS, u32

CPU = torch.device('cpu')
# layer -> origin yaw: a yaw in each quadrant but the first's mirror, so that the origin itself gives x_rot = -0.0 (c < 0,
# s < 0) on one layer and y_rot = -0.0 (c < 0, s > 0) on another
YAWS = {'berlin': 0.35, 'example_map': 1.9, 'generated': -2.0}


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


def rotated(f110, dmap, yaw):
    h = dmap.host
    return f110.DeviceMap(f110.maps.HostMap(h.dt, h.resolution, (h.orig_x, h.orig_y, yaw)), CPU)


def generated_host(f110, seed=3):
    """A generated track (0.0625 m) rasterised and distance-transformed on the host, as trackgen.device_map does on the
    device (test_trackgen.raster_numpy is the rasteriser's arithmetic in numpy)."""
    from scipy.ndimage import distance_transform_edt as edt
    from f1tenth_gym_b200 import trackgen as tg
    from test_trackgen import raster_numpy
    t = tg.random_tracks(seed, 1)[0]
    lo, hi = t.wall_band()
    occ, _ = raster_numpy(t, t.canvas, t.canvas, lo, hi)
    return f110.maps.HostMap(t.resolution * edt((occ == 0).astype(np.float64)), t.resolution, t.origin)


@pytest.fixture(scope='module')
def plain(f110):
    """berlin, vegas, example_map and a generated track, unrotated."""
    names = [TRACKS[0], TRACKS[1], ('example_map', '.png')]
    out = [f110.DeviceMap.from_yaml(os.path.join(MAPS, n + '.yaml'), e, CPU) for n, e in names]
    return out + [f110.DeviceMap(generated_host(f110), CPU)]


@pytest.fixture(scope='module')
def layers(f110, plain):
    """rotated berlin, vegas, rotated example_map, rotated generated track."""
    b, v, em, g = plain
    return [rotated(f110, b, YAWS['berlin']), v, rotated(f110, em, YAWS['example_map']), rotated(f110, g, YAWS['generated'])]


# ----------------------------------------------------------------------------- canvas build
def test_canvas_build(f110, layers):
    st = f110.DeviceMap.stack(layers, mixed_resolution=True, rotated_origins=True)
    hs = [m.host for m in layers]
    assert sorted({h.resolution for h in hs}) == [0.05, 0.0625]
    Hc, Wc = max(h.height for h in hs), max(h.width for h in hs)
    assert (st.c.height, st.c.width, st.c.num_layers, st.c.fast_path) == (Hc, Wc, 4, 0)
    assert st.dt_cells is None and st.dt_cells_pad is None and st.dt_codes is None and st.dt_lut is None
    assert not st.c.dt_cells and not st.c.dt_cells_pad and not st.c.dt_codes and not st.c.dt_codes_pad and not st.c.dt_lut
    dt = st.dt.numpy()
    for l, h in enumerate(hs):
        assert np.array_equal(dt[l, :h.height, :h.width], h.dt)
        pad = np.ones((Hc, Wc), bool)
        pad[:h.height, :h.width] = False
        assert np.all(dt[l][pad] == h.dt[-1, -1])
        assert list(st.layer_geom_host[l]) == [h.orig_x, h.orig_y, h.width * h.resolution, h.height * h.resolution,
                                               h.width, h.height]
        assert list(st.layer_res_host[l]) == [h.resolution, 1.0 / h.resolution]
        assert list(st.layer_rot_host[l]) == [h.orig_c, h.orig_s]
    assert [tuple(r) for r in st.layer_rot_host[[0, 2, 3]]] == [(math.cos(y), math.sin(y)) for y in
                                                               (YAWS['berlin'], YAWS['example_map'], YAWS['generated'])]
    assert tuple(st.layer_rot_host[1]) == (1.0, 0.0)
    for t in ('layer_geom', 'layer_res', 'layer_rot'):
        assert getattr(st.c, t) == getattr(st, t).data_ptr() and np.array_equal(getattr(st, t).numpy(), getattr(st, t + '_host'))
    assert (st.c.layer_res_min, st.c.layer_res_max) == (0.05, 0.0625)
    assert st.c.layer_orig_max == max(max(abs(h.orig_x), abs(h.orig_y)) for h in hs)
    assert (st.c.resolution, st.c.orig_x, st.c.orig_c, st.c.orig_s) == (hs[0].resolution, hs[0].orig_x, hs[0].orig_c,
                                                                         hs[0].orig_s)
    assert st.c.dt == st.dt.data_ptr() and st.c.dt_min_positive == min(m.c.dt_min_positive for m in layers)


def test_one_resolution_carries_layer_res(f110, layers):
    """Rotated berlin with vegas (both 0.05 m): no mixed_resolution needed, and layer_res is there all the same."""
    st = f110.DeviceMap.stack(layers[:2], rotated_origins=True)
    assert st.c.layer_res and st.c.layer_rot and st.c.layer_geom and st.c.fast_path == 0
    assert (st.c.layer_res_min, st.c.layer_res_max) == (0.05, 0.05)
    assert np.array_equal(st.layer_res_host, [[0.05, 20.0], [0.05, 20.0]])


def test_same_geometry_rotated_stack(f110, layers):
    """Copies of one rotated map share size, resolution and origin: without the flag that stack used to pass as a plain
    layered stack that f110_step then refused; now it raises, and with the flag it becomes a canvas stack."""
    rb = layers[0]
    with pytest.raises(ValueError):
        f110.DeviceMap.stack([rb, rb])
    st = f110.DeviceMap.stack([rb, rb], rotated_origins=True)
    assert st.c.num_layers == 2 and st.c.layer_geom and st.c.layer_res and st.c.layer_rot
    assert np.array_equal(st.layer_rot_host, [[rb.host.orig_c, rb.host.orig_s]] * 2)


def test_value_errors(f110, layers, plain):
    for ls in (layers, layers[:2], [plain[0], layers[2]]):
        for mixed in (False, True):
            with pytest.raises(ValueError):
                f110.DeviceMap.stack(ls, mixed_resolution=mixed)
    with pytest.raises(ValueError):
        f110.DeviceMap.stack(layers, rotated_origins=True)          # 0.05 and 0.0625 m: also needs mixed_resolution


def test_no_rotated_layer_ignores_the_flag(f110, plain):
    tracks = [f110.DeviceMap.from_yaml(os.path.join(MAPS, n + '.yaml'), e, CPU) for n, e in TRACKS]
    _same_struct(f110.DeviceMap.stack(tracks, rotated_origins=True), f110.DeviceMap.stack(tracks))
    em = plain[2]
    _same_struct(f110.DeviceMap.stack([em, em], rotated_origins=True), f110.DeviceMap.stack([em, em]))
    _same_struct(f110.DeviceMap.stack(plain, mixed_resolution=True, rotated_origins=True),
                 f110.DeviceMap.stack(plain, mixed_resolution=True))
    for st in (f110.DeviceMap.stack(tracks, rotated_origins=True), f110.DeviceMap.stack(plain, mixed_resolution=True,
                                                                                        rotated_origins=True)):
        assert not st.c.layer_rot and not hasattr(st, 'layer_rot_host')


# ----------------------------------------------------------------------------- host model of the lookup
def frame(h, x, y, c=None, s=None):
    """x_rot, y_rot as xy_2_rc and the kernel round them (numpy fp64: every product and sum rounded on its own)."""
    c = h.orig_c if c is None else c
    s = h.orig_s if s is None else s
    tx, ty = x - h.orig_x, y - h.orig_y
    return tx * c + ty * s, -tx * s + ty * c


def rot_lookup(canvas, geom, Hc, Wc, res, rot, x, y):
    """k_march_lean_rot's lookup: (x_rot, y_rot) in the layer's frame; c = floor(RN(x_rot / res_l)) (the FMA-corrected
    quotient, which equals the IEEE division: checked on the band points in test_rot_lookup_model); idx = r * Wc + c unless
    c >= Wc, r >= Hc, x_rot >= x_max_l or y_rot >= y_max_l (-> the slice's last cell)."""
    tx, ty = x - geom[0], y - geom[1]
    xr, yr = tx * rot[0] + ty * rot[1], -tx * rot[1] + ty * rot[0]
    c, r = u32(np.floor(xr / res)), u32(np.floor(yr / res))
    off = (c >= Wc) | (r >= Hc) | (xr >= geom[2]) | (yr >= geom[3])
    idx = np.where(off, Hc * Wc - 1, r * Wc + np.where(off, 0, c))
    return canvas.reshape(-1)[idx]


def oracle_lookup(h, x, y):
    """The oracle's dt_lookup at each point: orc_get_scan with eps = max_range = 1e300 returns the first lookup."""
    import oracle
    om = oracle.OracleMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.0), eps=1e300, max_range=1e300)
    om.c.orig_c, om.c.orig_s = h.orig_c, h.orig_s
    L = oracle.lib()
    fov = 4.7
    inc = oracle.theta_index_increment(2, fov, om.theta_dis)
    pose, scan = np.zeros(3), np.zeros(2)
    pp, sp = pose.ctypes.data_as(C.POINTER(C.c_double)), scan.ctypes.data_as(C.POINTER(C.c_double))
    out = np.empty(x.size)
    for k in range(x.size):
        pose[0], pose[1] = x[k], y[k]
        L.orc_get_scan(C.byref(om.c), pp, 2, fov, inc, sp, None)
        out[k] = scan[0]
    return out


def _ulp(v):
    return np.spacing(np.abs(v))


def world(h, xr, yr, rng, search=4):
    """World points whose x_rot, y_rot (as `frame` rounds them) lie as close as the fp64 grid allows to the targets (xr, yr):
    the exact inverse rotation rounded, then the best of (2 search + 1)^2 neighbours a few ulps away on both axes."""
    tx, ty = h.orig_c * xr - h.orig_s * yr, h.orig_s * xr + h.orig_c * yr
    x0, y0 = tx + h.orig_x, ty + h.orig_y
    best, bx, by = np.full(x0.size, np.inf), x0.copy(), y0.copy()
    steps = np.arange(-search, search + 1)
    for i in steps:
        for j in steps:
            x, y = x0 + i * _ulp(x0), y0 + j * _ulp(y0)
            a, b = frame(h, x, y)
            err = np.abs(a - xr) / _ulp(xr + 1e-300) + np.abs(b - yr) / _ulp(yr + 1e-300)
            take = err < best
            best[take], bx[take], by[take] = err[take], x[take], y[take]
    return bx, by


def edge_ulps(v, res):
    """Distance of v to the nearest cell edge k * res, in ulps of v."""
    return np.abs(v - np.rint(v / res) * res) / _ulp(v)


def rotated_probe_points(h, rng, n):
    """>= n world points around one rotated layer and the band builders; returns (x, y, bands) with bands a dict of index
    arrays, each checked to land in its band."""
    res, W, H = h.resolution, h.width * h.resolution, h.height * h.resolution
    xs, ys, bands = [], [], {}

    def add(name, x, y):
        at = sum(v.size for v in xs)
        xs.append(x); ys.append(y)
        bands[name] = np.arange(at, at + x.size)
    # uniform over (and well beyond) the map in its own frame, and far off
    add('uniform', *world(h, rng.uniform(-0.2 * W, 1.2 * W, n), rng.uniform(-0.2 * H, 1.2 * H, n), rng, search=0))
    add('far', rng.uniform(-1e4, 1e4, 200), rng.uniform(-1e4, 1e4, 200))
    # x_rot (y_rot) within 8 ulps of a cell edge, the other coordinate on the map
    for axis, Lc, other in ((0, h.width, H), (1, h.height, W)):
        t, _ = bi.cell_boundary_points(res, max(2, Lc), 3000, rng)
        o = rng.uniform(0, other, t.size)
        x, y = world(h, t, o, rng) if axis == 0 else world(h, o, t, rng)
        v = frame(h, x, y)[axis]
        keep = (edge_ulps(v, res) <= 8) & (np.rint(v / res) >= 1)
        add('edge_%s' % 'xy'[axis], x[keep], y[keep])
    # just below W * res (H * res): within 32 ulps under the extent, and at it
    for axis, Lc, other in ((0, h.width, H), (1, h.height, W)):
        ext = Lc * res
        t = np.concatenate([bi.far_edge_points(Lc, res, 32)[0], [ext, math.nextafter(ext, 1e9)]])
        t = np.repeat(t, 8)
        o = rng.uniform(0, other, t.size)
        x, y = world(h, t, o, rng) if axis == 0 else world(h, o, t, rng)
        v = frame(h, x, y)[axis]
        keep = (v < ext) & (v >= ext - 32 * _ulp(ext))
        add('below_extent_%s' % 'xy'[axis], x[keep], y[keep])
        keep = (v >= ext) & (v <= ext + 32 * _ulp(ext))
        add('at_extent_%s' % 'xy'[axis], x[keep], y[keep])
    # tiny negative x_rot (y_rot), and -0.0
    for axis, other in ((0, H), (1, W)):
        t = -np.abs(rng.uniform(0, 1e-13, 4000))
        o = rng.uniform(0, other, t.size)
        x, y = world(h, t, o, rng) if axis == 0 else world(h, o, t, rng)
        v = frame(h, x, y)[axis]
        add('tiny_negative_%s' % 'xy'[axis], x[(v < 0) & (v > -1e-12)], y[(v < 0) & (v > -1e-12)])
    cand = np.array([h.orig_x, math.nextafter(h.orig_x, 1e9), math.nextafter(h.orig_x, -1e9)])
    cx, cy = np.meshgrid(cand, np.array([h.orig_y, math.nextafter(h.orig_y, 1e9), math.nextafter(h.orig_y, -1e9)]))
    cx, cy = cx.ravel(), cy.ravel()
    xr, yr = frame(h, cx, cy)
    zero = ((xr == 0) & np.signbit(xr)) | ((yr == 0) & np.signbit(yr))
    add('minus_zero', cx[zero], cy[zero])
    x, y = np.concatenate(xs), np.concatenate(ys)
    # every builder lands in its band
    xr, yr = frame(h, x, y)
    for axis, v in ((0, xr), (1, yr)):
        a = 'xy'[axis]
        e = bands['edge_' + a]
        assert e.size >= 500 and np.all(edge_ulps(v[e], res) <= 8), (a, e.size)
        ext = (h.width if axis == 0 else h.height) * res
        b = bands['below_extent_' + a]
        assert b.size >= 16 and np.all((v[b] < ext) & (v[b] >= ext - 32 * _ulp(ext))), (a, b.size)
        b = bands['at_extent_' + a]
        assert np.all(v[b] >= ext)
        b = bands['tiny_negative_' + a]
        assert b.size >= 100 and np.all((v[b] < 0) & (v[b] > -1e-12)), (a, b.size)
    z = bands['minus_zero']
    assert np.all(((xr[z] == 0) & np.signbit(xr[z])) | ((yr[z] == 0) & np.signbit(yr[z])))
    return x, y, bands


def test_rot_lookup_model(f110, layers):
    """The model equals the oracle on every layer (>= 1e5 points each, band builders included); the FMA-corrected
    quotient equals the IEEE division on the band points; without the rotation, or with another rotated layer's (c, s), the
    model disagrees."""
    st = f110.DeviceMap.stack(layers, mixed_resolution=True, rotated_origins=True)
    Hc, Wc = st.c.height, st.c.width
    canvas = st.dt.numpy()
    rng = np.random.default_rng(11)
    minus_zero = {'x': 0, 'y': 0}
    for l, m in enumerate(layers):
        h = m.host
        res, rot = st.layer_res_host[l, 0], st.layer_rot_host[l]
        x, y, bands = rotated_probe_points(h, rng, 100000)
        assert x.size >= 100000
        want = oracle_lookup(h, x, y)
        got = rot_lookup(canvas[l], st.layer_geom_host[l], Hc, Wc, res, rot, x, y)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (l, x[bad[:3]], y[bad[:3]], got[bad[:3]], want[bad[:3]])
        xr, yr = frame(h, x, y)
        z = bands['minus_zero']
        minus_zero['x'] += int(((xr[z] == 0) & np.signbit(xr[z])).sum())
        minus_zero['y'] += int(((yr[z] == 0) & np.signbit(yr[z])).sum())
        # the kernel's quotient on the band points (exact rational FMA, boundary_inputs.fma_quotient)
        for name in ('edge_x', 'below_extent_x', 'at_extent_x', 'tiny_negative_x', 'edge_y', 'below_extent_y',
                     'at_extent_y', 'tiny_negative_y'):
            v = (xr if name.endswith('x') else yr)[bands[name]]
            for t in v[:300]:
                assert bi.fma_quotient(float(t), res) == t / res, (l, name, t)
        if rot[1] != 0.0:
            dropped = rot_lookup(canvas[l], st.layer_geom_host[l], Hc, Wc, res, (1.0, 0.0), x, y)
            assert (dropped != want).sum() > 0, l
            for k in range(len(layers)):
                if k != l and st.layer_rot_host[k, 1] != 0.0:
                    other = rot_lookup(canvas[l], st.layer_geom_host[l], Hc, Wc, res, st.layer_rot_host[k], x, y)
                    assert (other != want).sum() > 0, (l, k)
    assert minus_zero['x'] > 0 and minus_zero['y'] > 0, minus_zero


# ----------------------------------------------------------------------------- resource budget
# k_march_lean_rot<NOISE, COUNT, PT, MINB> -> (registers, stack bytes), DESIGN.md §3.2
ROT_BUDGET = {(0, 0): (32, 96), (1, 0): (32, 96), (0, 1): (32, 96)}


def test_rot_kernel_resource_budget():
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
    for (noise, count), want in ROT_BUDGET.items():
        for pt, minb in ((512, 4), (1024, 2)):
            name = '_ZN4f11016k_march_lean_rotI%s%sLi%dELi%dEEEvNS_5LeanKENS_8RotGeomKENS_10MarchQueueE' % (
                b(noise), b(count), pt, minb)
            assert usage.get(name) == want, (name, usage.get(name))
