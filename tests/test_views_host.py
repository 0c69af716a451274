"""f110_render_views on the CPU: the export, the header declaration and the unchanged ABI version, every argument combination
it must refuse before anything is enqueued, the Python-side ValueErrors, the register and stack budget of k_render_views
(DESIGN.md §3.6), and a numpy model of the pixel rule (csrc/render.cuh) whose map lookup is checked against the oracle.

The oracle check reads the oracle's xy_2_rc through orc_get_scan on a table that holds each cell's flat index (eps and
max_range out of reach, so that a beam returns its first lookup): an in-map point returns its cell's index and an off-map
point the last cell's, which is what the reference reads there (numba wraps (-1, -1)).  The model's cell must equal the
oracle's index, and every point the model puts off the map must read the last cell.  That reading cannot tell an off-map point
from the layer's top-right cell, so test_top_right_cell_against_the_oracle adds the oracle on a map with one more row and
column (where that cell is not the last one) and the extent tests on the row and column next to it.
tests/test_gpu_views.py compares the kernel with this model byte for byte.
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

import boundary_inputs as bi
from test_multimap_host import MAPS, TRACKS
from test_rotated_host import generated_host, rotated_probe_points

CPU = torch.device('cpu')
INVALID, NO_MAP = -1, -2
SIX = TRACKS + [('stata_basement', '.png'), ('example_map', '.png')]


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


def load(f110, name, ext, device=CPU):
    return f110.DeviceMap.from_yaml(os.path.join(MAPS, name + '.yaml'), ext, device)


# ----------------------------------------------------------------------------- the pixel rule, restated
def pixel_centres(x, y, cs, sn, H, W, s, f, heading_up):
    """World coordinates (H, W) of a view's pixel centres, in the kernel's operation order (numpy fp64: every product and sum
    rounded on its own, as the kernel without FMA contraction)."""
    x, y, cs, sn, s, f = (np.float64(v) for v in (x, y, cs, sn, s, f))
    cx, cy = x + f * cs, y + f * sn
    h = s * np.float64(0.5)
    u = (2 * np.arange(W) + 1 - W).astype(np.float64) * h
    v = (H - 2 * np.arange(H) - 1).astype(np.float64) * h
    U, V = np.broadcast_to(u[None, :], (H, W)), np.broadcast_to(v[:, None], (H, W))
    if heading_up:
        return cx + (U * sn + V * cs), cy + (V * sn - U * cs)
    return cx + U, cy + V


def map_cells(px, py, geom, res, rot):
    """xy_2_rc on one layer: (row, col, on).  geom = (orig_x, orig_y, x_max, y_max, W_l, H_l), rot = (c, s)."""
    with np.errstate(invalid='ignore', over='ignore'):
        tx, ty = px - geom[0], py - geom[1]
        xr = tx * rot[0] + ty * rot[1]
        yr = (-tx) * rot[1] + ty * rot[0]
        on = (xr >= 0) & (xr < geom[2]) & (yr >= 0) & (yr < geom[3])
        col = np.where(on, np.floor(np.where(on, xr, 0.0) / res), 0.0)
        row = np.where(on, np.floor(np.where(on, yr, 0.0) / res), 0.0)
    on &= (col < geom[4]) & (row < geom[5])
    return np.where(on, row, 0).astype(np.int64), np.where(on, col, 0).astype(np.int64), on


def in_car(px, py, v):
    """The bounding-box-guarded edge test of a car quad v (4, 2) (rl, rr, fr, fl) at the pixel centres."""
    with np.errstate(invalid='ignore', over='ignore'):
        inside = (px >= v[:, 0].min()) & (px <= v[:, 0].max()) & (py >= v[:, 1].min()) & (py <= v[:, 1].max())
        for e in range(4):
            a, b = v[e], v[(e + 1) % 4]
            ex, ey = b[0] - a[0], b[1] - a[1]
            inside &= (ex * (py - a[1]) - ey * (px - a[0])) >= 0
    return inside


def layer_tables(dmap):
    """(per-layer geometry rows, per-layer resolution, per-layer rotation, dt [L][Hc][Wc]) of any DeviceMap, as the kernel
    reads them: layer_geom / layer_res / layer_rot, or the struct's values."""
    c = dmap.c
    L = max(1, int(c.num_layers))
    dt = dmap.dt.cpu().numpy().reshape(L, c.height, c.width)
    if c.layer_geom:
        geom = dmap.layer_geom_host
        res = dmap.layer_res_host[:, 0] if c.layer_res else np.full(L, c.resolution)
        rot = dmap.layer_rot_host if c.layer_rot else np.tile([c.orig_c, c.orig_s], (L, 1))
    else:
        geom = np.tile([c.orig_x, c.orig_y, c.width * c.resolution, c.height * c.resolution, c.width, c.height], (L, 1))
        res, rot = np.full(L, c.resolution), np.tile([c.orig_c, c.orig_s], (L, 1))
    return geom, res, rot, dt


def views_model(tables, state, cos_sin, verts, env_layer, A, agent_ids, H, W, s, f, heading_up):
    """uint8 (V, H, W): the kernel's classes.  state (7, N*A) fp64, cos_sin (N*A, 2) the device's (cos, sin) of state[4],
    verts (N*A, 4, 2) from f110_get_vertices, env_layer (N,) or None."""
    geom, res, rot, dt = tables
    NA = state.shape[1]
    out = np.empty((len(agent_ids), H, W), np.uint8)
    fin = np.isfinite(state[0]) & np.isfinite(state[1]) & np.isfinite(state[4])
    for k, a in enumerate(agent_ids):
        a = int(a)
        l = int(env_layer[a // A]) if (env_layer is not None and 0 <= a < NA) else 0
        if not (0 <= a < NA) or not fin[a] or not (0 <= l < dt.shape[0]):
            out[k] = 255
            continue
        px, py = pixel_centres(state[0, a], state[1, a], cos_sin[a, 0], cos_sin[a, 1], H, W, s, f, heading_up)
        row, col, on = map_cells(px, py, geom[l], res[l], rot[l])
        cls = np.where(on, np.where(dt[l][row, col] == 0, 2, 1), 0).astype(np.uint8)
        env = a // A
        other = np.zeros((H, W), bool)
        for j in range(env * A, env * A + A):
            if j != a and fin[j]:
                other |= in_car(px, py, verts[j])
        cls[other] = 3
        cls[in_car(px, py, verts[a])] = 4
        out[k] = cls
    return out


# ----------------------------------------------------------------------------- the lookup against the oracle
def oracle_cells(h, x, y):
    """The oracle's xy_2_rc at each point, as a flat index into the layer's own [H][W] table (off-map: the last cell)."""
    import oracle
    idx = np.arange(h.height * h.width, dtype=np.float64).reshape(h.height, h.width)
    om = oracle.OracleMap(idx, h.resolution, (h.orig_x, h.orig_y, 0.0), eps=1e300, max_range=1e300)
    om.c.orig_c, om.c.orig_s = h.orig_c, h.orig_s
    L = oracle.lib()
    inc = oracle.theta_index_increment(2, 4.7, om.theta_dis)
    pose, scan = np.zeros(3), np.zeros(2)
    pp, sp = pose.ctypes.data_as(C.POINTER(C.c_double)), scan.ctypes.data_as(C.POINTER(C.c_double))
    out = np.empty(x.size, np.int64)
    for k in range(x.size):
        pose[0], pose[1] = x[k], y[k]
        L.orc_get_scan(C.byref(om.c), pp, 2, 4.7, inc, sp, None)
        out[k] = int(scan[0])
    return out


def model_flat(h, geom, res, rot, x, y):
    """The model's cell as a flat index into the layer's own table, -1 off the map."""
    row, col, on = map_cells(x, y, geom, res, rot)
    return np.where(on, row * h.width + col, -1)


def agrees(h, got, want):
    last = h.height * h.width - 1
    return np.where(got >= 0, got == want, want == last)


@pytest.fixture(scope='module')
def lookup_cases(f110):
    """name -> (stacked or single DeviceMap, [the HostMap of each layer])."""
    six = [load(f110, n, e) for n, e in SIX]
    b = six[0].host
    rot_berlin = f110.DeviceMap(f110.maps.HostMap(b.dt, b.resolution, (b.orig_x, b.orig_y, 0.35)), CPU)
    gen = f110.DeviceMap(generated_host(f110), CPU)
    cases = {n: (m, [m.host]) for (n, _), m in zip(SIX, six)}
    cases['rot_berlin'] = (rot_berlin, [rot_berlin.host])
    cases['trackgen'] = (gen, [gen.host])
    cases['canvas4'] = (f110.DeviceMap.stack(six[:4]), [m.host for m in six[:4]])
    rl = []
    for m, yaw in zip(six[:4], (0.35, -0.8, 1.9, 3.0)):
        h = m.host
        rl.append(f110.DeviceMap(f110.maps.HostMap(h.dt, h.resolution, (h.orig_x, h.orig_y, yaw)), CPU))
    cases['rot4'] = (f110.DeviceMap.stack(rl, rotated_origins=True), [m.host for m in rl])
    return cases


@pytest.mark.parametrize('case', ['berlin', 'vegas', 'skirk', 'levine', 'stata_basement', 'example_map', 'rot_berlin',
                                  'trackgen', 'canvas4', 'rot4'])
def test_lookup_model_against_the_oracle(f110, lookup_cases, case):
    """>= 1e5 points per layer, with the cell-edge, just-below-extent, tiny-negative and -0.0 builders (each checked to land
    in its band by rotated_probe_points): the model's cell equals the oracle's.  With another layer's geometry, or with the
    canvas extents in place of the layer's, the model disagrees."""
    dmap, hosts = lookup_cases[case]
    geom, res, rot, _ = layer_tables(dmap)
    rng = np.random.default_rng(sum(map(ord, case)))
    for l, h in enumerate(hosts):
        x, y, bands = rotated_probe_points(h, rng, 100000)
        assert x.size >= 100000
        want = oracle_cells(h, x, y)
        got = model_flat(h, geom[l], res[l], rot[l], x, y)
        ok = agrees(h, got, want)
        bad = np.flatnonzero(~ok)
        assert bad.size == 0, (case, l, x[bad[:3]], y[bad[:3]], got[bad[:3]], want[bad[:3]])
        assert (got >= 0).sum() > 1000 and (got < 0).sum() > 1000
        if len(hosts) > 1:
            k = (l + 1) % len(hosts)
            other = model_flat(h, geom[k], res[k], rot[k], x, y)
            assert (~agrees(h, other, want)).sum() > 0, (case, l, k)
            c = dmap.c
            wide = np.array(geom[l], dtype=np.float64)
            wide[2], wide[3] = c.width * res[l], c.height * res[l]
            wide[4], wide[5] = c.width, c.height
            canvas = model_flat(h, wide, res[l], rot[l], x, y)
            assert (~agrees(h, canvas, want)).sum() > 0 or (h.width, h.height) == (c.width, c.height), (case, l)


def corner_points(h, rng):
    """World points whose (x_rot, y_rot) fall in and around the layer's top-right cell: each coordinate from the largest
    floats below the extent, the extent and the float above it, and the inside of the last column / row; plus the same bands
    along the row below and the column left of it."""
    from test_rotated_host import world
    res = h.resolution

    def band(L):
        ext = L * res
        return np.concatenate([bi.far_edge_points(L, res, 32)[0], [ext, math.nextafter(ext, 1e9)],
                               (L - 1 + rng.random(48)) * res])
    bx, by = band(h.width), band(h.height)
    gx, gy = np.meshgrid(bx, by)
    xr = np.concatenate([gx.ravel(), bx, (h.width - 2 + rng.random(by.size)) * res])
    yr = np.concatenate([gy.ravel(), (h.height - 2 + rng.random(bx.size)) * res, by])
    x, y = world(h, xr, yr, rng)
    n = gx.size
    return x, y, np.arange(n), np.arange(n, x.size)


def oracle_cells_wider(h, x, y):
    """The oracle's xy_2_rc on the same origin, rotation and resolution with one more row and column, as (row, col) (-1 off
    that map): there the layer's top-right cell is not the last cell, so a point in it reads its own index."""
    import types
    wide = types.SimpleNamespace(height=h.height + 1, width=h.width + 1, resolution=h.resolution, orig_x=h.orig_x,
                                 orig_y=h.orig_y, orig_c=h.orig_c, orig_s=h.orig_s)
    flat = oracle_cells(wide, x, y)
    last = wide.height * wide.width - 1
    return np.where(flat == last, -1, flat // wide.width), np.where(flat == last, -1, flat % wide.width)


@pytest.mark.parametrize('case', ['berlin', 'levine', 'example_map', 'rot_berlin', 'canvas4', 'rot4'])
def test_top_right_cell_against_the_oracle(f110, lookup_cases, case):
    """The one cell where the oracle's off-map read and its last cell look alike.  The wider map's oracle pins the model's
    cell there, and on the row below and the column left of it (where an off-map read differs from the cell's own index) the
    oracle pins the model's two extent tests at the same coordinates; the model combines them with the same expression."""
    dmap, hosts = lookup_cases[case]
    geom, res, rot, _ = layer_tables(dmap)
    rng = np.random.default_rng(sum(map(ord, case)) + 1)
    for l, h in enumerate(hosts):
        x, y, corner, edges = corner_points(h, rng)
        got = model_flat(h, geom[l], res[l], rot[l], x, y)
        assert agrees(h, got, oracle_cells(h, x, y)).all(), (case, l)
        r, c = oracle_cells_wider(h, x, y)
        on = got >= 0
        assert np.array_equal(got[on], r[on] * h.width + c[on]), (case, l)
        assert on[corner].sum() > 0 and (~on[corner]).sum() > 0, (case, l)
        # next to the corner the oracle tells the two apart, and both outcomes occur
        assert on[edges].sum() > 0 and (~on[edges]).sum() > 0, (case, l)
        assert np.all(got[edges][on[edges]] != h.height * h.width - 1)


def test_model_classes_on_a_tiny_map(f110):
    """Hand-checked classes: a 4 x 3 map at 1 m, origin (-1, -2); a 1 x 1 view at each point is that point's class; the
    followed car covers its own centre, another car at the same place shows as 4 (priority), a NaN car is not drawn."""
    dt = np.array([[0., 1., 1., 0.], [1., 0., 1., 1.], [1., 1., 1., 0.]])
    dmap = f110.DeviceMap(f110.maps.HostMap(dt, 1.0, (-1.0, -2.0, 0.0)), CPU)
    tables = layer_tables(dmap)
    pts = [(-1.0, -2.0, 2), (-0.5, -1.5, 2), (0.5, -1.5, 1), (2.999, 0.5, 2), (3.0, 0.5, 0), (-1.0 - 1e-15, 0.0, 0),
           (0.5, -1.0, 2), (1.0, 1.0, 0), (1.5, 0.999, 1), (np.nan, 0.0, 255), (1e12, 1e12, 0)]
    for x, y, want in pts:
        state = np.zeros((7, 1))
        state[0, 0], state[1, 0] = x, y
        far = np.full((1, 4, 2), 1e9)
        got = views_model(tables, state, np.array([[1.0, 0.0]]), far, None, 1, [0], 1, 1, 0.1, 0.0, True)
        assert got[0, 0, 0] == want, (x, y, got[0, 0, 0], want)
    # two agents at one spot: the follower's own quad wins; a car with a NaN pose is not drawn
    state = np.zeros((7, 2))
    state[0], state[1] = 0.5, -0.5
    quad = np.array([[0.2, -0.4], [0.2, -0.6], [0.8, -0.6], [0.8, -0.4]])
    verts = np.stack([quad, quad])
    cs = np.array([[1.0, 0.0], [1.0, 0.0]])
    v = views_model(tables, state, cs, verts, None, 2, [0, 1], 3, 3, 0.05, 0.0, False)
    assert v[0, 1, 1] == 4 and v[1, 1, 1] == 4
    state[0, 1] = np.nan
    v = views_model(tables, state, cs, verts, None, 2, [0, 1], 3, 3, 0.5, 0.0, False)
    assert v[1].tolist() == [[255] * 3] * 3 and not np.any(v[0] == 3)


def test_pixel_centres_of_a_one_pixel_view():
    for hu in (True, False):
        px, py = pixel_centres(3.25, -7.5, math.cos(0.7), math.sin(0.7), 1, 1, 0.1, 0.0, hu)
        assert (px[0, 0], py[0, 0]) == (3.25, -7.5)
    # heading-up: the top row lies ahead of the car, the right column to its right
    px, py = pixel_centres(0.0, 0.0, 0.0, 1.0, 3, 3, 1.0, 0.0, True)      # yaw pi/2: heading +y
    assert (px[0, 1], py[0, 1]) == (0.0, 1.0) and (px[1, 2], py[1, 2]) == (1.0, 0.0)
    px, py = pixel_centres(0.0, 0.0, 0.0, 1.0, 3, 3, 1.0, 2.0, False)
    assert (px[1, 1], py[1, 1]) == (0.0, 2.0) and (px[0, 0], py[0, 0]) == (-1.0, 3.0)


def test_walls_are_the_thresholded_bitmap(f110):
    """dt == 0 is exactly the image's pixels <= 128 (row 0 = image bottom) on every bundled map."""
    for n, e in SIX:
        img, _, _ = f110.maps.load_bitmap(os.path.join(MAPS, n + '.yaml'), e)
        assert np.array_equal(load(f110, n, e).host.dt == 0, img == 0), n


# ----------------------------------------------------------------------------- the C entry's refusals
@pytest.fixture(scope='module')
def sim(f110):
    s = f110.Simulator(f110.maps.DEFAULT_PARAMS, 2, 0, num_envs=3, device=CPU)
    return s


@pytest.fixture(scope='module')
def maps(f110):
    berlin, vegas, em = load(f110, *TRACKS[0]), load(f110, *TRACKS[1]), load(f110, 'example_map', '.png')
    h = berlin.host
    rot = f110.DeviceMap(f110.maps.HostMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.35)), CPU)
    return {'single': berlin, 'rot_single': rot, 'same_size': f110.DeviceMap.stack([em, em]),
            'canvas': f110.DeviceMap.stack([berlin, vegas]),
            'mixres': f110.DeviceMap.stack([berlin, em], mixed_resolution=True),
            'rot': f110.DeviceMap.stack([rot, vegas], rotated_origins=True)}


def copy(st):
    return type(st).from_buffer_copy(st)


def call(f110, sc, mc, V=2, H=8, W=8, s=0.1, f=0.0, ids=True, out=True):
    """f110_render_views with host buffers standing in for device ones (never dereferenced when the call is refused)."""
    lid = np.zeros(max(V, 1), np.int32)
    o = np.zeros(8, np.uint8)
    return f110._native.lib().f110_render_views(C.byref(sc) if sc is not None else None,
                                                 C.byref(mc) if mc is not None else None,
                                                 lid.ctypes.data if ids else None, V, H, W, s, f, 1,
                                                 o.ctypes.data if out else None, None)


def layered(sim, n):
    sc = copy(sim.c)
    sc.env_layer = np.zeros(n, np.int32).ctypes.data     # any non-NULL address: only its presence is checked here
    return sc


def test_export_and_abi_version(f110):
    L = f110._native.lib()
    assert L.f110_abi_version() == 6 == f110._native.ABI_VERSION
    assert 'f110_render_views' in f110._native.SIGNATURES and hasattr(L, 'f110_render_views')
    with open(os.path.join(os.path.dirname(__file__), '..', 'include', 'f110_b200.h')) as fh:
        hdr = fh.read()
    assert re.search(r'int f110_render_views\(const f110_sim \*sim, const f110_map \*map, const int32_t \*agent_ids, '
                     r'int32_t V, int32_t height,\s+int32_t width, double metres_per_pixel, double forward_offset, '
                     r'int32_t heading_up, uint8_t \*out,\s+void \*stream\);', hdr)
    assert '#define F110_ABI_VERSION 6' in hdr


def test_pointers_and_sizes(f110, sim, maps):
    mc = maps['single'].c
    assert call(f110, None, mc) == INVALID
    assert call(f110, sim.c, None) == INVALID
    assert call(f110, sim.c, mc, ids=False) == INVALID
    assert call(f110, sim.c, mc, out=False) == INVALID
    sc = copy(sim.c); sc.state = None
    assert call(f110, sc, mc) == INVALID
    for V in (0, -1):
        assert call(f110, sim.c, mc, V=V) == INVALID
    for H, W in ((0, 8), (8, 0), (8193, 8), (8, 8193), (-1, 8)):
        assert call(f110, sim.c, mc, H=H, W=W) == INVALID, (H, W)
    for s in (0.0, -0.1, math.inf, math.nan):
        assert call(f110, sim.c, mc, s=s) == INVALID, s
    for f in (math.inf, -math.inf, math.nan):
        assert call(f110, sim.c, mc, f=f) == INVALID, f
    sc = copy(sim.c); sc.num_agents = 65
    assert call(f110, sc, mc) == INVALID


def test_no_map(f110, sim):
    assert call(f110, sim.c, f110.simulator.empty_map_struct()) == NO_MAP


def test_stack_without_env_layer(f110, sim, maps):
    for k in ('same_size', 'canvas', 'mixres', 'rot'):
        assert call(f110, sim.c, maps[k].c) == INVALID, k


def test_table_rules(f110, sim, maps):
    """The rules of f110_scan_layers: layer_res needs layer_geom and no fast_path; layer_rot needs both tables and no
    fast_path; a same-size stack cannot have a rotated origin."""
    sc = layered(sim, 3)
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
        assert call(f110, sc, mc) == INVALID, name


def test_python_value_errors(f110, sim, maps):
    """Host-side checks of Simulator.render_views and the local_map settings: nothing reaches the device."""
    sim.set_device_map(maps['single'])
    bad = [dict(size=(0, 8)), dict(size=(8, 8193)), dict(size=(8.5, 8)), dict(size=8), dict(size=(1, 2, 3)),
           dict(metres_per_pixel=0.0), dict(metres_per_pixel=float('nan')), dict(forward_offset=float('inf')),
           dict(agent_ids=[0, 6]), dict(agent_ids=[-1]), dict(agent_ids=[0.5]), dict(agent_ids=[]),
           dict(agent_ids=np.array([7])), dict(agent_ids=torch.tensor([6])),
           dict(out=torch.empty((6, 64, 64), dtype=torch.int32))]
    for kw in bad:
        with pytest.raises(ValueError):
            sim.render_views(**kw)
    for cfg in ({'size': (8, 8)}, {'metres_per_pixel': 0.1}, {'size': (0, 8), 'metres_per_pixel': 0.1},
                {'size': (8, 8), 'metres_per_pixel': -1.0}, {'size': (8, 8), 'metres_per_pixel': 0.1, 'zoom': 2}):
        with pytest.raises(ValueError):
            f110.F110Env._local_map_settings(cfg)
    assert f110.F110Env._local_map_settings({'size': (8, 16), 'metres_per_pixel': 0.1}) == ((8, 16), 0.1, 0.0)
    with pytest.raises(ValueError):        # refused by the constructor, before anything is allocated
        f110.F110Env(map='vegas', num_agents=65, device=CPU, local_map={'size': (8, 8), 'metres_per_pixel': 0.1})


# ----------------------------------------------------------------------------- resource budget
# k_render_views -> (registers, stack bytes), DESIGN.md §3.6
RENDER_BUDGET = (48, 40)


def test_render_kernel_resource_budget():
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    out = subprocess.run([tool, '-res-usage', nat.LIB_PATH], capture_output=True, text=True).stdout
    usage = {fn: (int(reg), int(stack)) for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out)}
    name = '_ZN4f11014k_render_viewsENS_7RenderKE'
    assert usage.get(name) == RENDER_BUDGET, (name, usage.get(name))
