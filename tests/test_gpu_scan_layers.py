"""ScanSimulator2D.scan(layer_ids=...) -> f110_scan_layers -> k_scan_lean: arbitrary poses, each on its own layer of any map
the Simulator accepts, against the reference goldens, the oracle's get_scan on the layer's own map (fp64, bit for bit, and
lookup counts), the tick's own scans, and f110_scan on single maps.  Every case asserts the kernel instance through the
launch record (scan=lean UNITS=cells|metres|rot layers=L).
"""
import math
import os
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import boundary_inputs as bi
from test_gpu_boundaries import _boundary_poses, far_edge_map, far_edge_poses
from test_gpu_rotated import YAWS, load, omap_of as rot_omap, to_world
from test_gpu_scale import cpu, near_wall_poses, random_actions

pytestmark = pytest.mark.gpu

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
G = os.path.join(os.path.dirname(__file__), 'golden')
TRACKS = [('berlin', '.png'), ('vegas', '.png'), ('skirk', '.png'), ('levine', '.pgm')]
SIX = TRACKS + [('stata_basement', '.png'), ('example_map', '.png')]
PER_LAYER = 10000


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def yaml_map(f110, dev, name, ext='.png'):
    return f110.DeviceMap.from_yaml(os.path.join(MAPS, name + '.yaml'), ext, dev)


@pytest.fixture(scope='module')
def six(f110, dev):
    return [yaml_map(f110, dev, n, e) for n, e in SIX]


def flipped(f110, dev, dmap, k):
    h = dmap.host
    dt = [h.dt[::-1, :], h.dt[:, ::-1], h.dt[::-1, ::-1]][k]
    return f110.DeviceMap(f110.maps.HostMap(np.ascontiguousarray(dt), h.resolution, (h.orig_x, h.orig_y, 0.0)), dev)


def crops(f110, dev, em):
    from scipy.ndimage import distance_transform_edt as edt
    h = em.host
    out = []
    for r0, c0, H, W in ((100, 300, 900, 1100), (450, 40, 1150, 700)):
        free = (h.dt[r0:r0 + H, c0:c0 + W] > 0).astype(np.float64) * 255.
        hm = f110.maps.HostMap(h.resolution * edt(free), h.resolution,
                               (h.orig_x + c0 * h.resolution, h.orig_y + r0 * h.resolution, 0.0))
        out.append(f110.DeviceMap(hm, dev))
    return out


@pytest.fixture(scope='module')
def kinds(f110, dev, six):
    """map kind -> (DeviceMap, [per-layer DeviceMap], expected UNITS)."""
    em = six[5]
    berlin = six[0]
    rb = load(f110, dev, 'berlin', '.png', YAWS['berlin'])
    rot_layers = [rb, load(f110, dev, 'vegas', '.png'), load(f110, dev, 'example_map', '.png', YAWS['example_map'], 0.0625),
                  load(f110, dev, 'skirk', '.png', YAWS['skirk']), load(f110, dev, 'levine', '.pgm', -2.6)]
    same = [em] + [flipped(f110, dev, em, k) for k in range(3)]
    cell_canvas = [em] + crops(f110, dev, em)
    return {
        'single_metres': (berlin, [berlin], 'metres'),
        'single_cells': (em, [em], 'cells'),
        'single_rot': (rb, [rb], 'rot'),
        'same_size': (f110.DeviceMap.stack(same), same, 'cells'),
        'cell_canvas': (f110.DeviceMap.stack(cell_canvas), cell_canvas, 'cells'),
        'metre_canvas': (f110.DeviceMap.stack(six[:4]), six[:4], 'metres'),
        'layer_res': (f110.DeviceMap.stack(six, mixed_resolution=True), six, 'metres'),
        'layer_rot': (f110.DeviceMap.stack(rot_layers, mixed_resolution=True, rotated_origins=True), rot_layers, 'rot'),
    }


def oracle_scans(h, poses, B=1080, fov=4.7):
    """orc_get_scan at every pose on the host map h -> (scans [M][B] fp64, lookups [M]); chunks on a thread pool (ctypes
    releases the GIL)."""
    import oracle
    om = rot_omap(h)
    M = poses.shape[0]
    out, nl = np.empty((M, B)), np.empty(M, np.int64)

    def run(lo):
        for k in range(lo, min(M, lo + 256)):
            out[k], nl[k] = oracle.get_scan(om, poses[k], B, fov, count=True)
    with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        list(ex.map(run, range(0, M, 256)))
    return out, nl


def record(f110):
    rec = f110._native.lib().f110_debug_last_launch().decode()
    return dict(kv.split('=', 1) for kv in rec.split())


def expect(f110, units, layers, count=None):
    d = record(f110)
    assert d.get('scan') == 'lean' and d.get('UNITS') == units and d.get('layers') == str(layers), d
    if count is not None:
        assert d.get('COUNT') == str(int(count)), d
    return d


def scanner(f110, dev, dmap, B=1080, fov=4.7):
    ss = f110.ScanSimulator2D(B, fov, device=dev)
    ss.set_device_map(dmap)
    return ss


class _Frame(object):
    def __init__(self, h):
        self.dt, self.resolution, self.height, self.width = h.dt, h.resolution, h.height, h.width
        self.orig_x = self.orig_y = 0.0


def population(h, rng, n):
    """n poses on map h in five groups: on-track (DT >= 0.3 m), free space, inside walls (DT = 0), hugging the map border
    from both sides, off the map.  Built in the map's own frame and turned into world coordinates."""
    f = _Frame(h)
    W, H = h.width * h.resolution, h.height * h.resolution
    k = n // 5
    parts = []
    for cond in (h.dt >= 0.3, h.dt > 0, h.dt == 0):
        cells = np.argwhere(cond)
        sel = cells[rng.choice(cells.shape[0], k, replace=k > cells.shape[0])]
        parts.append(np.stack([(sel[:, 1] + rng.uniform(0, 1, k)) * f.resolution,
                               (sel[:, 0] + rng.uniform(0, 1, k)) * f.resolution], axis=1))
    side = rng.integers(0, 4, k)
    t = rng.uniform(0, 1, k)
    d = rng.uniform(-0.05, 0.05, k)
    x = np.where(side == 0, d, np.where(side == 1, W + d, t * W))
    y = np.where(side == 2, d, np.where(side == 3, H + d, t * H))
    parts.append(np.stack([x, y], axis=1))
    m = n - 4 * k
    ang = rng.uniform(0, 2 * np.pi, m)
    rad = rng.uniform(1.0, 40.0, m) + 0.5 * math.hypot(W, H)
    parts.append(np.stack([0.5 * W + rad * np.cos(ang), 0.5 * H + rad * np.sin(ang)], axis=1))
    xy = np.concatenate(parts)
    p = np.concatenate([xy, rng.uniform(0, 2 * np.pi, (n, 1))], axis=1)
    return to_world(h, p)


def scan_layers(ss, poses, ids, **kw):
    return ss.scan(poses, layer_ids=torch.from_numpy(np.asarray(ids, np.int32)), **kw)


# ----------------------------------------------------------------------------- 1. reference goldens
def test_goldens_on_every_layer(f110, dev, six, kinds):
    """One call on the six-map layer_res stack with layer ids interleaved: the scans_wide_<map> and scans_<map> poses of all
    six maps equal the reference golden bit for bit (on its beam_idx where it has one); example_map also at 270, 540 and
    2160 beams."""
    st = kinds['layer_res'][0]
    names = [n for n, _ in SIX]
    files = {}

    def npz(name):
        if name not in files:
            files[name] = np.load(os.path.join(G, name))
        return files[name]
    poses, ids, want = [], [], []
    for l, n in enumerate(names):
        w = npz('scans_wide_%s.npz' % n)
        poses.append(w['poses'])
        ids += [l] * w['poses'].shape[0]
        want += [(l, 'wide', j) for j in range(w['poses'].shape[0])]
        if n != 'levine':
            g = npz('scans_%s.npz' % n)
            poses.append(g['poses'])
            ids += [l] * g['poses'].shape[0]
            want += [(l, 'plain', j) for j in range(g['poses'].shape[0])]
    poses = np.concatenate(poses)
    ids = np.asarray(ids)
    order = np.random.default_rng(600).permutation(ids.size)      # interleave the layers
    ss = scanner(f110, dev, st)
    got = cpu(scan_layers(ss, poses[order], ids[order], out_f64=True))
    expect(f110, 'metres', 6)
    assert len(set(ids[order][:12].tolist())) > 1
    inv = np.empty_like(order)
    inv[order] = np.arange(order.size)
    got = got[inv]
    for row, (l, kind, j) in enumerate(want):
        n = names[l]
        if kind == 'wide':
            w = npz('scans_wide_%s.npz' % n)
            if 'beam_idx' in w.files:
                assert np.array_equal(got[row][w['beam_idx'][j]], w['scan_1080_sub'][j]), (n, j)
            else:
                assert np.array_equal(got[row], w['scan_1080'][j]), (n, j)
        else:
            g = npz('scans_%s.npz' % n)
            assert np.array_equal(got[row], g['scan_1080'][j]), (n, 'plain', j)
    em = np.load(os.path.join(G, 'scans_example_map.npz'))
    wide = np.load(os.path.join(G, 'scans_wide_example_map.npz'))
    for B in (270, 540, 2160):
        ssb = scanner(f110, dev, st, B=B)
        p, ref = [em['poses']], [em['scan_%d' % B]]
        if 'scan_%d' % B in wide.files:
            p.append(wide['poses'][:48]); ref.append(wide['scan_%d' % B])
        p, ref = np.concatenate(p), np.concatenate(ref)
        got = cpu(scan_layers(ssb, p, np.full(p.shape[0], 5), out_f64=True))
        assert np.array_equal(got, ref), B


def test_golden_rotated_origin(f110, dev, six):
    """scans_rotated_origin.npz on a layer of a rotated stack and as a single rotated map."""
    k = np.load(os.path.join(G, 'scans_rotated_origin.npz'))
    em = six[5].host
    rm = f110.DeviceMap(f110.maps.HostMap(em.dt, float(k['resolution']), tuple(k['origin'])), dev)
    st = f110.DeviceMap.stack([six[1], rm], mixed_resolution=True, rotated_origins=True)
    P = k['poses']
    for dmap, l, layers in ((rm, 0, 1), (st, 1, 2)):
        got = cpu(scan_layers(scanner(f110, dev, dmap), P, np.full(P.shape[0], l), out_f64=True))
        expect(f110, 'rot', layers)
        assert np.array_equal(got, k['scan_1080'])


# ----------------------------------------------------------------------------- 2. oracle at scale on each map kind
@pytest.mark.parametrize('kind', ['single_metres', 'single_cells', 'single_rot', 'same_size', 'cell_canvas', 'metre_canvas',
                                  'layer_res', 'layer_rot'])
def test_oracle_at_scale(f110, dev, kinds, kind):
    dmap, layers, units = kinds[kind]
    rng = np.random.default_rng(zlib.crc32(kind.encode()))
    L = len(layers)
    poses = np.concatenate([population(m.host, rng, PER_LAYER) for m in layers])
    ids = np.repeat(np.arange(L), PER_LAYER)
    perm = rng.permutation(ids.size)
    ss = scanner(f110, dev, dmap)
    got, n = scan_layers(ss, poses[perm], ids[perm], out_f64=True, count_lookups=True)
    expect(f110, units, L, count=True)
    got = cpu(got)
    inv = np.empty_like(perm)
    inv[perm] = np.arange(perm.size)
    got = got[inv]
    total = 0
    for l, m in enumerate(layers):
        sl = slice(l * PER_LAYER, (l + 1) * PER_LAYER)
        ref, nl = oracle_scans(m.host, poses[sl])
        bad = np.argwhere(got[sl] != ref)
        assert bad.size == 0, (kind, l, bad[:5], got[sl][tuple(bad[0])], ref[tuple(bad[0])])
        total += int(nl.sum())
        # per-layer lookup totals: the layer's poses alone
        _, nlay = scan_layers(ss, poses[sl], np.full(PER_LAYER, l), out_f64=True, count_lookups=True)
        assert nlay == int(nl.sum()), (kind, l)
    assert n == total


# ----------------------------------------------------------------------------- 3. guard bands on every layer
def guard_poses(h, rng, rotated):
    """Cell edges, LUT guard yaws (270, 1080, 2160 beams), and, on a rotated layer, the rotated-frame builders (tiny negative
    x_rot / y_rot, -0.0, just below the extents); each builder is checked to land in its band."""
    out = {}
    if rotated:
        from test_rotated_host import rotated_probe_points
        x, y, bands = rotated_probe_points(h, rng, 1000)
        pick = np.concatenate([rng.permutation(v)[:64] for k, v in bands.items() if k not in ('uniform', 'far')])
        out['rotated_frame'] = np.stack([x[pick], y[pick], rng.uniform(0, 2 * np.pi, pick.size)], axis=1)
    else:
        p, n_edge, n_mism, n_matter = _boundary_poses(h, rng, n=32)
        assert n_edge > 0 and n_matter > 0
        out['cell_edges'] = p
    for B in (270, 1080, 2160):
        yaws, info = bi.lut_boundary_yaws(B, 4.7, n=32, rng=rng)
        assert info['replayed'] > 0 and info['wrong_plain'] > 0 and info['wrong_unreplayed'] == 0
        free = np.argwhere(h.dt > 0.6)
        sel = free[rng.choice(free.shape[0], yaws.size)]
        xy = to_world(h, np.stack([sel[:, 1] * h.resolution + 0.011, sel[:, 0] * h.resolution + 0.017, yaws], axis=1))
        xy[:, 2] = yaws                     # the world yaw alone sets the LUT index
        out['lut_%d' % B] = xy
    big = np.array([6e7, -6e7, 3e9, -3e9, 1e15])
    xy = np.stack([rng.choice(big, 40), rng.choice(big, 40)], axis=1) * rng.uniform(0.9, 1.1, (40, 2))
    out['absurd'] = np.concatenate([xy, rng.uniform(0, 2 * np.pi, (40, 1))], axis=1)
    return out


@pytest.mark.parametrize('kind', ['cell_canvas', 'layer_res', 'layer_rot'])
def test_guard_bands_on_every_layer(f110, dev, kinds, kind):
    dmap, layers, units = kinds[kind]
    rng = np.random.default_rng(700 + len(kind))
    for B in (270, 1080, 2160):
        ss = scanner(f110, dev, dmap, B=B)
        poses, ids = [], []
        for l, m in enumerate(layers):
            g = guard_poses(m.host, rng, m.host.orig_s != 0.0)
            for name, p in g.items():
                if name.startswith('lut_') and name != 'lut_%d' % B:
                    continue
                poses.append(p)
                ids.append(np.full(p.shape[0], l))
        poses, ids = np.concatenate(poses), np.concatenate(ids)
        got, n = scan_layers(ss, poses, ids, out_f64=True, count_lookups=True)
        d = expect(f110, units, len(layers))
        got = cpu(got)
        nref = 0
        for l, m in enumerate(layers):
            sel = ids == l
            ref, nl = oracle_scans(m.host, poses[sel], B)
            bad = np.argwhere(got[sel] != ref)
            assert bad.size == 0, (kind, B, l, bad[:5])
            nref += int(nl.sum())
        assert n == nref
    assert d['LITERAL'] == '0'


def test_far_edges(f110, dev, six):
    """Coordinates just below width * res on a map size where x / res rounds up to width, on layer 0 of a metre canvas."""
    h = far_edge_map(f110)
    fm = f110.DeviceMap(h, dev)
    st = f110.DeviceMap.stack([fm, six[0]])
    ss = scanner(f110, dev, st)
    for axis in ('x', 'y'):
        poses = far_edge_poses(h, axis)
        got = cpu(scan_layers(ss, poses, np.zeros(poses.shape[0]), out_f64=True))
        expect(f110, 'metres', 2)
        ref, _ = oracle_scans(h, poses)
        assert np.array_equal(got, ref), axis
        assert (got[:, 0] == 0.0).any()


# ----------------------------------------------------------------------------- 4. the tick's own scans
@pytest.mark.parametrize('kind', ['same_size', 'cell_canvas', 'metre_canvas', 'layer_res', 'layer_rot'])
def test_same_as_the_tick(f110, dev, kinds, kind):
    """A one-agent Simulator, noise off, 20 ticks of random actions; a third of the envs start 2 cm from a wall at 5 m/s so
    that iTTC fires.  After every tick the pose snapshot (Simulator.agent_poses) scanned on each env's layer reproduces the
    tick's scans bit for bit."""
    dmap, layers, units = kinds[kind]
    L = len(layers)
    N = 60 * L
    ids = np.arange(N) % L
    rng = np.random.default_rng(800 + len(kind))
    poses = np.zeros((N, 3))
    for l, m in enumerate(layers):
        e = np.flatnonzero(ids == l)
        h = m.host
        free = np.argwhere(h.dt > 0.6)
        sel = free[rng.choice(free.shape[0], e.size)]
        p = np.stack([sel[:, 1] * h.resolution + 0.011, sel[:, 0] * h.resolution + 0.017, rng.uniform(0, 2 * np.pi, e.size)], 1)
        poses[e] = to_world(h, p)
        wall = e[::3]
        f = _Frame(h)
        poses[wall] = to_world(h, near_wall_poses(f, rng, wall.size))
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 7, num_envs=N, device=dev, noise_std=0.0)
    sim.set_device_map(dmap, env_map_ids=ids)
    sim.reset(poses[:, None, :])
    v = np.where(np.arange(N) % (3 * L) < L, 5.0, 0.0)
    sim.state.view(7, N)[3] = torch.from_numpy(v).to(dev)
    ss = scanner(f110, dev, dmap)
    hits = 0
    for t in range(20):
        sim.step(random_actions(rng, N, 1))
        hits += int(cpu(sim.collisions).sum())
        got = scan_layers(ss, sim.agent_poses[:, :3], ids)
        expect(f110, units, L)
        assert torch.equal(got, sim.scans), (kind, t, np.argwhere(cpu(got) != cpu(sim.scans))[:5])
    assert hits > 0


# ----------------------------------------------------------------------------- 5. single maps against f110_scan
def test_single_maps_equal_f110_scan(f110, dev, six):
    rm = load(f110, dev, 'berlin', '.png', YAWS['berlin'])
    rng = np.random.default_rng(900)
    for m, units in [(m, 'cells' if m.host.fast_path else 'metres') for m in six] + [(rm, 'rot')]:
        ss = scanner(f110, dev, m)
        poses = population(m.host, rng, 4000)
        want, nw = ss.scan(poses, out_f64=True, count_lookups=True)
        got, ng = ss.scan(poses, out_f64=True, count_lookups=True, layer_ids=0)
        expect(f110, units, 1)
        assert torch.equal(got, want) and ng == nw


# ----------------------------------------------------------------------------- 6. invariance
@pytest.fixture(scope='module')
def batch(f110, dev, kinds):
    dmap, layers, _ = kinds['layer_res']
    rng = np.random.default_rng(1000)
    poses = np.concatenate([population(m.host, rng, 500) for m in layers])
    ids = np.repeat(np.arange(len(layers)), 500)
    perm = rng.permutation(ids.size)
    return dmap, poses[perm], ids[perm]


def test_permutation_and_single_pose(f110, dev, batch):
    dmap, poses, ids = batch
    ss = scanner(f110, dev, dmap)
    full = scan_layers(ss, poses, ids, out_f64=True)
    perm = np.random.default_rng(1).permutation(ids.size)
    assert torch.equal(scan_layers(ss, poses[perm], ids[perm], out_f64=True), full[torch.from_numpy(perm).to(dev)])
    for k in (0, 17, ids.size - 1):
        one = ss.scan(poses[k], out_f64=True, layer_ids=int(ids[k]))
        assert torch.equal(one[0], full[k])


def test_chunked_equals_unchunked(f110, dev, batch, monkeypatch):
    from f1tenth_gym_b200 import kernels
    dmap, poses, ids = batch
    ss = scanner(f110, dev, dmap)
    full, n = scan_layers(ss, poses, ids, out_f64=True, count_lookups=True)
    monkeypatch.setattr(kernels, 'SCAN_LAYERS_MAX_ELEMENTS', 7 * 1080 + 5)
    calls = []
    L = f110._native.lib()
    real = L.f110_scan_layers

    class Spy(object):
        def __call__(self, *a):
            calls.append(a[4])
            return real(*a)
    monkeypatch.setattr(L, 'f110_scan_layers', Spy())
    chunked, nc = scan_layers(ss, poses, ids, out_f64=True, count_lookups=True)
    assert max(calls) == 7 and len(calls) == -(-ids.size // 7)
    assert torch.equal(full, chunked) and n == nc


def test_two_streams(f110, dev, batch, kinds):
    dmap, poses, ids = batch
    rb = kinds['layer_rot'][0]
    ra = scanner(f110, dev, dmap)
    rr = scanner(f110, dev, rb)
    ids_r = ids % len(kinds['layer_rot'][1])
    serial_a = scan_layers(ra, poses, ids, out_f64=True)
    serial_b = scan_layers(rr, poses, ids_r, out_f64=True)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    with torch.cuda.stream(s1):
        a = scan_layers(ra, poses, ids, out_f64=True)
    with torch.cuda.stream(s2):
        b = scan_layers(rr, poses, ids_r, out_f64=True)
    torch.cuda.synchronize()
    assert torch.equal(a, serial_a) and torch.equal(b, serial_b)


def test_fp32_and_noise(f110, dev, batch):
    import philox_ref
    dmap, poses, ids = batch
    ss = scanner(f110, dev, dmap)
    f64 = scan_layers(ss, poses, ids, out_f64=True)
    f32 = scan_layers(ss, poses, ids)
    fin = torch.isfinite(f64)
    assert torch.equal(f32, f64.float())
    seed = 0xBEEF
    off0 = ss._noise_offset
    noisy = cpu(scan_layers(ss, poses, ids, rng=seed, std_dev=0.01))
    n = f32.numel()
    z = 0.01 * philox_ref.normal_sample(seed, 0xFFFFFFFF, np.uint64(off0) + np.arange(n, dtype=np.uint64))
    want = (cpu(f32).astype(np.float64).reshape(-1) + z).astype(np.float32).reshape(noisy.shape)
    assert np.all(np.abs(noisy - want) <= np.spacing(np.abs(want))) and fin.all()
    assert ss._noise_offset == off0 + n


# ----------------------------------------------------------------------------- 7. errors
def test_bad_layer_id_on_the_device(f110, dev, batch):
    """An out-of-range id passed straight to the C entry: NaN on that pose's beams only, every other pose exact, no
    lookups counted for it; the Python layer raises ValueError first."""
    import ctypes as C
    dmap, poses, ids = batch
    ss = scanner(f110, dev, dmap)
    want, n_want = scan_layers(ss, poses, ids, out_f64=True, count_lookups=True)
    bad = ids.astype(np.int32).copy()
    bad[[3, 11]] = [6, -1]
    keep = np.ones(ids.size, bool)
    keep[[3, 11]] = False
    p = torch.from_numpy(poses).to(dev).contiguous()
    lid = torch.from_numpy(bad).to(dev)
    out = torch.zeros((ids.size, 1080), dtype=torch.float64, device=dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    L = f110._native.lib()
    f110._native.check(L.f110_scan_layers(C.byref(dmap.c), C.byref(ss.beams.c), p.data_ptr(), lid.data_ptr(), ids.size, None,
                                          out.data_ptr(), cnt.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    torch.cuda.synchronize()
    assert torch.isnan(out[[3, 11]]).all()
    assert torch.equal(out[torch.from_numpy(keep).to(dev)], want[torch.from_numpy(keep).to(dev)])
    _, n_two = scan_layers(ss, poses[[3, 11]], ids[[3, 11]], out_f64=True, count_lookups=True)
    assert int(cnt.item()) == n_want - n_two
    for b in (bad, ids[:-1], np.full(ids.size, 2.0)):
        with pytest.raises(ValueError):
            ss.scan(poses, layer_ids=b)
    with pytest.raises(ValueError):
        ss.scan(poses, layer_ids=6)


def test_canvas_stack_without_layer_ids_still_raises(f110, dev, kinds):
    for k in ('cell_canvas', 'metre_canvas', 'layer_res', 'layer_rot'):
        ss = scanner(f110, dev, kinds[k][0])
        with pytest.raises(f110._native.F110Error):
            ss.scan(np.zeros((2, 3)))
