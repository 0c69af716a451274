"""The tick and the unit kernels against the CPU oracle on inputs built inside the guard bands of their exactness
shortcuts (tests/boundary_inputs.py), where random poses almost never land:

  LUT index           fixed-point index + replay (lean kernels), closed form + replay (k_raymarch, round-1 kernels),
                      and the first index equal to theta_dis
  metre cell index    FMA-corrected RN(t / res) at cell edges; coordinates just below width * res (far edge)
  opponent ray-cast   get_range_below's skips, all-beams window cone filter, nearest_beam ties, +-pi branch cut
  GJK                 contacts with the centres one body diagonal apart (the skip test's edge)
  iTTC                ranges within a few ulps of the threshold, v = +-0.0 and v < 0

Tolerances: beams the opponent did not shorten == fp32(oracle) bit for bit; lookup counts, collision flags and indices,
wall flags and ray-cast windows exact; the set of beams an opponent shortened equals the oracle's, values <= 4e-6.  Every
case prints how many of its inputs landed in their band and asserts that the count is not zero.
"""
import math
import os
import zlib

import numpy as np
import pytest
import torch

import boundary_inputs as bi

pytestmark = pytest.mark.gpu

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
TOL_OCCLUDED = 4e-6


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(autouse=True)
def default_variant(f110):
    L = f110._native.lib()
    L.f110_debug_set_variant(0)
    yield L.f110_debug_set_variant
    L.f110_debug_set_variant(0)


_MAP_CACHE = {}


def device_map(f110, dev, name):
    if name not in _MAP_CACHE:
        _MAP_CACHE[name] = f110.DeviceMap.from_yaml(os.path.join(MAPS, name + '.yaml'), '.png', dev)
    return _MAP_CACHE[name]


def cpu(t):
    return t.detach().cpu().numpy()


def omap_of(h, yaw=0.0):
    import oracle
    return oracle.OracleMap(h.dt, h.resolution, (h.orig_x, h.orig_y, yaw))


def launch_record(f110):
    rec = f110._native.lib().f110_debug_last_launch().decode()
    print('launch record:', rec)
    return dict(kv.split('=', 1) for kv in rec.split())


def tick_vs_oracle(f110, dev, dmap, poses, B=1080, fov=4.7, noise_std=0.0, omaps=None, env_map_ids=None, vel=None,
                   drive='step'):
    """Resets N envs at `poses` (N, A, 3) and runs one zero-action tick from rest (the pose does not move), on the device
    and on one oracle sim per env.  vel (N, A): longitudinal velocity written into both before the tick (the car then
    moves).  drive: 'step' = f110_step, 'tick' = the fused f110_tick without env-level logic.  Compares everything; returns
    (launch record, counts)."""
    import oracle
    import philox_ref
    N, A = poses.shape[:2]
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 12345, num_envs=N, num_beams=B, fov=fov, device=dev,
                         noise_std=noise_std, count_lookups=noise_std == 0.0, theta_dis=int(dmap.c.theta_dis))
    sim.set_device_map(dmap, env_map_ids=env_map_ids)
    sim.reset(poses)
    ids = np.zeros(N, int) if env_map_ids is None else np.asarray(env_map_ids)
    omaps = [omap_of(dmap.host)] if omaps is None else omaps
    osims = [oracle.OracleSim(omaps[ids[e]], num_agents=A, num_beams=B, fov=fov) for e in range(N)]
    for e in range(N):
        osims[e].reset(poses[e])
    act = np.zeros((N, A, 2))
    if vel is not None:
        sim.state.view(7, N, A)[3] = torch.from_numpy(vel).to(dev)
        for e in range(N):
            osims[e].state[:, 3] = vel[e]
        act[:, :, 1] = vel
    if drive == 'tick':
        sim.tick(act, env_level=False)
    else:
        sim.step(act)
    torch.cuda.synchronize()
    rec = launch_record(f110)
    tick = int(sim.tick_counter.item())
    noise = philox_ref.tick_noise(sim.c.noise_seed, tick, N * A, B, noise_std).reshape(N, A, B) if noise_std > 0 else None
    oracle.step_batch(osims, act, noise=noise)
    got = cpu(sim.scans).reshape(N, A, B)
    fin, pre = oracle.gather(osims, 'scans'), oracle.gather(osims, 'scans_pre')
    occ = fin < pre
    want = fin.astype(np.float32)
    bad = (~occ) & ((got != want) if noise is None else (np.abs(got - want) > np.spacing(np.abs(want))))
    assert not bad.any(), ('scan', [(tuple(i), float(got[tuple(i)]), fin[tuple(i)]) for i in np.argwhere(bad)[:5]])
    d = np.abs(got.astype(np.float64) - fin)[occ]
    assert d.size == 0 or d.max() <= TOL_OCCLUDED, d.max()
    got_occ = got < pre.astype(np.float32)
    assert np.array_equal(got_occ, occ), ('shortened beams differ', np.argwhere(got_occ != occ)[:5])
    assert np.array_equal(cpu(sim.collisions).reshape(N, A), oracle.gather(osims, 'collisions'))
    assert np.array_equal(cpu(sim.collision_idx).reshape(N, A).astype(np.float64), oracle.gather(osims, 'collision_idx'))
    wall = oracle.gather(osims, 'in_collision')
    assert np.array_equal(cpu(sim.wall_flag).reshape(N, A), wall)
    ds = np.abs(cpu(sim.state).reshape(7, N, A).transpose(1, 2, 0) - oracle.gather(osims, 'state')).max()
    assert ds <= 1e-9, ds
    if noise_std == 0.0:                           # (the lookup counter and the noise are separate builds)
        assert sim.lookups() == int(oracle.gather(osims, 'nlook').sum())
    return rec, dict(occluded=int(occ.sum()), wall=int(wall.sum()), gjk=int((oracle.gather(osims, 'collision_idx') >= 0).sum()))


def free_positions(h, n, rng, min_dt=0.6):
    free = np.argwhere(h.dt > min_dt)
    sel = free[rng.choice(free.shape[0], n, replace=n > free.shape[0])]
    return np.stack([sel[:, 1] * h.resolution + h.orig_x + 0.011, sel[:, 0] * h.resolution + h.orig_y + 0.017], axis=1)


def lut_poses(h, B, fov, rng, n=48):
    yaws, info = bi.lut_boundary_yaws(B, fov, n=n, rng=rng)
    print('B=%d fov=%g: %d yaws, %d beams replayed, %d beams whose plain fixed-point index is wrong, %d yaws at theta_dis'
          % (B, fov, yaws.size, info['replayed'], info['wrong_plain'], info['ti0_at_theta_dis'].size))
    assert info['replayed'] > 0 and info['wrong_plain'] > 0 and info['wrong_unreplayed'] == 0
    xy = free_positions(h, yaws.size, rng)
    return np.concatenate([xy, yaws[:, None]], axis=1)[:, None, :], info


# ----------------------------------------------------------------------------- LUT index
@pytest.mark.parametrize('name,B', [('example_map', 270), ('example_map', 1080), ('example_map', 1081),
                                    ('example_map', 2160), ('berlin', 1080), ('vegas', 2160), ('vegas', 1081)])
def test_lut_boundary_yaws_lean(f110, dev, name, B):
    """Lean kernel in cell units (example_map) and in metres (berlin, vegas): the Q16.48 index and its replay."""
    dmap = device_map(f110, dev, name)
    poses, info = lut_poses(dmap.host, B, 4.7, np.random.default_rng(B))
    rec, _ = tick_vs_oracle(f110, dev, dmap, poses, B=B)
    assert rec.get('march') == 'lean' and rec.get('CELLS') == ('1' if name == 'example_map' else '0'), rec


def test_lut_boundary_yaws_noise(f110, dev):
    dmap = device_map(f110, dev, 'example_map')
    poses, info = lut_poses(dmap.host, 1080, 4.7, np.random.default_rng(5))
    rec, _ = tick_vs_oracle(f110, dev, dmap, poses, noise_std=0.01)
    assert rec.get('NOISE') == '1', rec


@pytest.mark.parametrize('name', ['example_map', 'berlin'])
def test_lut_boundary_yaws_layered(f110, dev, name):
    import oracle
    dmap = device_map(f110, dev, name)
    h = dmap.host
    flipped = f110.maps.HostMap(np.ascontiguousarray(h.dt[::-1, ::-1]), h.resolution, (h.orig_x, h.orig_y, 0.0))
    stacked = f110.DeviceMap.stack([dmap, f110.DeviceMap(flipped, dev)])
    poses, _ = lut_poses(h, 1080, 4.7, np.random.default_rng(6))
    ids = np.arange(poses.shape[0]) % 2
    omaps = [omap_of(h), oracle.OracleMap(flipped.dt, h.resolution, (h.orig_x, h.orig_y, 0.0))]
    rec, _ = tick_vs_oracle(f110, dev, stacked, poses, omaps=omaps, env_map_ids=ids)
    assert rec.get('LAYERED') == '1', rec


@pytest.mark.parametrize('v', [1, 6, 7, 13])
@pytest.mark.parametrize('name', ['example_map', 'berlin'])
def test_lut_boundary_yaws_variants(f110, dev, default_variant, name, v):
    """Round-1 march kernels (closed form + replay, lidar.cuh beam_theta_index) and k_raymarch (variant 13)."""
    dmap = device_map(f110, dev, name)
    default_variant(v)
    poses, _ = lut_poses(dmap.host, 1080, 4.7, np.random.default_rng(100 + v))
    rec, _ = tick_vs_oracle(f110, dev, dmap, poses)
    assert rec.get('march') != 'lean', rec


@pytest.mark.parametrize('fov', [3.14, 1.5])
@pytest.mark.parametrize('name', ['example_map', 'berlin'])
def test_first_index_theta_dis_tick(f110, dev, name, fov):
    """Yaw one ulp below fov / 2: the first LUT index is exactly theta_dis (the reference reads one past its table; the
    index wraps to 0 everywhere here).  Lean kernel and k_raymarch (variant 13)."""
    dmap = device_map(f110, dev, name)
    y = math.nextafter(fov / 2., 0.)
    assert bi.theta_index0(y, fov) == 2000.0
    xy = free_positions(dmap.host, 8, np.random.default_rng(9))
    poses = np.concatenate([xy, np.full((8, 1), y)], axis=1)[:, None, :]
    tick_vs_oracle(f110, dev, dmap, poses, fov=fov)
    L = f110._native.lib()
    L.f110_debug_set_variant(13)
    tick_vs_oracle(f110, dev, dmap, poses, fov=fov)
    L.f110_debug_set_variant(1)
    tick_vs_oracle(f110, dev, dmap, poses, fov=fov)


@pytest.mark.parametrize('name', ['example_map', 'berlin', 'rotated'])
@pytest.mark.parametrize('B', [270, 1080, 1081, 2160])
def test_lut_boundary_yaws_scan_f64(f110, dev, name, B):
    """f110_scan (k_raymarch, fp64 out) against orc_get_scan: fast path (example_map), metre path (berlin), and a rotated
    origin (the general path with the rotation)."""
    import oracle
    if name == 'rotated':
        h0 = device_map(f110, dev, 'example_map').host
        h = f110.maps.HostMap(h0.dt, h0.resolution, (h0.orig_x, h0.orig_y, 0.3))
        dmap = f110.DeviceMap(h, dev)
    else:
        dmap = device_map(f110, dev, name)
        h = dmap.host
    poses = lut_poses(dmap.host if name != 'rotated' else device_map(f110, dev, 'example_map').host, B, 4.7,
                      np.random.default_rng(B + 1))[0][:, 0]
    for fov, extra in ((4.7, None), (3.14, math.nextafter(1.57, 0.))):
        if extra is not None:
            poses = poses[:8].copy()
            poses[:, 2] = extra
        ss = f110.ScanSimulator2D(B, fov, device=dev)
        ss.set_device_map(dmap)
        got, n = ss.scan(poses, out_f64=True, count_lookups=True)
        om = omap_of(h, 0.3 if name == 'rotated' else 0.0)
        ref = np.stack([oracle.get_scan(om, p, B, fov, count=True)[0] for p in poses])
        nref = sum(oracle.get_scan(om, p, B, fov, count=True)[1] for p in poses)
        assert np.array_equal(cpu(got), ref), np.argwhere(cpu(got) != ref)[:5]
        assert n == nref


# ----------------------------------------------------------------------------- metre-unit cell index
def _boundary_poses(h, rng, n=64, j_max=8, fov=4.7):
    """Positions whose x and y (relative to the origin) sit within j_max ulps of a cell edge, in free cells; yaw = fov / 2
    (beam 0 has LUT index 0: it runs along +x with y unchanged, so every lookup of that beam is on a row edge)."""
    free = np.argwhere(h.dt > 0.5)
    sel = free[rng.choice(free.shape[0], n, replace=False)]
    out = []
    for r, c in sel:
        for j in range(-j_max, j_max + 1, 2):
            tx = bi._ulps(float(c) * h.resolution, j)
            ty = bi._ulps(float(r) * h.resolution, -j)
            out.append([h.orig_x + tx, h.orig_y + ty, fov / 2.])
    poses = np.array(out)
    tx, ty = poses[:, 0] - h.orig_x, poses[:, 1] - h.orig_y
    on_edge = (np.abs(tx / h.resolution - np.round(tx / h.resolution)) < 1e-9) | \
              (np.abs(ty / h.resolution - np.round(ty / h.resolution)) < 1e-9)
    mism = (np.floor(tx * (1.0 / h.resolution)) != np.floor(tx / h.resolution)) | \
           (np.floor(ty * (1.0 / h.resolution)) != np.floor(ty / h.resolution))
    matter = bi.edges_that_matter(h.dt, ty, tx, h.resolution)
    return poses, int(on_edge.sum()), int(mism.sum()), int(matter.sum())


@pytest.mark.parametrize('v', [0, 1, 13])
@pytest.mark.parametrize('name', ['berlin', 'vegas', 'stata_basement'])
def test_cell_boundary_points(f110, dev, default_variant, name, v):
    """Lean metre kernel (0), round-1 persistent kernel (1), k_raymarch (13); the first lookup is k_dynamics'."""
    dmap = device_map(f110, dev, name)
    default_variant(v)
    poses, n_edge, n_mism, n_matter = _boundary_poses(dmap.host, np.random.default_rng(zlib.crc32(name.encode())))
    print('%s: %d poses on a cell edge, %d where t * (1 / res) alone names another cell, %d where the two cells at the '
          'edge hold different distances' % (name, n_edge, n_mism, n_matter))
    assert n_edge > 0 and n_mism > 0 and n_matter > 0
    rec, _ = tick_vs_oracle(f110, dev, dmap, poses[:, None, :])
    assert rec.get('march') == MARCH_OF_VARIANT[v] and rec.get('CELLS', '0') == '0', rec


# the march family each debug variant selects on a metre-unit map (launch record key `march`)
MARCH_OF_VARIANT = {0: 'lean', 1: 'persistent', 13: 'literal'}


# ----------------------------------------------------------------------------- far edge
def far_edge_map(f110, W=131, H=136, res=0.05, seed=3):
    from scipy.ndimage import distance_transform_edt as edt
    assert W in bi.far_edge_sizes(res, W, W + 1) and H in bi.far_edge_sizes(res, H, H + 1)
    rng = np.random.default_rng(seed)
    img = np.full((H, W), 255.0)
    for _ in range(40):
        r, c = rng.integers(0, H), rng.integers(0, W)
        img[max(r - 2, 0):r + 2, max(c - 2, 0):c + 2] = 0.0
    img[-1, -1] = 0.0                                  # dt[-1,-1] = 0 differs from every cell a far-edge read could name
    return f110.maps.HostMap(res * edt(img), res, (0.0, 0.0, 0.0))


def far_edge_poses(h, axis, fov=4.7):
    t, cell = bi.far_edge_points(h.width if axis == 'x' else h.height, h.resolution)
    assert (cell == (h.width if axis == 'x' else h.height)).any()
    other = (np.arange(t.size) * 7 % ((h.height if axis == 'x' else h.width) - 2) + 1) * h.resolution + 0.013
    poses = np.zeros((t.size, 3))
    poses[:, 0 if axis == 'x' else 1] = t
    poses[:, 1 if axis == 'x' else 0] = other
    # yaw fov / 2: beam 0 (LUT index 0) runs along +x; for the row edge it stays on the edge for every lookup
    poses[:, 2] = fov / 2. if axis == 'y' else fov / 2. + math.pi
    n_far = int((cell == (h.width if axis == 'x' else h.height)).sum())
    print('%s axis: %d of %d poses index one past the table' % (axis, n_far, t.size))
    return poses


@pytest.mark.parametrize('v', [0, 1, 13])
@pytest.mark.parametrize('axis', ['x', 'y'])
def test_far_edge_tick(f110, dev, default_variant, axis, v):
    h = far_edge_map(f110)
    dmap = f110.DeviceMap(h, dev)
    default_variant(v)
    rec, _ = tick_vs_oracle(f110, dev, dmap, far_edge_poses(h, axis)[:, None, :])
    assert rec.get('march') == MARCH_OF_VARIANT[v] and rec.get('CELLS', '0') == '0', rec


@pytest.mark.parametrize('axis', ['x', 'y'])
def test_far_edge_scan_f64(f110, dev, axis):
    import oracle
    h = far_edge_map(f110)
    dmap = f110.DeviceMap(h, dev)
    poses = far_edge_poses(h, axis)
    ss = f110.ScanSimulator2D(1080, 4.7, device=dev)
    ss.set_device_map(dmap)
    got = cpu(ss.scan(poses, out_f64=True))
    om = omap_of(h)
    ref = np.stack([oracle.get_scan(om, p, 1080, 4.7) for p in poses])
    assert np.array_equal(got, ref), np.argwhere(got != ref)[:5]
    assert (got[:, 0] == 0.0).any()               # the far-edge read really took dt[-1,-1] (= 0) somewhere


# ----------------------------------------------------------------------------- opponent ray-cast
@pytest.mark.parametrize('B', [270, 1080, 1081])
def test_ray_cast_edge_cases_standalone(f110, dev, B):
    import oracle
    beams = f110.DeviceBeams(B, 4.7, f110.maps.DEFAULT_PARAMS, dev)
    sa = cpu(beams.scan_angles)
    cases = bi.ray_cast_edge_cases(B)
    ego = np.stack([c[1] for c in cases])
    verts = np.stack([c[2] for c in cases])
    scan_in = np.full((len(cases), B), 30.0)
    out, win = f110.kernels.ray_cast(ego, scan_in, verts, beams, return_window=True)
    out, win = cpu(out).astype(np.float64), cpu(win)
    n_short = n_wide = n_graze = n_margin = n_wide_short = 0
    for k, (name, e, v) in enumerate(cases):
        ref = oracle.ray_cast(e, scan_in[k], sa, v)
        lo, hi = oracle.blocked_view_indices(e, v, sa)
        assert (win[k, 0], win[k, 1]) == (lo, hi), (name, win[k], lo, hi)
        differ = np.flatnonzero((out[k] < 30.0) != (ref < 30.0))
        # a ray through a vertex meets the edge at parameter 0 or 1 exactly; whether it counts is decided by the last ulp
        # of cos / sin(beam + pi / 2), which the device and the C library may round differently
        assert differ.size <= 2 and all(grazing(e, sa[i], v) for i in differ), \
            (name, [(i, grazing(e, sa[i], v)) for i in differ][:5])
        n_graze += differ.size
        if name == 'near_vertex':
            n_margin += len(bi.margin_sensitive_beams(e, sa, v))
        both = (out[k] < 30.0) & (ref < 30.0)
        assert not both.any() or np.abs(out[k] - ref)[both].max() <= TOL_OCCLUDED, (name, np.abs(out[k] - ref)[both].max())
        n_short += int((ref < 30.0).sum())
        n_wide += int(hi - lo >= 96)
        n_wide_short += int((ref < 30.0).sum()) if hi - lo >= 96 else 0
    print('%d cases, %d shortened beams compared (%d in all-beams windows), %d all-beams windows, %d beams a 1 - 1e-12 '
          'skip margin would change, %d grazing beams decided by a trig ulp'
          % (len(cases), n_short, n_wide_short, n_wide, n_margin, n_graze))
    assert n_short > 0 and n_wide > 0 and n_wide_short > 0 and n_margin > 0


def grazing(ego, angle, v, tol=1e-13):
    """True when beam `angle` of an ego pose meets an edge of the opponent polygon v (4, 2) at an edge parameter within
    tol of 0 or 1 (through a vertex), or runs within tol of parallel to an edge (laser_models.py get_range).  A few-ulp
    difference of cos / sin(beam + pi / 2) moves the parameter by about 1e-15 for these geometries: 1e-13 leaves a
    factor of 100, and stays below the 2e-13 that near_vertex cases sit from the vertex."""
    bt = ego[2] + angle
    v3 = np.array([math.cos(bt + math.pi / 2.), math.sin(bt + math.pi / 2.)])
    for j in range(4):
        va, vb = v[j], v[(j + 1) % 4]
        v2 = vb - va
        denom = v2 @ v3
        if abs(denom) <= tol * np.linalg.norm(v2):
            return True
        d2 = ((ego[:2] - va) @ v3) / denom
        if min(abs(d2), abs(d2 - 1.0)) < tol:
            return True
    return False


def _opponent_poses(B, rng, d_list=(0.9, 1.4, 2.5)):
    """Two-car envs on an open area: opponent behind (all-beams window, cone filter), straddling the rear cut within reach
    of the last beams, with a vertex a few 1e-13 of an edge off a beam (get_range_below's d2 <= 1 margin), on a beam
    direction, between two beams, on the first / last beam."""
    inc = 4.7 / (B - 1)
    out = []
    for phi, d, psi in bi.rear_straddle_params():
        out.append([[0.0, 0.0, 0.0], [d * math.cos(phi), d * math.sin(phi), psi]])
    for i, pose in bi.near_vertex_poses(B, 24, rng=rng, d_range=(0.8, 1.3)):
        out.append([[0.0, 0.0, 0.0], list(pose)])
    for d in d_list:
        for psi in (0.0, 0.7, math.pi / 2):
            out.append([[0.0, 0.0, 0.0], [-d, 0.0, psi]])
            out.append([[0.0, 0.0, 0.0], [-d, 1e-3, psi]])
        for i in rng.integers(B // 4, 3 * B // 4, 3):
            for a in (-4.7 / 2 + i * inc, -4.7 / 2 + (i + 0.5) * inc):
                out.append([[0.0, 0.0, 0.0], [d * math.cos(a), d * math.sin(a), float(rng.uniform(0, 2 * math.pi))]])
        for a in (-4.7 / 2, 4.7 / 2):
            out.append([[0.0, 0.0, 0.0], [d * math.cos(a), d * math.sin(a), a]])
    return np.array(out)


def expected_tail(drive, A):
    """Tail kernel of f110_step ('step') and of the fused f110_tick ('tick') at these batch sizes."""
    if 2 <= A <= 4:
        return 'k_tail2'
    if drive == 'step':
        return 'k_finalize'
    return 'k_tail<128,8>' if A == 1 else 'k_tail<1024,1>'


@pytest.mark.parametrize('drive', ['step', 'tick'])
@pytest.mark.parametrize('A', [1, 2, 3, 4, 6])
def test_ray_cast_edge_cases_tick(f110, dev, A, drive):
    """Through the tails: k_finalize (f110_step, A = 1 and A > 4), k_tail (f110_tick, A = 1 and A > 4) and k_tail2
    (A = 2 to 4).  A = 1 has no opponent and checks the plain tail on the same open-area poses."""
    h = device_map(f110, dev, 'example_map').host
    dmap = device_map(f110, dev, 'example_map')
    base = _opponent_poses(1080, np.random.default_rng(A))
    xy = free_positions(h, base.shape[0], np.random.default_rng(10 + A), min_dt=1.5)
    poses = np.zeros((base.shape[0], A, 3))
    for k in range(A):
        src = base[:, min(k, 1)].copy()
        if k >= 2:                                  # more opponents further out along the same bearing
            src[:, :2] *= 1.0 + 0.8 * (k - 1)
        poses[:, k] = src
    poses[:, :, :2] += xy[:, None, :]
    sa = f110.maps.beam_tables(1080, 4.7, f110.maps.DEFAULT_PARAMS)[0]
    n_margin = 0 if A == 1 else sum(len(bi.margin_sensitive_beams(poses[e, 0], sa, bi.car_vertices(*poses[e, 1])))
                                    for e in range(poses.shape[0]))
    rec, n = tick_vs_oracle(f110, dev, dmap, poses, drive=drive)
    print('tail', rec.get('tail'), n, '; beams a 1 - 1e-12 skip margin would change:', n_margin)
    assert rec.get('tail') == expected_tail(drive, A), rec
    if A > 1:
        assert n['occluded'] > 0 and n_margin > 0


# ----------------------------------------------------------------------------- GJK
def test_gjk_contacts_standalone(f110, dev):
    import oracle
    names, poses, beyond = bi.gjk_contact_poses()
    va = cpu(f110.kernels.get_vertices(poses[:, 0], 0.58, 0.31))
    vb = cpu(f110.kernels.get_vertices(poses[:, 1], 0.58, 0.31))
    ova = np.stack([oracle.get_vertices(p, 0.58, 0.31) for p in poses[:, 0]])
    ovb = np.stack([oracle.get_vertices(p, 0.58, 0.31) for p in poses[:, 1]])
    assert np.array_equal(va, ova) and np.array_equal(vb, ovb)
    got = cpu(f110.kernels.collision(va, vb))
    ref = np.array([oracle.collision(a, b) for a, b in zip(ova, ovb)])
    assert np.array_equal(got, ref), [names[i] for i in np.flatnonzero(got != ref)[:5]]
    col, idx = f110.kernels.collision_multiple(np.stack([va, vb], axis=1))
    for k in range(len(names)):
        rc, ri = oracle.collision_multiple(np.stack([ova[k], ovb[k]]))
        assert np.array_equal(cpu(col)[k], rc) and np.array_equal(cpu(idx)[k], ri), names[k]
    print('%d pairs, %d contacts' % (len(names), int(ref.sum())))
    assert ref.any() and not ref.all()


@pytest.mark.parametrize('drive', ['step', 'tick'])
@pytest.mark.parametrize('A', [2, 3, 6])
def test_gjk_contacts_tick(f110, dev, A, drive):
    """Contact pairs through the tails (k_tail2 for A = 2 and 3, k_finalize / k_tail for A = 6); extra agents far away."""
    dmap = device_map(f110, dev, 'example_map')
    names, pairs, beyond = bi.gjk_contact_poses()
    poses = np.zeros((len(names), A, 3))
    poses[:, :2] = pairs
    for k in range(2, A):
        poses[:, k] = pairs[:, 0] + np.array([3.0 * k, -4.0, 0.0])
    rec, n = tick_vs_oracle(f110, dev, dmap, poses, drive=drive)
    assert rec.get('tail') == expected_tail(drive, A), rec
    d2 = (pairs[:, 1, 0] - pairs[:, 0, 0]) ** 2 + (pairs[:, 1, 1] - pairs[:, 0, 1]) ** 2
    print('tail', rec.get('tail'), n, '; centres one diagonal apart:', int((d2 == 0.58 * 0.58 + 0.31 * 0.31).sum()))
    assert n['gjk'] > 0


# ----------------------------------------------------------------------------- iTTC
@pytest.mark.parametrize('B', [1080, 270])
def test_ttc_boundary_scans(f110, dev, B):
    import oracle
    beams = f110.DeviceBeams(B, 4.7, f110.maps.DEFAULT_PARAMS, dev)
    co, sd = cpu(beams.cosines), cpu(beams.side_distances)
    n_hit = n_rows = 0
    for v in (5.0, -3.0, 0.7, 19.9, 0.0, -0.0):
        scans, _ = bi.ttc_boundary_scans(sd, co, v)
        got = cpu(f110.kernels.check_ttc(scans, np.full(scans.shape[0], v), beams))
        ref = np.array([oracle.check_ttc(s, v, co, sd) for s in scans])
        assert np.array_equal(got, ref), (v, np.flatnonzero(got != ref)[:5])
        n_hit += int(ref.sum())
        n_rows += ref.size
    print('%d of %d boundary scans fire' % (n_hit, n_rows))
    assert 0 < n_hit < n_rows


def test_ttc_wall_at_threshold_tick(f110, dev):
    """Cars moving at v towards a wall from ranges around the iTTC threshold: per-agent pre-test + exact test in the lean
    kernel.  The start distances are spread finely over the band where the flag flips."""
    dmap = device_map(f110, dev, 'example_map')
    h = dmap.host
    gy, gx = np.gradient(h.dt)
    cells = np.argwhere((h.dt >= 0.20) & (h.dt <= 0.24) & (np.hypot(gx, gy) > 0))
    rng = np.random.default_rng(12)
    sel = cells[rng.choice(cells.shape[0], 256, replace=False)]
    r, c = sel[:, 0], sel[:, 1]
    yaw = np.mod(np.arctan2(-gy[r, c], -gx[r, c]), 2 * np.pi)
    poses = np.stack([(c + 0.5) * h.resolution + h.orig_x, (r + 0.5) * h.resolution + h.orig_y, yaw], axis=1)
    poses = np.repeat(poses, 8, axis=0)
    poses[:, 0] += np.tile(np.linspace(-0.02, 0.02, 8), 256) * np.cos(yaw.repeat(8))
    poses[:, 1] += np.tile(np.linspace(-0.02, 0.02, 8), 256) * np.sin(yaw.repeat(8))
    vel = np.tile(np.array([2.0, 5.0, 8.0, -1.0]), poses.shape[0] // 4)[:, None]
    rec, n = tick_vs_oracle(f110, dev, dmap, poses[:, None, :], vel=vel)
    print('wall hits', n['wall'], 'of', poses.shape[0])
    assert 0 < n['wall'] < poses.shape[0]
