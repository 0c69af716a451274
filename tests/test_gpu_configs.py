"""The production tick and the stand-alone scans against the CPU oracle off the default configuration: beam counts, field of
view, LUT size (theta_dis), range, eps, time step and integrator, lidar offset, ego index and body size.

step_impl (csrc/f110_b200.cu) derives launch constants and kernel choices from these knobs: the Q16.48 LUT step and its
replay band, tmax and eps in cell units, the iTTC and GJK skip radii, the opponent skip at max_range + half the body
diagonal, march_ipa = ceil(B / 32) and the 256-item queue limit, the 1080-beam limit of the brick table, and the lean
kernel's conditions fov < 2 pi, theta_dis < 32768 and eps below the smallest positive distance.  Each tick case runs one
configuration, asserts through f110_debug_last_launch which march it reached (and fails with the record if not), and
compares every env with the oracle at every tick with the tolerances of test_gpu_scale.run_vs_oracle:

  state <= 1e-9; collisions, collision_idx, wall flags, done, toggles and lap counts exact; lap times <= 1e-9;
  beams the opponent ray-cast did not shorten == fp32(oracle); occluded beams <= 4e-6.

The stand-alone scans (f110_scan and f110_scan_layers, on a single map and on a stack) are bit-exact in fp64 against the
oracle with equal lookup counts, and equal the reference's own scans of tests/golden/kat_configs.npz where those exist.
"""
import math
import os

import numpy as np
import pytest
import torch

import boundary_inputs as bi
from test_gpu_boundaries import tick_vs_oracle
from test_gpu_scale import (assert_events, default_launch_settings, expect_path, raceline_population, run_vs_oracle,  # noqa: F401
                            MAPS)

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), 'golden')
DT_MIN_EXAMPLE = 0.0625          # smallest positive distance of example_map (its resolution)


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


_HOST = {}


def host_map(f110, name):
    if name not in _HOST:
        _HOST[name] = f110.maps.load_map(os.path.join(MAPS, name + '.yaml'), '.png')
    return _HOST[name]


def maps_for(f110, dev, name='example_map', **kw):
    """(DeviceMap, OracleMap) built alike: theta_dis, eps, max_range."""
    import oracle
    h = host_map(f110, name)
    return f110.DeviceMap(h, dev, **kw), oracle.OracleMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.0), **kw)


def run_case(f110, dev, poses, check, map_kw=None, drive='tick', autoreset=True, env_level=True, seed=1, **kw):
    dmap, omap = maps_for(f110, dev, **(map_kw or {}))
    return run_vs_oracle(f110, dev, dmap, [omap], poses, drive, autoreset=autoreset, env_level=env_level, seed=seed,
                         on_first_tick=check, **kw)


def lean(f110, brick=None, **want):
    """Launch check: the lean march (cell units, single map); brick True / False: the brick table must / must not be used."""
    def check():
        d = expect_path(f110, dict({'march': 'lean', 'CELLS': 1, 'LAYERED': 0}, **want))
        if brick is not None:
            assert (d.get('layout') == 'brick4x4') == brick, d
    return check


def fallback(f110, **want):
    """Launch check: the queued non-lean march (k_march_persistent)."""
    return lambda: expect_path(f110, dict({'march': 'persistent', 'CELLS': 1}, **want))


def pop(f110, n, A, seed):
    return raceline_population(f110, host_map(f110, 'example_map'), np.random.default_rng(seed), n, A)


# ----------------------------------------------------------------------------- beam counts
@pytest.mark.parametrize('B', [2, 3, 31, 32, 33, 64, 100])
def test_beam_counts_small(f110, dev, B):
    """Scans of 2 .. 100 beams: one to four 32-beam items per agent, partial last items, the brick table."""
    ev = run_case(f110, dev, pop(f110, 1024, 2, B), lean(f110, brick=True), B=B, seed=B)
    assert_events(ev, occluded=B >= 31, wall=B >= 31)


@pytest.mark.parametrize('B', [1079, 1080, 1081])
def test_beam_counts_brick_limit(f110, dev, B):
    """F110_BRICK_MAX_BEAMS = 1080: the brick table up to 1080 beams, the row-major table above."""
    assert_events(run_case(f110, dev, pop(f110, 512, 2, B), lean(f110, brick=B <= 1080), B=B, seed=B))


@pytest.mark.parametrize('B', [8192, 8224])
def test_beam_counts_queue_limit(f110, dev, B):
    """256 items per agent (8192 beams) still run the queued lean march; 257 (8224) have no queue and take the
    block-per-tile march."""
    check = lean(f110, brick=False) if B == 8192 else (lambda: expect_path(f110, {'march': 'block-per-tile', 'CELLS': 1}))
    assert_events(run_case(f110, dev, pop(f110, 96, 2, B), check, B=B, seed=B), gjk=False, resets=False)


def test_march_item_beams_64_odd(f110, dev):
    """march_item_beams=64 at an odd beam count: two 32-beam slices per queue item on the persistent march."""
    assert_events(run_case(f110, dev, pop(f110, 512, 2, 7), fallback(f110, SUB=2), B=1081, march_item_beams=64, seed=7))


# ----------------------------------------------------------------------------- field of view
@pytest.mark.parametrize('fov', [0.1, math.pi, 6.28])
def test_fov_lean(f110, dev, fov):
    ev = run_case(f110, dev, pop(f110, 512, 2, 11), lean(f110), B=270, fov=fov, seed=11)
    assert_events(ev, occluded=fov > 1, wall=fov > 1)


@pytest.mark.parametrize('fov', [2 * math.pi, 7.0])
def test_fov_full_circle_fallback(f110, dev, fov):
    """fov >= 2 pi: the doubled LUT of the lean march no longer covers a scan, so the persistent march runs."""
    assert_events(run_case(f110, dev, pop(f110, 512, 2, 12), fallback(f110), B=270, fov=fov, seed=12))


# ----------------------------------------------------------------------------- theta_dis
def lut_poses(f110, B, fov, T, rng, n=48):
    yaws, info = bi.lut_boundary_yaws(B, fov, n=n, rng=rng, theta_dis=T)
    print('theta_dis=%d B=%d fov=%g: %d yaws, %d beams replayed, %d plain indices wrong, %d wrong unreplayed'
          % (T, B, fov, yaws.size, info['replayed'], info['wrong_plain'], info['wrong_unreplayed']))
    assert info['replayed'] > 0 and info['wrong_unreplayed'] == 0
    h = host_map(f110, 'example_map')
    free = np.argwhere(h.dt > 0.6)
    sel = free[rng.choice(free.shape[0], yaws.size, replace=yaws.size > free.shape[0])]
    xy = np.stack([sel[:, 1] * h.resolution + h.orig_x + 0.011, sel[:, 0] * h.resolution + h.orig_y + 0.017], axis=1)
    return np.concatenate([xy, yaws[:, None]], axis=1)


@pytest.mark.parametrize('T', [1000, 2047, 2048, 4000, 16384, 32767, 32768])
def test_theta_dis(f110, dev, T):
    """Map LUT and beam tables built with theta_dis = T.  The lean march below 32768 (Q16.48 index), the persistent march at
    32768.  Yaws whose LUT index of some beam falls inside the replay band go through the tick (one tick from rest) and,
    below 32768, through f110_scan_layers, bit-exact in fp64 with equal lookup counts."""
    import oracle
    check = lean(f110) if T < 32768 else fallback(f110)
    assert_events(run_case(f110, dev, pop(f110, 256, 2, T), check, map_kw=dict(theta_dis=T), B=1080, seed=T % 97))
    dmap, omap = maps_for(f110, dev, theta_dis=T)
    rng = np.random.default_rng(T)
    for B, fov in ((1080, 4.7), (1081, 4.7), (270, math.pi)):
        poses = lut_poses(f110, B, fov, T, rng)
        rec, _ = tick_vs_oracle(f110, dev, dmap, poses[:, None, :], B=B, fov=fov, omaps=[omap])
        assert rec.get('march') == ('lean' if T < 32768 else 'persistent'), rec
        ss = f110.ScanSimulator2D(B, fov, theta_dis=T, device=dev)
        ss.set_device_map(dmap)
        want = [oracle.get_scan(omap, p, B, fov, count=True) for p in poses]
        if T < 32768:
            got, n = ss.scan(poses, out_f64=True, count_lookups=True, layer_ids=0)
            assert np.array_equal(got.cpu().numpy(), np.stack([w[0] for w in want])), (T, B)
            assert n == sum(w[1] for w in want)
        else:
            with pytest.raises(f110._native.F110Error):
                ss.scan(poses, layer_ids=0)
        got, n = ss.scan(poses, out_f64=True, count_lookups=True)
        assert np.array_equal(got.cpu().numpy(), np.stack([w[0] for w in want])) and n == sum(w[1] for w in want)


# ----------------------------------------------------------------------------- max_range, eps
def far_opponents(f110, n, A, rng):
    """Agents along the raceline 20-150 waypoints (about 4-30 m) apart: whether an opponent can shorten a beam depends on
    max_range."""
    wp = f110.maps.load_waypoints()
    k = rng.integers(0, wp.shape[0], n)
    gap = rng.integers(20, 76, n)
    return np.stack([wp[(k - gap * i) % wp.shape[0]] for i in range(A)], axis=1)


@pytest.mark.parametrize('mr', [5.0, 10.0])
def test_max_range_opponent_skip(f110, dev, mr):
    """max_range 5 m and 10 m with opponents 4-30 m away: the tail skips an opponent farther than max_range plus half its
    body diagonal, which now decides for most pairs."""
    rng = np.random.default_rng(int(mr))
    poses = far_opponents(f110, 512, 3, rng)
    d = np.hypot(*(poses[:, 1:, :2] - poses[:, :1, :2]).transpose(2, 0, 1))
    half_diag = 0.5 * math.hypot(0.58, 0.31)
    print('opponent distances: %d within max_range, %d beyond max_range + half diagonal' % ((d < mr).sum(), (d > mr + half_diag).sum()))
    assert (d < mr).sum() > 20 and (d > mr + half_diag).sum() > 100
    ev = run_case(f110, dev, poses, lean(f110), map_kw=dict(max_range=mr), seed=int(mr), autoreset=False)
    assert_events(ev, gjk=False, wall=False, resets=False, occluded=mr > 5)


def test_max_range_40(f110, dev):
    assert_events(run_case(f110, dev, pop(f110, 512, 2, 40), lean(f110, brick=True), map_kw=dict(max_range=40.0), seed=40))


@pytest.mark.parametrize('eps', [1e-6, DT_MIN_EXAMPLE, 0.1])
def test_eps(f110, dev, eps):
    """eps below the map's smallest positive distance: the lean march (`d > eps` is `d != 0`); at or above it the persistent
    march, which compares with eps."""
    check = lean(f110) if eps < DT_MIN_EXAMPLE else fallback(f110)
    assert_events(run_case(f110, dev, pop(f110, 256, 2, 50), check, map_kw=dict(eps=eps), seed=51))


# ----------------------------------------------------------------------------- dynamics knobs
@pytest.mark.parametrize('integrator', [1, 2])
@pytest.mark.parametrize('time_step', [0.002, 0.02, 0.05])
def test_time_step(f110, dev, time_step, integrator):
    """At 0.05 s the single-track model is unstable once a car passes 0.5 m/s, in the reference as here: within a few ticks
    yaw and yaw rate leave any sensible range (|yaw| ~ 1e3 by the fifth RK4 tick), which the opponent ray-cast must still
    handle as the reference does.  That RK4 run stops after 5 ticks, before the magnitudes make a 1e-9 state comparison
    meaningless."""
    ticks = 5 if (time_step == 0.05 and integrator == 1) else 12
    ev = run_case(f110, dev, pop(f110, 256, 2, 60 + integrator), lean(f110), time_step=time_step, integrator=integrator,
                  seed=61, ticks=ticks)
    assert_events(ev, gjk=time_step > 0.002, wall=time_step > 0.002, resets=time_step > 0.002)


def test_lidar_dist(f110, dev, sms):
    """lidar_dist 0.27 m at 4096 x 2 (scaled to the SM count): the scan pose ahead of the centre on the dynamic-tail lean
    march.  (No iTTC wall hits: a car a few centimetres from a wall scans from inside it, and a range of 0 never triggers.)"""
    n = int(4096 * sms / 132)
    assert_events(run_case(f110, dev, pop(f110, n, 2, 70), lean(f110, DYN=1), lidar_dist=0.27, seed=71), wall=False)


@pytest.mark.parametrize('A,N', [(2, 1024), (3, 1024), (8, 512)])
def test_ego_idx(f110, dev, A, N):
    """ego_idx = A - 1: `done`, the lap frame and the device auto-reset follow the ego.  An env where only the ego collided
    restarts; an env where only agent 0 collided goes on (the oracle does not restart it, and the state comparison holds
    the device to that)."""
    ev = run_case(f110, dev, pop(f110, N, A, 80 + A), lean(f110), ego_idx=A - 1, seed=81 + A)
    assert_events(ev)
    assert ev['ego_only'] > 0 and ev['agent0_only'] > 0, ev


@pytest.mark.parametrize('length,width', [(0.9, 0.45), (0.3, 0.2)])
def test_body_size(f110, dev, length, width):
    """Body size set at construction: GJK's skip radius, the opponent vertices of the ray-cast and the iTTC side distances."""
    params = dict(f110.maps.DEFAULT_PARAMS, length=length, width=width)
    poses = pop(f110, 512, 2, 90)
    if length < 0.5:            # trains 1 - 2 waypoints (0.2 - 0.4 m) apart, so that the short cars touch too
        wp = f110.maps.load_waypoints()
        k = np.random.default_rng(92).integers(0, wp.shape[0], 512)
        train = np.arange(512) % 3 == 1
        gap = 1 + (np.arange(512) // 3) % 2
        poses[train, 0] = wp[k][train]
        poses[train, 1] = wp[(k - gap) % wp.shape[0]][train]
    ev = run_case(f110, dev, poses, lean(f110), params=params, seed=91)
    assert_events(ev)


@pytest.mark.parametrize('A,drive', [(2, 'step'), (5, 'step'), (5, 'tick')])
def test_opponent_raycast_far_yaw(f110, dev, A, drive):
    """Ego yaws far outside [0, 2 pi) (the reference wraps the yaw once per step only, so a blown-up integration or a reset
    pose leaves it anywhere) with an opponent close behind the rear cut of the field of view: the ray-cast window is all
    beams and the wide-window cone filter picks the beams (k_tail2 at A = 2, k_finalize and k_tail at A = 5).  One tick from
    rest; everything equals the oracle."""
    import oracle
    dmap = f110.DeviceMap(host_map(f110, 'example_map'), dev)
    h = dmap.host
    rng = np.random.default_rng(100 + A)
    N = 256
    free = np.argwhere(h.dt > 1.2)
    sel = free[rng.choice(free.shape[0], N, replace=False)]
    yaws = np.array([351.14494331204725, -904.8591123984007, 6283.4, 0.7])[np.arange(N) % 4] + rng.uniform(-0.1, 0.1, N)
    poses = np.zeros((N, A, 3))
    poses[:, 0, 0] = sel[:, 1] * h.resolution + h.orig_x + 0.011
    poses[:, 0, 1] = sel[:, 0] * h.resolution + h.orig_y + 0.017
    poses[:, 0, 2] = yaws
    rel = yaws + np.where(rng.random(N) < 0.5, 1, -1) * rng.uniform(2.55, 2.95, N)
    dist = rng.uniform(0.45, 0.75, N)
    poses[:, 1, 0] = poses[:, 0, 0] + dist * np.cos(rel)
    poses[:, 1, 1] = poses[:, 0, 1] + dist * np.sin(rel)
    poses[:, 1, 2] = rng.uniform(0, 2 * np.pi, N)
    for i in range(2, A):                   # the others far away (skipped by the range test)
        poses[:, i, :2] = poses[:, 0, :2] + 40.0 * i
    sa = oracle.beam_tables(1080, 4.7, oracle.DEFAULT_PARAMS)[0]
    wide = sum(np.subtract(*oracle.blocked_view_indices(poses[e, 0], oracle.get_vertices(poses[e, 1], 0.58, 0.31), sa)[::-1])
               >= 96 for e in range(N))
    rec, ev = tick_vs_oracle(f110, dev, dmap, poses, B=1080, drive=drive)
    print('wide windows', wide, 'events', ev)
    assert wide > N // 4 and ev['occluded'] > 0, (wide, ev)
    assert rec.get('tail') == ('k_tail2' if A == 2 else 'k_finalize' if drive == 'step' else 'k_tail<1024,1>'), rec


# ----------------------------------------------------------------------------- stand-alone scans
def golden_configs():
    k = np.load(os.path.join(G, 'kat_configs.npz'))
    return [(str(n), int(c[0]), float(c[1]), float(c[2]), int(c[3]), float(c[4])) for n, c in zip(k['names'], k['configs'])]


EXTRA = [('td2047', 100, 4.7, 1e-4, 2047, 30.0), ('td2048', 100, 4.7, 1e-4, 2048, 30.0),
         ('td16384', 100, 4.7, 1e-4, 16384, 30.0), ('td32768', 100, 4.7, 1e-4, 32768, 30.0),
         ('eps1e-6', 100, 4.7, 1e-6, 2000, 30.0), ('eps0.0625', 100, 4.7, DT_MIN_EXAMPLE, 2000, 30.0),
         ('fov2pi', 33, 2 * math.pi, 1e-4, 2000, 30.0), ('b1079', 1079, 4.7, 1e-4, 2000, 30.0)]


@pytest.mark.parametrize('cfg', golden_configs() + EXTRA, ids=lambda c: c[0])
@pytest.mark.parametrize('name', ['example_map', 'berlin'])
def test_standalone_scans(f110, dev, name, cfg):
    """ScanSimulator2D(B, fov, eps=, theta_dis=, max_range=): scan() (f110_scan), scan(layer_ids=0) (k_scan_lean) and
    scan(layer_ids=...) on the map stacked with its 180-degree flip.  fp64 output bit-exact against the oracle with equal
    lookup counts; against the reference's scans where the golden has them.  Where the lean scan's preconditions fail
    (fov >= 2 pi, theta_dis >= 32768, eps not below every positive distance) scan(layer_ids=...) refuses."""
    import oracle
    label, B, fov, eps, td, mr = cfg
    kw = dict(eps=eps, theta_dis=td, max_range=mr)
    h = host_map(f110, name)
    ss = f110.ScanSimulator2D(B, fov, device=dev, **kw)
    ss.set_map(os.path.join(MAPS, name + '.yaml'), '.png')
    omap = oracle.OracleMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.0), **kw)
    k = np.load(os.path.join(G, 'kat_configs.npz'))
    poses = k['poses_' + name][:16 if B > 1080 else None]
    want = [oracle.get_scan(omap, p, B, fov, count=True) for p in poses]
    want_s, want_n = np.stack([w[0] for w in want]), sum(w[1] for w in want)
    names = [str(n) for n in k['names']]
    if label in names:
        assert np.array_equal(want_s, k['scan_%d_%s' % (names.index(label), name)])
    got, n = ss.scan(poses, out_f64=True, count_lookups=True)
    assert np.array_equal(got.cpu().numpy(), want_s) and n == want_n, label
    lean_ok = fov < 2 * math.pi and td < 32768 and eps < float(ss.map.c.dt_min_positive)
    if not lean_ok:
        with pytest.raises(f110._native.F110Error):
            ss.scan(poses, layer_ids=0)
        return
    got, n = ss.scan(poses, out_f64=True, count_lookups=True, layer_ids=0)
    rec = f110._native.lib().f110_debug_last_launch().decode()
    print(label, name, rec)
    assert np.array_equal(got.cpu().numpy(), want_s) and n == want_n, (label, rec)
    # a stack of the map and its flip: pose j on layer j % 2
    flipped = f110.maps.HostMap(np.ascontiguousarray(h.dt[::-1, ::-1]), h.resolution, (h.orig_x, h.orig_y, 0.0))
    ss.set_device_map(f110.DeviceMap.stack([ss.map, f110.DeviceMap(flipped, dev, **kw)]))
    ofl = oracle.OracleMap(flipped.dt, h.resolution, (h.orig_x, h.orig_y, 0.0), **kw)
    ids = np.arange(poses.shape[0]) % 2
    want = [oracle.get_scan(omap if i == 0 else ofl, p, B, fov, count=True) for p, i in zip(poses, ids)]
    got, n = ss.scan(poses, out_f64=True, count_lookups=True, layer_ids=ids)
    assert np.array_equal(got.cpu().numpy(), np.stack([w[0] for w in want])) and n == sum(w[1] for w in want), label


# ----------------------------------------------------------------------------- refusals and the packed scan block
def test_theta_dis_mismatch_refused(f110, dev):
    """Beam tables and map LUT of different theta_dis are refused; a matching non-default pair runs (test_theta_dis)."""
    dmap, _ = maps_for(f110, dev, theta_dis=4000)
    with pytest.raises(ValueError):
        f110.Simulator(f110.maps.DEFAULT_PARAMS, 2, 0, num_envs=2, device=dev).set_device_map(dmap)
    with pytest.raises(ValueError):
        f110.ScanSimulator2D(100, 4.7, device=dev).set_device_map(dmap)
    f110.Simulator(f110.maps.DEFAULT_PARAMS, 2, 0, num_envs=2, device=dev, theta_dis=4000).set_device_map(dmap)
    f110.ScanSimulator2D(100, 4.7, theta_dis=4000, device=dev).set_device_map(dmap)


def test_packed_u24_range(f110, dev):
    """The 24-bit scan block holds ranges below 32 m.  A 31 m map with a scan count not divisible by 4 (the kernel's
    unaligned tail) decodes to round(fp32 * 2^19) * 2^-19 for every beam, the 31 m ranges of the two cars outside the map
    included; a 40 m map or noise that reaches 32 m is refused by make_host_pipeline, and by step_host_async once the map or
    the noise changed."""
    N, A, B, T = 5, 1, 1081, 3
    assert (N * A * B) % 4 != 0
    dmap, _ = maps_for(f110, dev, max_range=31.0)
    poses = pop(f110, N, A, 5)
    h = host_map(f110, 'example_map')
    poses[3:, 0] = [[h.orig_x - 12.0, h.orig_y - 9.0, 0.3], [h.orig_x + 3.0, h.orig_y - 0.5, 4.0]]
    sims = []
    for packed in (False, True):
        sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 3, num_envs=N, num_beams=B, device=dev)
        sim.set_device_map(dmap)
        sim.env_reset(poses)
        sims.append((sim, sim.make_host_pipeline(depth=1, packed_scans=packed)))
    rng = np.random.default_rng(5)
    for t in range(T):
        act = np.stack([rng.uniform(-0.4, 0.4, N * A), rng.uniform(0, 2, N * A)], axis=1)
        for sim, sets in sims:
            sets[0]['actions'].copy_(torch.from_numpy(act))
            sim.step_host_async(sets[0])
            sim.wait_host(sets[0])
        f32 = sims[0][1][0]['scans'].numpy()
        dec = f110.Simulator.unpack_scans_u24(sims[1][1][0]['scans_u24'])
        expect = (np.rint(np.clip(f32, 0, None).astype(np.float64) * 2.0 ** 19) * 2.0 ** -19).astype(np.float32)
        assert np.array_equal(dec, expect), t
    assert (f32 == 31.0).sum() > B and (f32 < 30.0).sum() > B, f32.max()
    sim, sets = sims[1]
    d40, _ = maps_for(f110, dev, max_range=40.0)
    sim.set_device_map(d40)
    with pytest.raises(ValueError):
        sim.step_host_async(sets[0])
    with pytest.raises(ValueError):
        sim.make_host_pipeline(packed_scans=True)
    sim.set_device_map(dmap)
    sim.step_host_async(sets[0])
    sim.wait_host(sets[0])
    sim.set_noise(0.2)                       # 31 + 8 * 0.2 > 32
    with pytest.raises(ValueError):
        sim.step_host_async(sets[0])
