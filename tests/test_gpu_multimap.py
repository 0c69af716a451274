"""Multi-track batches on a canvas stack (DeviceMap.stack of maps that differ in size and origin): k_march_lean_het and the
per-map auto-reset start tables, against the oracle on each env's own map.

Every case compares every env at every tick with an oracle sim on that env's map, with the tolerances of test_gpu_scale.py
(state <= 1e-9; collisions, indices, wall flags, done, toggles, lap counts exact; beams no opponent shortened ==
fp32(oracle), or within one fp32 ulp of fp32(oracle + numpy noise); occluded beams <= 4e-6), and asserts its launch path
through f110_debug_last_launch (HET=1, layers=L, block shape, NOISE / COUNT).  The auto-reset draw is restated per layer:
an env on layer l restarts at table_l[(k - gap i) mod K_l] with k = min(floor(u K_l), K_l - 1).
"""
import os

import numpy as np
import pytest
import torch

import philox_ref
from test_gpu_scale import (AR_SEED, POSE_GAP, TOL_OCCLUDED, TOL_STATE, assert_events, cpu, expect_path, free_space_population,
                            mix64, M64, random_actions)

pytestmark = pytest.mark.gpu

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
TRACKS = [('berlin', '.png'), ('vegas', '.png'), ('skirk', '.png'), ('levine', '.pgm')]
T = 12


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


@pytest.fixture(scope='module')
def tracks(f110, dev):
    return [f110.DeviceMap.from_yaml(os.path.join(MAPS, n + '.yaml'), e, dev) for n, e in TRACKS]


@pytest.fixture(scope='module')
def cell_layers(f110, dev):
    """example_map and two crops of it with other sizes and shifted origins, EDT recomputed from the cropped images."""
    from scipy.ndimage import distance_transform_edt as edt
    em = f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', dev)
    h = em.host
    out = [em]
    for r0, c0, H, W in ((100, 300, 900, 1100), (450, 40, 1150, 700)):
        free = (h.dt[r0:r0 + H, c0:c0 + W] > 0).astype(np.float64) * 255.
        hm = f110.maps.HostMap(h.resolution * edt(free), h.resolution, (h.orig_x + c0 * h.resolution, h.orig_y + r0 * h.resolution, 0.0))
        out.append(f110.DeviceMap(hm, dev))
    return out


@pytest.fixture(autouse=True)
def default_launch_settings(f110):
    L = f110._native.lib()

    def defaults():
        L.f110_debug_set_variant(0)
        L.f110_debug_set_chunk(3)
        L.f110_debug_set_dyn(50, 4)
        L.f110_debug_set_ipt(-1, -1, -1, -1)
        L.f110_debug_set_tail(-2)
        L.f110_debug_set_tail2(256, 64)
        L.f110_debug_set_pdl(0)
    defaults()
    yield
    defaults()


def omap_of(h):
    import oracle
    return oracle.OracleMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.0))


def start_table(h, rng, K=64):
    """Seeded free-space start poses of one map (distance transform >= 0.6 m)."""
    free = np.argwhere(h.dt >= 0.6)
    sel = free[rng.choice(free.shape[0], K, replace=False)]
    return np.stack([sel[:, 1] * h.resolution + h.orig_x + 0.013, sel[:, 0] * h.resolution + h.orig_y + 0.007,
                     rng.uniform(0, 2 * np.pi, K)], axis=1)


def mixed_population(hosts, ids, rng, A):
    poses = np.zeros((ids.size, A, 3))
    for l, h in enumerate(hosts):
        m = ids == l
        poses[m] = free_space_population(h, rng, int(m.sum()), A)
    return poses


def layer_draw(table, seed, tick, env, A, gap):
    K = table.shape[0]
    hh = mix64((seed + 0x9E3779B97F4A7C15 * (tick + 1) + 0xD1B54A32D192ED03 * (env + 1)) & M64)
    k = min(int(float(hh >> 11) * (1.0 / 9007199254740992.0) * K), K - 1)
    return np.stack([table[(k - gap * i) % K] for i in range(A)])


def run_multi(f110, dev, dmap, hosts, ids, poses, drive, tables=None, env_level=True, noise_std=0.0, count=False, seed=1,
              check=None, ticks=T, actions=None):
    """T ticks of the CUDA path (drive 'tick' = f110_tick, 'step' = f110_step, 'graph' = a captured CUDA graph) against one
    oracle sim per env on its own map; returns event counts."""
    import oracle
    N, A = poses.shape[:2]
    NA, B = N * A, 1080
    rng = np.random.default_rng(seed)
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=N, num_beams=B, device=dev, noise_std=noise_std,
                         count_lookups=count)
    sim.set_device_map(dmap, env_map_ids=ids)
    sim.env_reset(poses)
    omaps = [omap_of(h) for h in hosts]
    osims = [oracle.OracleSim(omaps[ids[e]], num_agents=A, num_beams=B) for e in range(N)]
    for e in range(N):
        osims[e].env_restart(poses[e])
    dtabs = None if tables is None else [torch.from_numpy(t).to(dev) for t in tables]
    if drive == 'graph':
        abuf = torch.zeros((NA, 2), dtype=torch.float64, device=dev)
        sim.capture_graph(abuf, autoreset_poses=dtabs, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=env_level)
    ev = dict(gjk=0, occluded=0, wall=0, resets=0)
    for t in range(ticks):
        act = random_actions(rng, N, A) if actions is None else actions(t, N, A)
        if drive == 'graph':
            abuf.copy_(torch.from_numpy(act.reshape(NA, 2)))
            sim.replay()
        elif drive == 'tick':
            sim.tick(act, env_level=env_level, autoreset_poses=dtabs, pose_gap=POSE_GAP, seed=AR_SEED)
        else:
            sim.step(act)
        torch.cuda.synchronize()
        if t == 0 and check is not None:
            check()
        tick = int(sim.tick_counter.item())
        noise = philox_ref.tick_noise(sim.c.noise_seed, tick, NA, B, noise_std).reshape(N, A, B) if noise_std > 0 else None
        oracle.step_batch(osims, act, noise=noise, env_level=env_level)
        where = 'tick %d' % t
        got = cpu(sim.scans).reshape(N, A, B)
        fin, pre = oracle.gather(osims, 'scans'), oracle.gather(osims, 'scans_pre')
        occ = fin < pre
        want32 = fin.astype(np.float32)
        bad = (~occ) & ((got != want32) if noise is None else (np.abs(got - want32) > np.spacing(np.abs(want32))))
        assert not bad.any(), (where, 'scan', [(tuple(i), ids[i[0]], float(got[tuple(i)]), fin[tuple(i)]) for i in np.argwhere(bad)[:5]])
        d_occ = np.abs(got.astype(np.float64) - fin)[occ]
        assert d_occ.size == 0 or d_occ.max() <= TOL_OCCLUDED, (where, 'occluded', d_occ.max())
        ev['occluded'] += int(occ.sum())
        col = oracle.gather(osims, 'collisions')
        assert np.array_equal(cpu(sim.collisions).reshape(N, A), col), (where, 'collisions')
        cidx = oracle.gather(osims, 'collision_idx')
        assert np.array_equal(cpu(sim.collision_idx).reshape(N, A).astype(np.float64), cidx), (where, 'collision_idx')
        ev['gjk'] += int((cidx >= 0).sum())
        wall = oracle.gather(osims, 'in_collision')
        ev['wall'] += int(wall.sum())
        if env_level:
            assert np.array_equal(cpu(sim.done).astype(np.float64), oracle.gather(osims, 'done')), (where, 'done')
            assert np.array_equal(cpu(sim.lap_counts).reshape(N, A), oracle.gather(osims, 'lap_counts')), (where, 'laps')
            assert np.abs(cpu(sim.lap_times).reshape(N, A) - oracle.gather(osims, 'lap_times')).max() <= 1e-9, (where, 'lap_times')
        reset = np.zeros(N, bool)
        if tables is not None:
            reset = col[:, 0] != 0
            st = cpu(sim.state).reshape(7, N, A)
            for e in np.flatnonzero(reset):
                p = layer_draw(tables[ids[e]], AR_SEED, tick, int(e), A, POSE_GAP)
                assert np.array_equal(st[[0, 1, 4], e].T, p) and not st[[2, 3, 5, 6], e].any(), (where, 'auto-reset', e, ids[e])
                osims[e].env_restart(p)
            ev['resets'] += int(reset.sum())
        assert np.array_equal(cpu(sim.wall_flag).reshape(N, A)[~reset], wall[~reset]), (where, 'wall flags')
        st = cpu(sim.state).reshape(7, N, A).transpose(1, 2, 0)
        ds = np.abs(st - oracle.gather(osims, 'state')).max()
        assert ds <= TOL_STATE, (where, 'state', ds)
        if env_level:
            assert np.array_equal(cpu(sim.toggle_list).reshape(N, A), oracle.gather(osims, 'toggle_list')), (where, 'toggles')
    if count:
        assert sim.lookups() == int(oracle.gather(osims, 'nlook').sum())
    return ev


def het_path(f110, layers, cells, pt, noise=0, count=0):
    return lambda: expect_path(f110, {'march': 'lean-het', 'HET': 1, 'layers': layers, 'CELLS': cells, 'PT': pt,  # noqa: E731
                                      'MINB': 4 if pt == 512 else 2, 'NOISE': noise, 'COUNT': count})


# ----------------------------------------------------------------------------- the cases
@pytest.mark.parametrize('shape', ['4x512', '2x1024'])
def test_four_tracks_tick_with_per_layer_autoreset(f110, dev, sms, tracks, shape):
    """berlin / vegas / skirk / levine (metre units) through f110_tick with env level and per-layer auto-reset; sized from the
    SM count to reach both block shapes (2 x 1024 threads from 1400 queue items per SM)."""
    A = 2
    n = 8 * sms if shape == '4x512' else 24 * sms
    assert (n * A * 34 >= 1400 * sms) == (shape == '2x1024')
    ids = np.arange(n) % 4
    hosts = [m.host for m in tracks]
    rng = np.random.default_rng(200)
    tables = [start_table(h, rng) for h in hosts]
    poses = mixed_population(hosts, ids, rng, A)
    ev = run_multi(f110, dev, f110.DeviceMap.stack(tracks), hosts, ids, poses, 'tick', tables=tables, seed=201,
                   check=het_path(f110, 4, 0, 512 if shape == '4x512' else 1024))
    assert_events(ev)


def test_cell_units_example_map_and_crops(f110, dev, sms, cell_layers):
    A = 2
    n = 8 * sms
    ids = np.arange(n) % 3
    hosts = [m.host for m in cell_layers]
    rng = np.random.default_rng(210)
    tables = [start_table(h, rng) for h in hosts]
    poses = mixed_population(hosts, ids, rng, A)
    ev = run_multi(f110, dev, f110.DeviceMap.stack(cell_layers), hosts, ids, poses, 'tick', tables=tables, seed=211,
                   check=het_path(f110, 3, 1, 512))
    assert_events(ev)


@pytest.mark.parametrize('units', ['metres', 'cells'])
def test_guard_bands_on_every_layer(f110, dev, tracks, cell_layers, units):
    """Scan poses within 8 ulps of cell edges and just below / at W_l * res and H_l * res of each layer (boundary_inputs
    builders), cars at rest: every beam equals fp32(oracle)."""
    import boundary_inputs as bi
    layers = tracks if units == 'metres' else cell_layers
    hosts = [m.host for m in layers]
    rng = np.random.default_rng(220)
    per = 96
    xs, ids = [], []
    for l, h in enumerate(hosts):
        res = h.resolution
        t, _ = bi.cell_boundary_points(res, min(h.width, h.height) - 1, per // 2, rng)
        t = rng.permutation(t)[:per]
        edge_x = bi.far_edge_points(h.width, res, 4)[0]
        edge_y = bi.far_edge_points(h.height, res, 4)[0]
        px = np.concatenate([t, edge_x, rng.uniform(0, h.width * res, 4)])
        py = np.concatenate([rng.permutation(t), rng.uniform(0, h.height * res, 4), edge_y])
        p = np.stack([px + h.orig_x, py + h.orig_y, rng.uniform(0, 2 * np.pi, px.size)], axis=1)
        xs.append(p)
        ids.append(np.full(px.size, l))
    poses = np.concatenate(xs)[:, None, :]
    ids = np.concatenate(ids)
    zero = lambda t, N, A: np.zeros((N, A, 2))  # noqa: E731
    run_multi(f110, dev, f110.DeviceMap.stack(layers), hosts, ids, poses, 'step', env_level=False, seed=221, ticks=2,
              actions=zero, check=lambda: expect_path(f110, {'march': 'lean-het', 'HET': 1, 'layers': len(layers)}))


def test_noise_build(f110, dev, sms, tracks):
    A = 2
    n = 8 * sms | 1
    ids = np.arange(n) % 4
    hosts = [m.host for m in tracks]
    rng = np.random.default_rng(230)
    poses = mixed_population(hosts, ids, rng, A)
    ev = run_multi(f110, dev, f110.DeviceMap.stack(tracks), hosts, ids, poses, 'tick', noise_std=0.01, seed=231,
                   check=het_path(f110, 4, 0, 512, noise=1))
    assert_events(ev, resets=False)


def test_count_build(f110, dev, sms, tracks):
    A = 2
    n = 8 * sms
    ids = np.arange(n) % 4
    hosts = [m.host for m in tracks]
    rng = np.random.default_rng(240)
    poses = mixed_population(hosts, ids, rng, A)
    run_multi(f110, dev, f110.DeviceMap.stack(tracks), hosts, ids, poses, 'step', env_level=False, count=True, seed=241,
              check=het_path(f110, 4, 0, 512, count=1))


def _sim(f110, dev, N, A, noise):
    return f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=N, device=dev, noise_std=noise)


def test_batch_equals_separate_runs(f110, dev, sms, tracks):
    """Each layer's envs in the mixed batch equal, bit for bit, the same envs of a single-map Simulator over all N envs
    (same poses, actions, seeds, per-layer auto-reset table): scans, state, collisions, done and laps."""
    A, n = 2, 4 * sms
    ids = np.arange(n) % 4
    hosts = [m.host for m in tracks]
    rng = np.random.default_rng(250)
    tables = [torch.from_numpy(start_table(h, rng)).to(dev) for h in hosts]
    poses = mixed_population(hosts, ids, rng, A)
    acts = [random_actions(rng, n, A) for _ in range(T)]
    mixed = _sim(f110, dev, n, A, 0.01)
    mixed.set_device_map(f110.DeviceMap.stack(tracks), env_map_ids=ids)
    mixed.env_reset(poses)
    singles = []
    for l, m in enumerate(tracks):
        s = _sim(f110, dev, n, A, 0.01)
        s.set_device_map(m)
        s.env_reset(poses)
        singles.append(s)
    fields = ('scans', 'state', 'collisions', 'collision_idx', 'done', 'lap_times', 'lap_counts', 'toggle_list')
    resets = 0
    for t in range(T):
        mixed.tick(acts[t], autoreset_poses=tables, seed=AR_SEED)
        assert 'HET=1' in f110._native.lib().f110_debug_last_launch().decode()
        resets += int(cpu(mixed.collisions).reshape(n, A)[:, 0].astype(bool).sum())
        for l, s in enumerate(singles):
            s.tick(acts[t], autoreset_poses=tables[l], seed=AR_SEED)
            envs = np.flatnonzero(ids == l)
            for f in fields:
                a, b = cpu(getattr(mixed, f)), cpu(getattr(s, f))
                if f == 'state':
                    a, b = a.reshape(7, n, A)[:, envs], b.reshape(7, n, A)[:, envs]
                elif f == 'done':
                    a, b = a[envs], b[envs]
                else:
                    a, b = a.reshape(n, A, -1)[envs], b.reshape(n, A, -1)[envs]
                assert np.array_equal(a, b), ('tick %d' % t, f, l)
    assert resets > 0


def test_graph_equals_eager_tick(f110, dev, sms, tracks):
    A, n = 2, 4 * sms
    ids = np.arange(n) % 4
    hosts = [m.host for m in tracks]
    rng = np.random.default_rng(260)
    tables = [torch.from_numpy(start_table(h, rng)).to(dev) for h in hosts]
    poses = mixed_population(hosts, ids, rng, A)
    stacked = f110.DeviceMap.stack(tracks)
    g, e = _sim(f110, dev, n, A, 0.01), _sim(f110, dev, n, A, 0.01)
    for s in (g, e):
        s.set_device_map(stacked, env_map_ids=ids)
        s.env_reset(poses)
    abuf = torch.zeros((n * A, 2), dtype=torch.float64, device=dev)
    g.capture_graph(abuf, autoreset_poses=tables, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True)
    resets = 0
    for t in range(T):
        act = random_actions(rng, n, A)
        abuf.copy_(torch.from_numpy(act.reshape(-1, 2)))
        g.replay()
        e.tick(act, env_level=True, autoreset_poses=tables, pose_gap=POSE_GAP, seed=AR_SEED)
        resets += int(cpu(e.collisions).reshape(n, A)[:, 0].astype(bool).sum())
        for f in ('scans', 'state', 'collisions', 'done', 'lap_counts', 'lap_times', 'tick_counter'):
            assert np.array_equal(cpu(getattr(g, f)), cpu(getattr(e, f))), ('tick %d' % t, f)
    assert resets > 0


def test_f110env_with_a_map_list(f110, dev, tracks):
    names = [n for n, _ in TRACKS]
    exts = [e for _, e in TRACKS]
    N, A = 8, 2
    env = f110.F110Env(map=names, map_ext=exts, num_envs=N, num_agents=A, scan_noise_std=0.0)
    ids = np.arange(N) % 4
    hosts = [m.host for m in tracks]
    poses = mixed_population(hosts, ids, np.random.default_rng(270), A)
    ref = _sim(f110, dev, N, A, 0.0)
    ref.set_device_map(f110.DeviceMap.stack(tracks), env_map_ids=ids)
    obs, _, done, _ = env.reset(poses)
    ref.env_reset(poses)
    want = ref.step(np.zeros((N, A, 2)))
    ref.env_post_step()
    assert obs['scans'].shape == (N, A, 1080) and done.shape == (N,)
    for t in range(5):
        act = random_actions(np.random.default_rng(t), N, A)
        obs, _, done, _ = env.step(act)
        want = ref.step(act)
        ref.env_post_step()
        for k in ('scans', 'poses_x', 'poses_y', 'poses_theta', 'collisions'):
            assert torch.equal(obs[k], want[k]), (t, k)
        assert torch.equal(done, ref.done.bool())
    with pytest.raises(ValueError):
        f110.F110Env(map=names, map_ext=exts)                         # single-env mode
    with pytest.raises(ValueError):
        f110.F110Env(map=names, map_ext=exts[:2], num_envs=N)
    with pytest.raises(ValueError):
        env.sim.tick(np.zeros((N, A, 2)), autoreset_poses=[torch.zeros((4, 3), dtype=torch.float64, device=dev)] * 3)
