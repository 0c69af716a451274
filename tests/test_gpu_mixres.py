"""Multi-track batches whose maps differ in resolution (DeviceMap.stack(maps, mixed_resolution=True)): k_march_lean_het_res
and the per-layer resolution of k_dynamics' first lookup, against the oracle on each env's own map.

The six bundled maps (0.05, 0.0504 and 0.0625 m) and generated tracks (0.0625 m) stacked with real ones, with the
tolerances and the restated per-layer auto-reset of test_gpu_multimap.run_multi; every case asserts its launch path (HET=1,
RES=1, layers=L, block shape, NOISE / COUNT).  A mixed batch also equals single-map simulators bit for bit, example_map's
on its cell-unit kernel.
"""
import os

import numpy as np
import pytest
import torch

from test_gpu_multimap import MAPS, T, TRACKS, _sim, mixed_population, run_multi, start_table
from test_gpu_scale import AR_SEED, POSE_GAP, assert_events, cpu, expect_path, random_actions

pytestmark = pytest.mark.gpu

SIX = TRACKS + [('stata_basement', '.png'), ('example_map', '.png')]


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
def six(f110, dev):
    return [f110.DeviceMap.from_yaml(os.path.join(MAPS, n + '.yaml'), e, dev) for n, e in SIX]


@pytest.fixture(scope='module')
def six_stack(f110, six):
    return f110.DeviceMap.stack(six, mixed_resolution=True)


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


def res_path(f110, layers, pt=None, noise=0, count=0):
    want = {'march': 'lean-het', 'HET': 1, 'RES': 1, 'CELLS': 0, 'layers': layers, 'NOISE': noise, 'COUNT': count}
    if pt is not None:
        want.update(PT=pt, MINB=4 if pt == 512 else 2)
    return lambda: expect_path(f110, want)  # noqa: E731


def generated(f110, dev, seed, count):
    """Generated tracks (trackgen.device_map, 0.0625 m) and host copies of their tables for the oracle."""
    from f1tenth_gym_b200 import trackgen as tg
    tracks = tg.random_tracks(seed, count)
    layers = [tg.device_map(t, dev) for t in tracks]
    hosts = [f110.maps.HostMap(m.dt.cpu().numpy(), m.host.resolution, (m.host.orig_x, m.host.orig_y, 0.0)) for m in layers]
    return tracks, layers, hosts


# ----------------------------------------------------------------------------- the cases
@pytest.mark.parametrize('shape', ['4x512', '2x1024'])
def test_six_maps_tick_with_per_layer_autoreset(f110, dev, sms, six, six_stack, shape):
    A = 2
    n = 8 * sms if shape == '4x512' else 24 * sms
    assert (n * A * 34 >= 1400 * sms) == (shape == '2x1024')
    ids = np.arange(n) % 6
    hosts = [m.host for m in six]
    rng = np.random.default_rng(300)
    tables = [start_table(h, rng) for h in hosts]
    poses = mixed_population(hosts, ids, rng, A)
    ev = run_multi(f110, dev, six_stack, hosts, ids, poses, 'tick', tables=tables, seed=301,
                   check=res_path(f110, 6, 512 if shape == '4x512' else 1024))
    assert_events(ev)


def test_generated_and_real_tracks(f110, dev, sms, six):
    """Three generated tracks with berlin and stata_basement, per-map auto-reset."""
    _, gen, ghosts = generated(f110, dev, 5, 3)
    layers = gen + [six[0], six[4]]
    hosts = ghosts + [six[0].host, six[4].host]
    A, n = 2, 8 * sms
    ids = np.arange(n) % 5
    rng = np.random.default_rng(310)
    tables = [start_table(h, rng) for h in hosts]
    poses = mixed_population(hosts, ids, rng, A)
    ev = run_multi(f110, dev, f110.DeviceMap.stack(layers, mixed_resolution=True), hosts, ids, poses, 'tick', tables=tables,
                   seed=311, check=res_path(f110, 5, 512))
    assert_events(ev)


def test_guard_bands_on_every_layer(f110, dev, six, six_stack):
    """Scan poses within 8 ulps of cell edges and just below / at W_l * res_l and H_l * res_l of each layer, cars at rest
    (f110_step): every beam equals fp32(oracle)."""
    import boundary_inputs as bi
    hosts = [m.host for m in six]
    rng = np.random.default_rng(320)
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
        xs.append(np.stack([px + h.orig_x, py + h.orig_y, rng.uniform(0, 2 * np.pi, px.size)], axis=1))
        ids.append(np.full(px.size, l))
    poses = np.concatenate(xs)[:, None, :]
    ids = np.concatenate(ids)
    zero = lambda t, N, A: np.zeros((N, A, 2))  # noqa: E731
    run_multi(f110, dev, six_stack, hosts, ids, poses, 'step', env_level=False, seed=321, ticks=2, actions=zero,
              check=res_path(f110, 6))


def test_noise_build(f110, dev, sms, six, six_stack):
    A, n = 2, 8 * sms | 1
    ids = np.arange(n) % 6
    hosts = [m.host for m in six]
    poses = mixed_population(hosts, ids, np.random.default_rng(330), A)
    ev = run_multi(f110, dev, six_stack, hosts, ids, poses, 'tick', noise_std=0.01, seed=331,
                   check=res_path(f110, 6, 512, noise=1))
    assert_events(ev, resets=False)


def test_count_build(f110, dev, sms, six, six_stack):
    A, n = 2, 8 * sms
    ids = np.arange(n) % 6
    hosts = [m.host for m in six]
    poses = mixed_population(hosts, ids, np.random.default_rng(340), A)
    run_multi(f110, dev, six_stack, hosts, ids, poses, 'step', env_level=False, count=True, seed=341,
              check=res_path(f110, 6, 512, count=1))


def test_batch_equals_separate_runs(f110, dev, sms, six, six_stack):
    """Each layer's envs in the six-map batch equal, bit for bit, the same envs of a single-map Simulator over all N envs
    (example_map's on the cell-unit kernel): scans, state, collisions, done, laps, and lookup counts in a counting run."""
    A, n = 2, 4 * sms
    ids = np.arange(n) % 6
    hosts = [m.host for m in six]
    rng = np.random.default_rng(350)
    tables = [torch.from_numpy(start_table(h, rng)).to(dev) for h in hosts]
    poses = mixed_population(hosts, ids, rng, A)
    acts = [random_actions(rng, n, A) for _ in range(T)]
    L = f110._native.lib()
    mixed = _sim(f110, dev, n, A, 0.01)
    mixed.set_device_map(six_stack, env_map_ids=ids)
    mixed.env_reset(poses)
    singles = []
    for m in six:
        s = _sim(f110, dev, n, A, 0.01)
        s.set_device_map(m)
        s.env_reset(poses)
        singles.append(s)
    fields = ('scans', 'state', 'collisions', 'collision_idx', 'done', 'lap_times', 'lap_counts', 'toggle_list')
    resets = 0
    for t in range(T):
        mixed.tick(acts[t], autoreset_poses=tables, seed=AR_SEED)
        assert 'HET=1 layers=6 RES=1' in L.f110_debug_last_launch().decode()
        resets += int(cpu(mixed.collisions).reshape(n, A)[:, 0].astype(bool).sum())
        for l, s in enumerate(singles):
            s.tick(acts[t], autoreset_poses=tables[l], seed=AR_SEED)
            rec = L.f110_debug_last_launch().decode()
            assert 'HET=0' in rec and ('CELLS=1' in rec) == (SIX[l][0] == 'example_map'), rec
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
    # lookup counts: each layer alone (the other envs of the batch parked on that layer's map would add their own)
    for l, m in enumerate(six):
        envs = np.flatnonzero(ids == l)
        counted = []
        for dmap, eids in ((six_stack, ids[envs]), (m, None)):
            s = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=envs.size, device=dev, noise_std=0.0,
                               count_lookups=True)
            s.set_device_map(dmap, env_map_ids=eids) if eids is not None else s.set_device_map(dmap)
            s.env_reset(poses[envs])
            for t in range(3):
                s.step(acts[t][envs])
            counted.append(s.lookups())
        assert counted[0] == counted[1] > 0, (l, counted)


def test_graph_equals_eager_tick(f110, dev, sms, six, six_stack):
    A, n = 2, 4 * sms
    ids = np.arange(n) % 6
    hosts = [m.host for m in six]
    rng = np.random.default_rng(360)
    tables = [torch.from_numpy(start_table(h, rng)).to(dev) for h in hosts]
    poses = mixed_population(hosts, ids, rng, A)
    g, e = _sim(f110, dev, n, A, 0.01), _sim(f110, dev, n, A, 0.01)
    for s in (g, e):
        s.set_device_map(six_stack, env_map_ids=ids)
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


def test_f110env_with_six_maps(f110, dev, six, six_stack):
    names = [n for n, _ in SIX]
    exts = [e for _, e in SIX]
    N, A = 12, 2
    with pytest.raises(ValueError):
        f110.F110Env(map=names, map_ext=exts, num_envs=N, num_agents=A)           # mixed resolutions are opt-in
    env = f110.F110Env(map=names, map_ext=exts, num_envs=N, num_agents=A, scan_noise_std=0.0, mixed_resolution=True)
    ids = np.arange(N) % 6
    poses = mixed_population([m.host for m in six], ids, np.random.default_rng(370), A)
    ref = _sim(f110, dev, N, A, 0.0)
    ref.set_device_map(six_stack, env_map_ids=ids)
    obs, _, done, _ = env.reset(poses)
    ref.env_reset(poses)
    ref.step(np.zeros((N, A, 2)))
    ref.env_post_step()
    for t in range(5):
        act = random_actions(np.random.default_rng(t), N, A)
        obs, _, done, _ = env.step(act)
        want = ref.step(act)
        ref.env_post_step()
        for k in ('scans', 'poses_x', 'poses_y', 'poses_theta', 'collisions'):
            assert torch.equal(obs[k], want[k]), (t, k)
        assert torch.equal(done, ref.done.bool())
    assert 'RES=1' in f110._native.lib().f110_debug_last_launch().decode()
    env.update_map([os.path.join(MAPS, n + '.yaml') for n in names[:4]], exts[:4], env_map_ids=np.arange(N) % 4,
                   mixed_resolution=False)
    env.step(np.zeros((N, A, 2)))
    assert 'HET=1 layers=4 CELLS=0' in f110._native.lib().f110_debug_last_launch().decode()


def test_closed_loop_generated_tracks_with_berlin(f110, dev, six):
    """Pure pursuit on per-env waypoint tables: envs on three generated tracks (0.0625 m) stacked with berlin (0.05 m) drive
    two clean laps; the berlin envs stand still on free-space poses."""
    tracks, gen, _ = generated(f110, dev, 11, 3)
    stacked = f110.DeviceMap.stack(gen + [six[0]], mixed_resolution=True)
    N = 8
    ids = np.arange(N) % 4
    on_gen = ids < 3
    still = mixed_population([six[0].host], np.zeros(N, int), np.random.default_rng(380), 1)
    starts = np.stack([tracks[ids[e]].start_pose(40 * e)[None] if on_gen[e] else still[e] for e in range(N)])
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 3, num_envs=N, device=dev)
    sim.set_device_map(stacked, env_map_ids=ids)
    sim.env_reset(starts)
    pl = f110.PurePursuitPlanner(device=dev, waypoints=[t.raceline(speed=5.0) for t in tracks], xind=0, yind=1, vind=2)
    tid = torch.as_tensor(np.where(on_gen, ids, 0), device=dev)
    park = torch.as_tensor(~on_gen, device=dev)
    obs = sim.observations()
    longest = max(np.linalg.norm(np.roll(t.waypoints, -1, 0) - t.waypoints, axis=1).sum() for t in tracks)
    gen_mask = torch.as_tensor(on_gen, device=dev)
    for k in range(int(2.6 * longest / 5.0 / 0.01)):
        act = pl.plan_actions(obs, 1.2, 1.0, table_ids=tid).clone()
        act[park] = 0.0
        obs = sim.tick(act)
        if k % 200 == 199 and bool(sim.done[gen_mask].all()):
            break
    assert 'RES=1' in f110._native.lib().f110_debug_last_launch().decode()
    laps = sim.lap_counts.cpu().numpy().reshape(N)
    assert bool(sim.done[gen_mask].all()), laps
    assert float(sim.collisions.sum()) == 0.0
    assert np.all(laps[on_gen] >= 2.0), laps


def test_layer_res_needs_the_metre_canvas_stack_path(f110, dev, six_stack):
    """layer_res without layer_geom, with fast_path, or on another march path (round-1 kernels: variant 1) returns
    F110_ERR_INVALID before anything is enqueued; the unmodified stack then steps."""
    N, A = 12, 2
    sim = _sim(f110, dev, N, A, 0.0)
    sim.set_device_map(six_stack, env_map_ids=np.arange(N) % 6)
    sim.env_reset(mixed_population([m.host for m in six_stack.layers], np.arange(N) % 6, np.random.default_rng(390), A))
    good = sim._map_struct
    no_geom = type(good).from_buffer_copy(good)
    no_geom.layer_geom = None
    cells = type(good).from_buffer_copy(good)
    cells.fast_path = 1
    zero = np.zeros((N, A, 2))
    try:
        for bad in (no_geom, cells):
            sim._map_struct = bad
            with pytest.raises(f110._native.F110Error):
                sim.step(zero)
        sim._map_struct = good
        f110._native.lib().f110_debug_set_variant(1)
        with pytest.raises(f110._native.F110Error):
            sim.step(zero)
    finally:
        sim._map_struct = good
    f110._native.lib().f110_debug_set_variant(0)
    sim.step(zero)
    assert 'RES=1' in f110._native.lib().f110_debug_last_launch().decode()
