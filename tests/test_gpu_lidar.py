"""Agents without a lidar (Simulator.set_lidar, C ABI f110_lidar) on the GPU.

Twin simulators from identical resets, one with a lidar mask and one without, under the same random actions and auto-reset
tables: after every call every buffer is bit-identical except the sensorless agents' scan rows and the march queue; the scans
of the agents that have a lidar are bit-identical, and the sensorless rows stay as set_lidar left them (NaN, or a sentinel
written over them) through auto-resets, box clips and repeat calls.  Masks (none / ego / opponents / alternating) x A in
{1, 2, 3, 4, 6}; the seven map kinds of the lean march; step, tick and tick_repeat with K in {1, 3}; boxes near the agents;
per-env parameters, Euler, 270 / 2160 beams, lidar_dist and absurd poses.  Then the full path (noise, the literal march), a slot
that gets its lidar back, the oracle, a captured graph and F110Env with a pure-pursuit opponent.
"""
import numpy as np
import pytest
import torch

from test_gpu_repeat import (dev, f110, kinds, make_sim, population, same_bits, tables_of)  # noqa: F401 (fixtures)
from test_gpu_scale import AR_SEED, POSE_GAP, random_actions

pytestmark = pytest.mark.gpu

N = 96
# every buffer of f110_sim but the scans and the march queue
BUFFERS = ('state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'march_rec', 'wall_flag', 'collisions', 'collision_idx',
           'current_time', 'lap_times', 'lap_counts', 'toggle_list', 'near_starts', 'start_xs', 'start_ys', 'start_thetas',
           'start_rot', 'done', 'checkpoint_done', 'tick_counter')
OBST = ('obstacle_boxes', 'obstacle_active', 'obstacle_hit')


@pytest.fixture(autouse=True)
def default_variant(f110):
    L = f110._native.lib()
    L.f110_debug_set_variant(0)
    yield
    L.f110_debug_set_variant(0)


def mask_of(kind, A):
    return {'none': [False] * A, 'ego': [i == 0 for i in range(A)], 'opponents': [i != 0 for i in range(A)],
            'alternating': [i % 2 == 0 for i in range(A)]}[kind]


def record(f110):
    return f110._native.lib().f110_debug_last_launch().decode()


def boxes_near(poses, K=3):
    """(N, K, 5) car-sized boxes 1.5 m, 3 m, ... ahead of each env's agent 0 at its start."""
    p0 = poses[:, 0]
    d = 1.5 * (1 + np.arange(K))[None, :]
    x = p0[:, None, 0] + d * np.cos(p0[:, None, 2])
    y = p0[:, None, 1] + d * np.sin(p0[:, None, 2])
    return np.stack([x, y, np.repeat(p0[:, None, 2], K, 1) + 0.3, np.full_like(x, 0.58), np.full_like(x, 0.31)], axis=2)


def check_twins(a, b, mask, step, sentinel=None):
    for name in BUFFERS + (OBST if a.obstacle_boxes is not None else ()):
        assert same_bits(getattr(a, name), getattr(b, name)), (name, step)
    A, B = a.num_agents, a.num_beams
    sa, sb = a.scans.view(-1, A, B), b.scans.view(-1, A, B)
    on = [i for i in range(A) if mask[i]]
    off = [i for i in range(A) if not mask[i]]
    if on:
        assert same_bits(sa[:, on].contiguous(), sb[:, on].contiguous()), ('scans', step)
    if off:
        rows = sa[:, off]
        assert (bool(torch.isnan(rows).all()) if sentinel is None else bool((rows == sentinel).all())), ('sensorless rows', step)


def twin(f110, dev, case, A, mask, call, ticks=120, seed=1, obstacles=False, configure=None, poses_hook=None, sentinel=None,
         expect='short', **kw):
    """Masked twin a and plain twin b over `ticks` physics ticks of `call`; returns (a, b, events)."""
    dmap, hosts, kind, _ = case
    rng = np.random.default_rng(seed)
    ids = np.arange(N) % len(hosts)
    poses = population(kind, hosts, ids, rng, A)
    if poses_hook is not None:
        poses_hook(poses)
    tabs = tables_of(kind, hosts, rng, dev)
    a = make_sim(f110, dev, dmap, ids, poses, A, **kw)
    b = make_sim(f110, dev, dmap, ids, poses, A, **kw)
    for s in (a, b):
        if configure is not None:
            configure(s)
        if obstacles:
            s.set_obstacles(boxes_near(poses))
    a.set_lidar(mask)
    assert a.lidar == tuple(mask) and b.lidar == (True,) * A
    if sentinel is not None:
        a.scans.view(N, A, -1)[:, [i for i in range(A) if not mask[i]]] = sentinel
    K = {'step': 1, 'tick': 1, 'repeat1': 1, 'repeat3': 3}[call]
    ev = dict(resets=0, wall=0, box=0)
    S = sum(mask)
    for step in range(max(1, ticks // K)):
        act = torch.from_numpy(random_actions(rng, N, A)).to(dev)
        if call == 'step':
            a.step(act)
        elif call == 'tick':
            a.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        else:
            a.tick_repeat(act, K, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        if step == 0:
            rec = record(f110)
            want = ' lidar=%d/%d' % (S, A) if expect == 'short' else ' lidar=full'
            assert want in rec, (want, rec)
        if call == 'step':
            b.step(act)
        elif call == 'tick':
            b.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        else:
            b.tick_repeat(act, K, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        if call != 'step':
            ev['resets'] += int(b.done.sum())
        ev['wall'] += int(((b.collisions != 0) & (b.collision_idx < 0)).sum())
        if obstacles:
            ev['box'] += int((b.obstacle_hit >= 0).sum())
        if expect == 'short':
            check_twins(a, b, mask, step, sentinel)
        else:
            for name in BUFFERS + ('scans',):
                assert same_bits(getattr(a, name), getattr(b, name)), (name, step)
    return a, b, ev


@pytest.mark.parametrize('A', [1, 2, 3, 4, 6])
@pytest.mark.parametrize('mask', ['none', 'ego', 'opponents', 'alternating'])
def test_masks_and_agent_counts(f110, dev, kinds, mask, A):
    m = mask_of(mask, A)
    if all(m):
        pytest.skip('the mask gives every slot a lidar')
    _, _, ev = twin(f110, dev, kinds['example_map'], A, m, 'tick', ticks=300, seed=A * 5 + len(mask))
    print('events', ev)
    assert ev['resets'] > 0 and ev['wall'] > 0, ev


@pytest.mark.parametrize('call', ['step', 'tick', 'repeat1', 'repeat3'])
@pytest.mark.parametrize('name', ['example_map', 'no_brick', 'berlin', 'tracks4', 'mixed_resolution', 'rotated', 'rot4'])
def test_map_kinds_and_calls(f110, dev, kinds, name, call):
    if name == 'no_brick':
        f110._native.lib().f110_debug_set_variant(90)       # the single cell-unit map on the padded row-major table
    twin(f110, dev, kinds['example_map' if name == 'no_brick' else name], 3, [True, False, True], call, seed=11)
    twin(f110, dev, kinds['example_map' if name == 'no_brick' else name], 2, [False, True], call, seed=12)


@pytest.mark.parametrize('call', ['tick', 'repeat3', 'step'])
@pytest.mark.parametrize('name', ['example_map', 'tracks4', 'rotated'])
def test_obstacles_near_the_agents(f110, dev, kinds, name, call):
    _, _, ev = twin(f110, dev, kinds[name], 2, [True, False], call, ticks=150, seed=13, obstacles=True)
    print('events', ev)
    assert ev['box'] > 0, ev


@pytest.mark.parametrize('variant', ['env_params', 'euler', 'beams270', 'beams2160', 'lidar_dist', 'absurd'])
def test_off_the_default_configuration(f110, dev, kinds, variant):
    kw, configure, hook = {}, None, None
    if variant == 'env_params':
        def configure(sim):
            sim.update_params(dict(f110.maps.DEFAULT_PARAMS, mu=0.7, length=0.5, width=0.28), env_mask=torch.arange(N) % 2 == 0)
    elif variant == 'euler':
        kw['integrator'] = f110.Integrator.Euler
    elif variant == 'beams270':
        kw['num_beams'] = 270
    elif variant == 'beams2160':
        kw['num_beams'] = 2160
    elif variant == 'lidar_dist':
        kw['lidar_dist'] = 0.275
    else:
        def hook(poses):           # absurd coordinates: the literal march of the tick's kernel, listed by k_ttc_select
            poses[::4, :, 0] += 3e9
    for name in ('example_map', 'berlin'):
        for mask in ([True, False, False], [False, True, True]):
            twin(f110, dev, kinds[name], 3, mask, 'tick', ticks=80, seed=17, configure=configure, poses_hook=hook, **kw)


def test_sensorless_rows_are_never_written(f110, dev, kinds):
    """A sentinel in the sensorless rows survives ticks with auto-resets, box clips and repeat calls."""
    for call in ('tick', 'repeat3', 'step'):
        _, _, ev = twin(f110, dev, kinds['example_map'], 3, [True, False, False], call, ticks=150, seed=19, obstacles=True,
                        sentinel=123.0)
        if call != 'step':
            assert ev['resets'] > 0 and ev['box'] > 0, ev


@pytest.mark.parametrize('why', ['noise', 'literal'])
def test_full_path_equals_the_unmasked_call(f110, dev, kinds, why):
    kw = {'noise_std': 0.01} if why == 'noise' else {}
    if why == 'literal':
        f110._native.lib().f110_debug_set_variant(13)
    for call in ('tick', 'repeat3', 'step'):
        twin(f110, dev, kinds['example_map'], 2, [True, False], call, ticks=60, seed=23, expect='full', **kw)


def test_slot_gets_its_lidar_back(f110, dev, kinds):
    a, b, _ = twin(f110, dev, kinds['example_map'], 2, [True, False], 'tick', ticks=40, seed=29)
    dmap, hosts, kind, _ = kinds['example_map']
    tabs = tables_of(kind, hosts, np.random.default_rng(0), dev)
    rng = np.random.default_rng(31)
    a.set_lidar([True, True])
    assert a.lidar == (True, True)
    for step in range(30):
        act = torch.from_numpy(random_actions(rng, N, 2)).to(dev)
        a.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        assert 'lidar=' not in record(f110)
        b.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        for name in BUFFERS + ('scans',):
            assert same_bits(getattr(a, name), getattr(b, name)), (name, step)


def test_against_the_oracle(f110, dev, kinds):
    import oracle
    import test_gpu_rotated as rotated
    dmap, hosts, kind, _ = kinds['example_map']
    A, n = 2, 24
    rng = np.random.default_rng(37)
    poses = population(kind, hosts, np.zeros(n, dtype=np.int64), rng, A)
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=n, device=dev)
    sim.set_device_map(dmap)
    sim.env_reset(poses)
    sim.set_lidar([True, False])
    osims = [oracle.OracleSim(rotated.omap_of(hosts[0]), num_agents=A) for _ in range(n)]
    for e in range(n):
        osims[e].env_restart(poses[e])
    hits = 0
    for step in range(40):
        act = random_actions(rng, n, A)
        obs = sim.tick(act)
        assert 'lidar=1/2' in record(f110)
        oracle.step_batch(osims, act, env_level=True)
        st = sim.state.cpu().numpy().reshape(7, n, A).transpose(1, 2, 0)
        assert np.abs(st - oracle.gather(osims, 'state')).max() < 1e-8, step
        assert np.array_equal(obs['collisions'].cpu().numpy(), oracle.gather(osims, 'collisions')), step
        scans = obs['scans'].cpu().numpy()
        assert np.abs(scans[:, 0] - oracle.gather(osims, 'scans')[:, 0]).max() < 1e-4, step
        assert np.isnan(scans[:, 1]).all(), step
        hits += int(oracle.gather(osims, 'in_collision').sum())
    assert hits > 0


def test_graph_with_mask_equals_eager_ticks(f110, dev, kinds):
    dmap, hosts, kind, _ = kinds['example_map']
    wp = f110.maps.load_waypoints()
    A = 2
    rng = np.random.default_rng(41)
    k = rng.integers(0, wp.shape[0], N)
    poses = np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1)
    table = torch.from_numpy(wp).to(dev)
    g, e = (make_sim(f110, dev, dmap, None, poses, A) for _ in range(2))
    for s in (g, e):
        s.set_centerlines(wp[:, :2])
        s.set_lidar([True, False])
    abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
    g.capture_graph(abuf, autoreset_poses=table, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True, progress=True)
    resets = 0
    for step in range(150):
        act = torch.from_numpy(random_actions(rng, N, A)).to(dev)
        abuf.copy_(act.reshape(N * A, 2))
        g.replay()
        e.tick(act, autoreset_poses=table, pose_gap=POSE_GAP, seed=AR_SEED)
        e.update_progress()
        for name in BUFFERS + ('scans', 'track_s', 'track_progress', 'track_seg', 'track_d'):
            assert same_bits(getattr(g, name), getattr(e, name)), (name, step)
        resets += int(e.done.sum())
    assert resets > 0
    g.set_lidar(None)
    assert g._graph is None


def test_env_with_a_pure_pursuit_opponent(f110, dev):
    A, n = 2, 32
    kw = dict(map='example_map', map_ext='.png', num_agents=A, num_envs=n, scan_noise_std=0.0, device=dev)
    ea, eb = f110.F110Env(lidar=[True, False], **kw), f110.F110Env(**kw)
    wp = f110.maps.load_waypoints()
    rng = np.random.default_rng(43)
    k = rng.integers(0, wp.shape[0], n)
    poses = np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1)
    pl = f110.PurePursuitPlanner(device=dev)
    oa, _, _, _ = ea.reset(poses)
    ob, _, _, _ = eb.reset(poses)
    assert torch.isnan(oa['scans'][:, 1]).all() and not torch.isnan(ob['scans']).any()
    for step in range(200):
        opp = pl.plan_actions(ob, 0.82461887897713965, 0.90338203837889)[:, 1]
        act = torch.from_numpy(random_actions(rng, n, A)).to(dev)
        act[:, 1] = opp
        oa, ra, da, _ = ea.step(act)
        ob, rb, db, _ = eb.step(act)
        for key in ('poses_x', 'poses_y', 'poses_theta', 'linear_vels_x', 'ang_vels_z', 'collisions', 'lap_times', 'lap_counts'):
            assert same_bits(oa[key], ob[key]), (key, step)
        assert same_bits(oa['scans'][:, 0].contiguous(), ob['scans'][:, 0].contiguous()), step
        assert torch.isnan(oa['scans'][:, 1]).all(), step
        assert same_bits(torch.as_tensor(ra), torch.as_tensor(rb)) and torch.equal(da, db), step
    for bad in ([True], [True, False, True]):
        with pytest.raises(ValueError):
            f110.F110Env(lidar=bad, **kw)


def test_records_without_a_mask_carry_no_lidar_key(f110, dev, kinds):
    dmap, hosts, kind, _ = kinds['example_map']
    poses = population(kind, hosts, np.zeros(N, dtype=np.int64), np.random.default_rng(47), 2)
    sim = make_sim(f110, dev, dmap, None, poses, 2)
    act = torch.zeros((N, 2, 2), dtype=torch.float64, device=dev)
    sim.tick(act)
    plain = record(f110)
    assert 'lidar=' not in plain
    sim.set_lidar([True, True])
    sim.tick(act)
    assert record(f110) == plain
    sim.set_lidar([False, False])
    sim.tick(act)
    assert record(f110).startswith('march=none tail=k_tail_noscan') and record(f110).endswith(' lidar=0/2')
    with pytest.raises(ValueError):
        sim.set_lidar([True])
    with pytest.raises(ValueError):
        sim.step_profile(act)
    with pytest.raises(ValueError):
        sim.make_host_io()
    big = f110.Simulator(f110.maps.DEFAULT_PARAMS, 33, AR_SEED, num_envs=2, device=dev)
    with pytest.raises(ValueError):
        big.set_lidar([True] * 32 + [False])
    big.set_lidar([True] * 33)
