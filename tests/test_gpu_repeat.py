"""f110_tick_repeat (Simulator.tick_repeat, capture_graph(repeat=), F110Env(action_repeat=)) on the GPU.

Twin simulators from identical resets, one on tick_repeat(K) and one on K x tick(), under random actions with auto-reset:
after every call every buffer the header's contract names is bit-identical, the scans are the last tick's, done_any is the OR
and done_tick the first index of the plain run's per-tick done.  On every map kind the short path has an arithmetic of its
own for (cell units on the brick map, metres, a canvas stack, a mixed-resolution stack, a rotated map and a rotated stack),
with per-env parameters, Euler, other beam counts and fields of view, and with scan noise (the call then runs plain ticks and
says so).  Then against the oracle directly, through a captured graph with the progress tracker, and through F110Env.
"""
import os

import numpy as np
import pytest
import torch

import test_gpu_rotated as rotated
from test_gpu_multimap import MAPS, TRACKS, mixed_population, start_table
from test_gpu_scale import AR_SEED, POSE_GAP, random_actions

pytestmark = pytest.mark.gpu

N = 96
TICKS = 600        # physics ticks per case: 600 // K policy steps (300 at K = 2)
# every buffer of f110_sim the contract names (scans are compared too: they are the last tick's)
BUFFERS = ('state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'march_rec', 'wall_flag', 'collisions', 'collision_idx',
           'current_time', 'lap_times', 'lap_counts', 'toggle_list', 'near_starts', 'start_xs', 'start_ys', 'start_thetas',
           'start_rot', 'done', 'checkpoint_done', 'tick_counter', 'scans')


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(autouse=True)
def default_launch_settings(f110):
    L = f110._native.lib()
    L.f110_debug_set_variant(0)
    yield
    L.f110_debug_set_variant(0)


@pytest.fixture(scope='module')
def kinds(f110, dev):
    """name -> (device map, host maps of its layers, per-layer pose builders, UNITS the record must show)."""
    def plain(name, ext='.png'):
        return f110.DeviceMap.from_yaml(os.path.join(MAPS, name + '.yaml'), ext, dev)
    out = {}
    em, be = plain('example_map'), plain('berlin')
    out['example_map'] = (em, [em.host], 'plain', 'cells')
    out['berlin'] = (be, [be.host], 'plain', 'metres')
    tr = [plain(n, e) for n, e in TRACKS]
    out['tracks4'] = (f110.DeviceMap.stack(tr), [m.host for m in tr], 'plain', 'metres')
    mix = [em, be, tr[1]]
    out['mixed_resolution'] = (f110.DeviceMap.stack(mix, mixed_resolution=True), [m.host for m in mix], 'plain', 'metres')
    rb = rotated.load(f110, dev, 'berlin', '.png', rotated.YAWS['berlin'])
    out['rotated'] = (rb, [rb.host], 'rot', 'rot')
    rs = [rb, rotated.load(f110, dev, 'vegas', '.png'), rotated.load(f110, dev, 'skirk', '.png', rotated.YAWS['skirk']),
          rotated.load(f110, dev, 'example_map', '.png', rotated.YAWS['example_map'], 0.0625)]
    out['rot4'] = (f110.DeviceMap.stack(rs, mixed_resolution=True, rotated_origins=True), [m.host for m in rs], 'rot', 'rot')
    return out


def same_bits(x, y):
    """torch.equal on the bit patterns: NaN equals NaN (the record of an agent at absurd coordinates may hold one)."""
    if x.dtype == torch.float64:
        x, y = x.view(torch.int64), y.view(torch.int64)
    elif x.dtype == torch.float32:
        x, y = x.view(torch.int32), y.view(torch.int32)
    return torch.equal(x, y)


def population(kind, hosts, ids, rng, A):
    return rotated.population(hosts, ids, rng, A) if kind == 'rot' else mixed_population(hosts, ids, rng, A)


def tables_of(kind, hosts, rng, dev):
    tabs = [(rotated.start_table if kind == 'rot' else start_table)(h, rng) for h in hosts]
    tabs = [torch.from_numpy(np.ascontiguousarray(t)).to(dev) for t in tabs]
    return tabs if len(tabs) > 1 else tabs[0]


def make_sim(f110, dev, dmap, ids, poses, A, **kw):
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=poses.shape[0], device=dev, **kw)
    sim.set_device_map(dmap, env_map_ids=ids if len(getattr(dmap, 'layers', [])) > 1 else None)
    sim.env_reset(poses)
    return sim


def twin_run(f110, dev, case, K, A, steps=None, seed=3, configure=None, expect_sub='ttc', **kw):
    """steps calls of tick_repeat(K) against steps x K plain ticks; returns the event counts."""
    dmap, hosts, kind, units = case
    steps = max(1, min(300, TICKS // K)) if steps is None else steps
    rng = np.random.default_rng(seed)
    ids = np.arange(N) % len(hosts)
    poses = population(kind, hosts, ids, rng, A)
    tabs = tables_of(kind, hosts, rng, dev)
    a = make_sim(f110, dev, dmap, ids, poses, A, **kw)
    b = make_sim(f110, dev, dmap, ids, poses, A, **kw)
    if configure is not None:
        configure(a), configure(b)
    ev = dict(wall=0, gjk=0, resets=0, mid_call_done=0, toggles=0, marched=0.0)
    wall, gjk = torch.zeros((), dtype=torch.int64, device=dev), torch.zeros((), dtype=torch.int64, device=dev)
    for step in range(steps):
        act = torch.from_numpy(random_actions(rng, N, A)).to(dev)
        obs = a.tick_repeat(act, K, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        if step == 0:
            rec = f110._native.lib().f110_debug_last_launch().decode()
            want = 'repeat=%d sub=%s UNITS=%s' % (K, expect_sub if K > 1 else 'full', units)
            assert want in rec, (want, rec)
        dones = []
        for _ in range(K):
            b.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
            dones.append(b.done.clone())
            wall += ((b.collisions != 0) & (b.collision_idx < 0)).sum()     # (the auto-reset clears wall_flag)
            gjk += (b.collision_idx >= 0).sum()
        for name in BUFFERS:
            assert torch.equal(getattr(a, name), getattr(b, name)), (name, step)
        d = torch.stack(dones).bool()                               # (K, N)
        first = torch.where(d.any(0), d.int().argmax(0), torch.full((N,), -1, device=dev)).int()
        assert torch.equal(obs['done_any'].bool(), d.any(0)), step
        assert torch.equal(obs['done_tick'], first), step
        ev['resets'] += int(d.sum())
        ev['mid_call_done'] += int(((first >= 0) & (first < K - 1)).sum())
        ev['toggles'] = max(ev['toggles'], float(b.toggle_list.max()))
    ev['wall'], ev['gjk'], ev['marched'] = int(wall), int(gjk), a.marched_fraction()
    print('events', ev)
    assert ev['wall'] > 0 and ev['resets'] > 0 and ev['toggles'] > 0, ev
    if A > 1:
        assert ev['gjk'] > 0, ev
    if K > 2:
        assert ev['mid_call_done'] > 0, ev
    return ev


@pytest.mark.parametrize('A', [1, 2, 4])
@pytest.mark.parametrize('K', [1, 2, 5, 10])
@pytest.mark.parametrize('name', ['example_map', 'berlin', 'tracks4', 'mixed_resolution', 'rot4', 'rotated'])
def test_repeat_equals_plain_ticks(f110, dev, kinds, name, K, A):
    ev = twin_run(f110, dev, kinds[name], K, A, seed=K * 7 + A)
    if K > 1:
        assert 0.0 < ev['marched'] < 1.0, ev
    else:
        assert ev['marched'] is None


@pytest.mark.parametrize('variant', ['env_params', 'euler', 'beams270', 'beams2160', 'fov'])
def test_repeat_off_the_default_configuration(f110, dev, kinds, variant):
    kw, configure = {}, None
    if variant == 'env_params':
        def configure(sim):
            p = dict(f110.maps.DEFAULT_PARAMS, mu=0.7, length=0.5, width=0.28)
            sim.update_params(p, env_mask=torch.arange(N) % 2 == 0)
    elif variant == 'euler':
        kw['integrator'] = f110.Integrator.Euler
    elif variant == 'beams270':
        kw['num_beams'] = 270
    elif variant == 'beams2160':
        kw['num_beams'] = 2160
    else:
        kw['fov'] = 2 * np.pi - 1e-3
    for name in ('example_map', 'berlin'):
        twin_run(f110, dev, kinds[name], 5, 2, steps=80, configure=configure, **kw)


def test_repeat_with_noise_runs_plain_ticks(f110, dev, kinds):
    ev = twin_run(f110, dev, kinds['example_map'], 4, 2, steps=100, noise_std=0.01, expect_sub='full')
    assert ev['marched'] == 1.0


def test_huge_finite_poses_are_marched(f110, dev, kinds):
    """Agents at absurd coordinates (the literal march of the tick's kernel) are always listed and change nothing else."""
    for name in ('example_map', 'berlin', 'rotated'):
        dmap, hosts, kind, _ = kinds[name]
        rng = np.random.default_rng(5)
        poses = population(kind, hosts, np.zeros(N, dtype=np.int64), rng, 2)
        poses[::4, :, 0] += 3e9
        a = make_sim(f110, dev, dmap, None, poses, 2)
        b = make_sim(f110, dev, dmap, None, poses, 2)
        for step in range(20):
            act = torch.from_numpy(random_actions(rng, N, 2)).to(dev)
            a.tick_repeat(act, 3)
            for _ in range(3):
                b.tick(act)
            for n in BUFFERS:
                assert same_bits(getattr(a, n), getattr(b, n)), (name, n, step)
        assert a.marched_fraction() >= 0.25


@pytest.mark.parametrize('name', ['example_map', 'berlin', 'rotated'])
def test_repeat_against_the_oracle(f110, dev, kinds, name):
    import oracle
    dmap, hosts, kind, _ = kinds[name]
    K, A, n = 4, 2, 24
    rng = np.random.default_rng(17)
    poses = population(kind, hosts, np.zeros(n, dtype=np.int64), rng, A)
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=n, device=dev)
    sim.set_device_map(dmap)
    sim.env_reset(poses)
    om = rotated.omap_of(hosts[0])
    osims = [oracle.OracleSim(om, num_agents=A) for _ in range(n)]
    for e in range(n):
        osims[e].env_restart(poses[e])
    hits = 0
    for step in range(10):
        act = random_actions(rng, n, A)
        obs = sim.tick_repeat(act, K)
        any_done = np.zeros(n, dtype=bool)
        for _ in range(K):
            oracle.step_batch(osims, act, env_level=True)
            any_done |= oracle.gather(osims, 'done') != 0
        st = sim.state.cpu().numpy().reshape(7, n, A).transpose(1, 2, 0)
        assert np.abs(st - oracle.gather(osims, 'state')).max() < 1e-8, step
        assert np.array_equal(obs['collisions'].cpu().numpy(), oracle.gather(osims, 'collisions')), step
        assert np.array_equal(sim.toggle_list.cpu().numpy().reshape(n, A), oracle.gather(osims, 'toggle_list')), step
        assert np.array_equal(obs['done_any'].cpu().numpy() != 0, any_done), step
        assert np.abs(obs['scans'].cpu().numpy() - oracle.gather(osims, 'scans')).max() < 1e-4, step
        hits += int(oracle.gather(osims, 'in_collision').sum())
    assert hits > 0


def test_graph_replays_equal_eager_calls_and_track_progress(f110, dev, kinds):
    dmap, hosts, kind, _ = kinds['example_map']
    wp = f110.maps.load_waypoints()
    K, A = 4, 2
    rng = np.random.default_rng(23)
    k = rng.integers(0, wp.shape[0], N)
    poses = np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1)
    table = torch.from_numpy(wp).to(dev)
    sims = [make_sim(f110, dev, dmap, None, poses, A) for _ in range(3)]
    for s in sims:
        s.set_centerlines(wp[:, :2])
    g, e, p = sims
    abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
    g.capture_graph(abuf, autoreset_poses=table, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True, progress=True, repeat=K)
    for step in range(60):
        act = torch.from_numpy(random_actions(rng, N, A)).to(dev)
        abuf.copy_(act.reshape(N * A, 2))
        g.replay()
        e.tick_repeat(act, K, autoreset_poses=table, pose_gap=POSE_GAP, seed=AR_SEED, progress=True)
        total = torch.zeros((N * A,), dtype=torch.float64, device=dev)
        for _ in range(K):
            p.tick(act, autoreset_poses=table, pose_gap=POSE_GAP, seed=AR_SEED)
            total = total + p.update_progress()['delta'].reshape(-1)
        for name in BUFFERS + ('track_s', 'track_progress', 'track_seg', 'track_d'):
            assert torch.equal(getattr(g, name), getattr(p, name)), (name, step)
            assert torch.equal(getattr(e, name), getattr(p, name)), (name, step)
        assert torch.equal(g.track_delta_sum, total) and torch.equal(e.track_delta_sum, total), step
        assert torch.equal(g.done_any, e.done_any) and torch.equal(g.done_tick, e.done_tick), step
    assert float(p.track_progress.max()) > 1.0


def test_env_action_repeat_equals_four_steps(f110, dev):
    wp = f110.maps.load_waypoints()
    K, A, n = 4, 2, 32
    kw = dict(map='example_map', map_ext='.png', num_agents=A, num_envs=n, scan_noise_std=0.0, centerline=wp[:, :2],
              reward='progress', device=dev)
    ea, eb = f110.F110Env(action_repeat=K, **kw), f110.F110Env(**kw)
    rng = np.random.default_rng(31)
    k = rng.integers(0, wp.shape[0], n)
    poses = np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1)
    ra, rb = ea.reset(poses), eb.reset(poses)
    assert torch.equal(ra[0]['scans'], rb[0]['scans']) and float(ea.sim.current_time[0]) == pytest.approx(0.01)
    ever_done = False
    for step in range(50):
        act = torch.from_numpy(random_actions(rng, n, A)).to(dev)
        oa, rwa, da, ia = ea.step(act)
        total, dones = torch.zeros((n,), dtype=torch.float64, device=dev), []
        for _ in range(K):
            ob, rwb, db, ib = eb.step(act)
            total = total + rwb
            dones.append(db.clone())
        d = torch.stack(dones)
        for key in ('scans', 'poses_x', 'poses_y', 'poses_theta', 'linear_vels_x', 'ang_vels_z', 'collisions', 'lap_times',
                    'lap_counts', 'track_s', 'progress'):
            assert torch.equal(oa[key], ob[key]), (key, step)
        assert torch.equal(rwa, total) and torch.equal(da, d.any(0)), step
        assert torch.equal(ia['done_tick'], torch.where(d.any(0), d.int().argmax(0), torch.full((n,), -1, device=dev)).int())
        assert torch.equal(ia['checkpoint_done'], ib['checkpoint_done'])
        ever_done |= bool(da.any())
    assert ever_done
    plain = f110.F110Env(action_repeat=3, **dict(kw, centerline=None, reward='timestep'))
    plain.reset(poses)
    assert plain.step(torch.zeros((n, A, 2), dtype=torch.float64, device=dev))[1] == pytest.approx(0.03)
