"""Centerline progress on the H100: f110_track_project equals the reference golden (tests/golden/kat_progress.npz) bit for bit,
and k_track_progress equals the numpy tracker model of tests/test_progress_host.py bit for bit after every tick of

  * a PurePursuitPlanner lap of example_map, its raceline as the centerline (progress at the lap line: L - sqrt(0.1) m);
  * a stack of four generated tracks with per-map auto-reset on random actions (auto-reset agents re-acquire at 0);
  * a synthetic hairpin (two straights 1 m apart: the tracker keeps its branch where the global projection jumps) and a
    teleport beyond reacquire_dist;
plus a CUDA graph against eager ticks, two streams, tick outputs with and without tracking, and F110Env's obs keys and
reward='progress' in batched and single-env modes.
"""
import os

import numpy as np
import pytest
import torch

from test_progress_host import TrackerModel, golden, hairpin, project_model, records

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MAPS = os.path.join(HERE, '..', 'f1tenth_gym_b200', 'maps')
TLAD, VGAIN = 0.82461887897713965, 1.375
POSE_GAP, AR_SEED = 5, 99


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def raceline():
    return np.loadtxt(os.path.join(MAPS, 'example_waypoints.csv'), delimiter=';', skiprows=3)[:, 1:3]


def cpu(t):
    return t.detach().cpu().numpy()


def assert_tracker_equal(sim, model, tag):
    got = {k: cpu(getattr(sim, 'track_' + k)) for k in ('seg', 's', 'd', 'heading_error', 'progress', 'delta')}
    want = {'seg': model.seg, 's': model.s, 'd': model.d, 'heading_error': model.e, 'progress': model.progress,
            'delta': model.delta}
    for k in got:
        assert np.array_equal(got[k].astype(want[k].dtype), want[k], equal_nan=True), (tag, k)


def model_step(sim, model, table_of_agent):
    model.update(cpu(sim.state), cpu(sim.steer_cnt), table_of_agent)


# ----------------------------------------------------------------------------- stateless projection
def test_project_equals_golden(f110, dev):
    g, T = golden()
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 1, device=dev)
    tabs = [g['table_%d' % k] for k in range(T)]
    sim.set_device_map(f110.DeviceMap.stack([f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', dev)] * T),
                       env_map_ids=[0])
    sim.set_centerlines(tabs)
    recs = [records(f110, t) for t in tabs]
    poses = np.concatenate([g['poses_%d' % k] for k in range(T)])
    ids = np.concatenate([np.full(g['poses_%d' % k].shape[0], k) for k in range(T)])
    ids[:7] = [-1, T, 1 << 30, -(1 << 30), T + 5, -2, 2 * T]                # bad table ids: NaN rows
    out = cpu(sim.project_centerline(poses, table_ids=ids))
    want = project_model(recs, poses, np.where((ids >= 0) & (ids < T), ids, -1))
    assert np.array_equal(out, want, equal_nan=True)
    assert np.isnan(out[:7]).all()
    start = 0
    for k in range(T):
        M = g['poses_%d' % k].shape[0]
        ref = g['seg_%d' % k].shape[0]
        o = out[start:start + M]
        lo = 7 if k == 0 else 0
        assert np.array_equal(o[lo:ref, 0].astype(np.int64), g['seg_%d' % k][lo:]), k
        assert np.array_equal(o[lo:ref, 1], g['t_%d' % k][lo:]), k
        assert np.array_equal(np.abs(o[lo:ref, 2]), g['dist_%d' % k][lo:]), k
        assert np.isnan(o[ref:]).all(), k
        start += M
    # a single table needs no ids
    single = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 1, device=dev)
    single.set_centerlines(tabs[0])
    o = cpu(single.project_centerline(g['poses_0']))
    assert np.array_equal(o, project_model(recs[:1], g['poses_0']), equal_nan=True)


def test_two_streams(f110, dev):
    g, _ = golden()
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 1, device=dev)
    sim.set_centerlines(g['table_0'])
    rec = records(f110, g['table_0'])
    rng = np.random.default_rng(4)
    pa = rng.uniform(-60, 60, (50000, 3))
    pb = rng.uniform(-60, 60, (50000, 3))
    da, db = torch.from_numpy(pa).to(dev), torch.from_numpy(pb).to(dev)
    s1, s2 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    torch.cuda.synchronize(dev)
    with torch.cuda.stream(s1):
        oa = sim.project_centerline(da)
    with torch.cuda.stream(s2):
        ob = sim.project_centerline(db)
    torch.cuda.synchronize(dev)
    assert np.array_equal(cpu(oa), project_model([rec], pa), equal_nan=True)
    assert np.array_equal(cpu(ob), project_model([rec], pb), equal_nan=True)


# ----------------------------------------------------------------------------- the tracker
def test_pure_pursuit_lap(f110, dev):
    e = np.load(os.path.join(HERE, 'golden', 'env_laps.npz'))
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 12345, device=dev, noise_std=0.0)
    sim.set_map(os.path.join(MAPS, 'example_map.yaml'), '.png')
    sim.set_centerlines(raceline())
    rec = records(f110, raceline())
    L = rec[-1, 5] + rec[-1, 6]
    model = TrackerModel([rec], 1)
    pl = f110.PurePursuitPlanner(device=dev)
    sim.env_reset(e['pose0'])
    obs = sim.observations()
    tab = np.zeros(1, np.int64)
    at_lap = None
    for t in range(6000):
        obs = sim.step(pl.plan_actions(obs, TLAD, VGAIN))
        sim.env_post_step()
        sim.update_progress()
        model_step(sim, model, tab)
        assert_tracker_equal(sim, model, t)
        if float(sim.lap_counts[0].item()) >= 1:
            at_lap = float(model.progress[0])
            break
    assert at_lap is not None, 'no lap in 6000 ticks'
    assert abs(at_lap - (L - np.sqrt(0.1))) < 0.5, (at_lap, L)
    assert np.abs(model.d[0]) < 1.0


def four_tracks(f110, dev):
    tg = f110.trackgen
    tracks = tg.random_tracks(21, 4)
    stacked, _ = tg.device_maps(tracks, dev)
    tables = [torch.from_numpy(np.stack([t.start_pose(k) for k in range(0, t.waypoints.shape[0], 7)])).to(dev)
              for t in tracks]
    return tracks, stacked, tables


def random_actions(rng, N, A):
    return np.stack([rng.uniform(-0.4189, 0.4189, (N, A)), rng.uniform(0.0, 9.0, (N, A))], axis=2)


def start_on_tracks(tracks, ids, A, rng):
    return np.stack([np.stack([tracks[l].start_pose((k - POSE_GAP * a) % tracks[l].waypoints.shape[0]) for a in range(A)])
                     for l, k in zip(ids, rng.integers(0, 200, len(ids)))])


def test_four_tracks_autoreset(f110, dev):
    tracks, stacked, tables = four_tracks(f110, dev)
    N, A = 96, 2
    ids = np.arange(N) % 4
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 5, num_envs=N, device=dev, noise_std=0.0)
    sim.set_device_map(stacked, env_map_ids=ids)
    sim.set_centerlines([t.waypoints for t in tracks])
    model = TrackerModel([records(f110, t.waypoints) for t in tracks], N * A)
    rng = np.random.default_rng(8)
    sim.env_reset(start_on_tracks(tracks, ids, A, rng))
    tab = np.repeat(ids, A)
    reacquired = tracked = 0
    for t in range(600):
        sim.tick(random_actions(rng, N, A), env_level=True, autoreset_poses=tables, pose_gap=POSE_GAP, seed=AR_SEED)
        sim.update_progress()
        model_step(sim, model, tab)
        assert_tracker_equal(sim, model, t)
        fresh = cpu(sim.steer_cnt) == 0
        assert (model.progress[fresh] == 0).all() and (model.delta[fresh] == 0).all()
        reacquired += int(fresh.sum())
        tracked += int((~fresh).sum())
    assert reacquired > 20 and tracked > 1000, (reacquired, tracked)


def test_hairpin_and_teleport(f110, dev):
    """Agents on the lower straight drift to 0.6 m towards the upper one: the tracker (window 2 back, 4 ahead) stays on its
    branch while the global projection jumps; then a teleport 20 m away re-acquires and keeps the progress."""
    tab = hairpin()
    rec = records(f110, tab)
    N, A = 4, 8
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 1, num_envs=N, device=dev)
    sim.set_centerlines(tab, window=(2, 4))
    model = TrackerModel([rec], N * A, back=2, fwd=4)
    NA = N * A
    x0 = np.linspace(0.3, 5.0, NA)        # up to x = 8 at y = 0.6: the window (seg - 2 .. seg + 4) never reaches y = 1
    tabid = np.zeros(NA, np.int64)

    def place(x, y, yaw, cnt):
        sim.state[0].copy_(torch.from_numpy(x))
        sim.state[1].copy_(torch.from_numpy(y))
        sim.state[4].copy_(torch.from_numpy(yaw))
        sim.steer_cnt.fill_(cnt)
        sim.update_progress()
        model_step(sim, model, tabid)
        assert_tracker_equal(sim, model, (x[0], y[0]))
    yaw = np.zeros(NA)
    place(x0, np.zeros(NA), yaw, 0)
    for k in range(1, 13):
        place(x0 + 0.25 * k, np.full(NA, 0.05 * k), yaw + 0.01 * k, 2)
    glob = project_model([rec], np.stack([x0 + 3.0, np.full(NA, 0.6), yaw], axis=1))
    seg = cpu(sim.track_seg)
    assert (seg < 10).all() and (glob[:, 0] > 10).all()           # the tracker stays on the lower straight, the global jumps
    assert (cpu(sim.track_d) > 0.59).all()
    before = cpu(sim.track_progress).copy()
    place(x0 + 3.0, np.full(NA, -20.0), yaw, 2)                     # teleport beyond reacquire_dist
    assert (cpu(sim.track_progress) != 0).all() and np.array_equal(cpu(sim.track_progress), before + cpu(sim.track_delta))
    bad = x0.copy()
    bad[::3] = np.nan
    place(bad, np.zeros(NA), yaw, 2)                                  # non-finite poses: NaN outputs, seg = -1
    assert (cpu(sim.track_seg)[::3] == -1).all()
    place(x0, np.zeros(NA), yaw, 2)                                   # and they re-acquire at 0
    assert (cpu(sim.track_progress)[::3] == 0).all()
    sim.reset(np.zeros((A, 3)), env_mask=np.array([1, 0, 0, 1], bool))
    assert (cpu(sim.track_seg).reshape(N, A)[[0, 3]] == -1).all() and (cpu(sim.track_seg).reshape(N, A)[[1, 2]] >= 0).all()


def test_graph_equals_eager(f110, dev):
    tracks, stacked, tables = four_tracks(f110, dev)
    N, A = 64, 2
    ids = np.arange(N) % 4
    sims = []
    rng = np.random.default_rng(9)
    poses = start_on_tracks(tracks, ids, A, rng)
    for _ in range(2):
        s = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 5, num_envs=N, device=dev, noise_std=0.0)
        s.set_device_map(stacked, env_map_ids=ids)
        s.set_centerlines([t.waypoints for t in tracks])
        s.env_reset(poses)
        sims.append(s)
    g, e = sims
    abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
    g.capture_graph(abuf, autoreset_poses=tables, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True, progress=True)
    for t in range(300):
        act = torch.from_numpy(random_actions(rng, N, A).reshape(N * A, 2)).to(dev)
        abuf.copy_(act)
        g.replay()
        e.tick(act, env_level=True, autoreset_poses=tables, pose_gap=POSE_GAP, seed=AR_SEED)
        e.update_progress()
        for k in ('state', 'track_seg', 'track_s', 'track_d', 'track_heading_error', 'track_progress', 'track_delta'):
            assert torch.equal(getattr(g, k), getattr(e, k)), (t, k)


def test_tick_outputs_unchanged_by_tracking(f110, dev):
    tracks, stacked, tables = four_tracks(f110, dev)
    N, A = 64, 2
    ids = np.arange(N) % 4
    rng = np.random.default_rng(10)
    poses = start_on_tracks(tracks, ids, A, rng)
    on, off = (f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 5, num_envs=N, device=dev, noise_std=0.0) for _ in range(2))
    for s in (on, off):
        s.set_device_map(stacked, env_map_ids=ids)
        s.env_reset(poses)
    on.set_centerlines([t.waypoints for t in tracks])
    for t in range(200):
        act = random_actions(rng, N, A)
        for s in (on, off):
            s.tick(act, env_level=True, autoreset_poses=tables, pose_gap=POSE_GAP, seed=AR_SEED)
        on.update_progress()
        for k in ('state', 'scans', 'collisions', 'lap_counts', 'lap_times', 'steer_cnt', 'done'):
            assert torch.equal(getattr(on, k), getattr(off, k)), (t, k)


# ----------------------------------------------------------------------------- F110Env
def test_env_progress_batched_and_single(f110, dev):
    e = np.load(os.path.join(HERE, 'golden', 'env_laps.npz'))
    kw = dict(map=os.path.join(MAPS, 'example_map'), map_ext='.png', num_agents=1, scan_noise_std=0.0, device=dev)
    batched = f110.F110Env(num_envs=2, centerline=raceline(), reward='progress', **kw)
    single = f110.F110Env(centerline=np.vstack([raceline()[:-1]]), reward='progress', **kw)
    plain = f110.F110Env(num_envs=2, **kw)
    pose = e['pose0']
    ob, rb, _, _ = batched.reset(np.repeat(pose[None], 2, axis=0))
    os_, rs, _, _ = single.reset(pose)
    op, rp, _, _ = plain.reset(np.repeat(pose[None], 2, axis=0))
    assert rp == 0.01 and 'progress' not in op
    pl = f110.PurePursuitPlanner(device=dev)
    total = 0.0
    kept = []
    for t in range(300):
        act = pl.plan_actions(ob, TLAD, VGAIN)
        ob, rb, _, _ = batched.step(act)
        kept.append((rb, cpu(rb).copy()))
        os_, rs, _, _ = single.step(cpu(act[0]))
        for k in ('track_s', 'track_d', 'track_heading_error', 'progress'):
            assert ob[k].shape == (2, 1) and ob[k].is_cuda
            assert isinstance(os_[k], np.ndarray) and os_[k].shape == (1,)
            assert np.array_equal(cpu(ob[k][0]), os_[k]), (t, k)
        assert rb.shape == (2,) and torch.equal(rb, batched.sim.track_delta.view(2, 1)[:, 0])
        assert isinstance(rs, float) and rs == float(cpu(rb)[0])
        total += rs
    assert total > 5.0 and abs(total - float(os_['progress'][0])) < 1e-9
    assert all(np.array_equal(cpu(r), v) for r, v in kept)           # rewards kept across steps stay as they were
    # update_map without a centerline is refused with reward='progress'; with one, tracking restarts
    with pytest.raises(ValueError):
        batched.update_map(os.path.join(MAPS, 'example_map.yaml'), '.png')
    batched.update_map(os.path.join(MAPS, 'example_map.yaml'), '.png', centerline=raceline())
    assert (batched.sim.track_seg == -1).all()
