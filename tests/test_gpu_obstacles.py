"""Static box obstacles (Simulator.set_obstacles / set_obstacle_draw, C ABI f110_*_obst) on the GPU.

  1. Parked-car parity: K boxes of the car's size equal, for agents 0..A-1, the oracle with A + K agents whose last K sit at the
     boxes' poses under the action (0, 0); step, tick and a captured graph, 200 ticks, with occlusion and contact both seen.
  2. Other sizes: contact changes no state, so a run with boxes has the plain run's state bit for bit; its scans are the plain
     scans clipped by the oracle's ray_cast against each box, its collisions the plain ones ORed with the oracle's GJK, and
     obstacle_hit the highest touching slot.
  3. Absent = off: slots that are inactive, not finite or of size 0 give every buffer of the plain run, on one map and a stack.
  4. Respawn: under a captured graph with auto-reset, exactly the restarted envs get new boxes, those of the numpy draw.
  5. Repeat: tick_repeat(a, 4) with boxes leaves every buffer as four obstacle ticks do.
  6. Errors: every rejected struct returns F110_ERR_INVALID before anything is enqueued; the host paths refuse obstacles.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from test_gpu_scale import AR_SEED, POSE_GAP, TOL_OCCLUDED, TOL_STATE, random_actions

pytestmark = pytest.mark.gpu

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
CAR = (0.58, 0.31)        # DEFAULT_PARAMS length, width


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def example_map(f110, dev):
    return f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', dev)


def cpu(t):
    return t.detach().cpu().numpy()


def raceline_setup(f110, rng, N, A, K):
    """Agents on the raceline (gap 3 waypoints), boxes on it ahead of agent 0 (first one 8-14 waypoints ahead, then every 5)."""
    wp = f110.maps.load_waypoints()
    n = wp.shape[0]
    k = rng.integers(0, n, N)
    poses = np.stack([wp[(k - 3 * i) % n] for i in range(A)], axis=1)
    ahead = k + rng.integers(8, 15, N)
    boxes = np.stack([wp[(ahead + 5 * j) % n] for j in range(K)], axis=1)
    # the yaw as the dynamics' single-shot wrap leaves it (a parked agent of the oracle holds its yaw from the first step on)
    boxes[:, :, 2] = np.where(boxes[:, :, 2] < 0, boxes[:, :, 2] + 2 * np.pi, boxes[:, :, 2])
    boxes = np.concatenate([boxes, np.broadcast_to(np.array(CAR), (N, K, 2))], axis=2)
    return poses, boxes


def make_sim(f110, dev, dmap, poses, ids=None, **kw):
    N, A = poses.shape[:2]
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=N, device=dev, **kw)
    sim.set_device_map(dmap, env_map_ids=ids)
    sim.env_reset(poses)
    return sim


# ----------------------------------------------------------------------------- 1. parked-car parity
@pytest.mark.parametrize('drive', ['step', 'tick', 'graph'])
@pytest.mark.parametrize('K', [1, 3])
@pytest.mark.parametrize('A', [1, 2])
def test_parked_car_parity(f110, dev, example_map, A, K, drive):
    import oracle
    N, T = 24, 200
    rng = np.random.default_rng(100 * A + 10 * K + len(drive))
    poses, boxes = raceline_setup(f110, rng, N, A, K)
    sim = make_sim(f110, dev, example_map, poses)
    sim.set_obstacles(boxes)
    h = example_map.host
    omap = oracle.OracleMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.0))
    osims = [oracle.OracleSim(omap, num_agents=A + K) for _ in range(N)]
    for e in range(N):
        osims[e].env_restart(np.concatenate([poses[e], boxes[e, :, :3]]))
    if drive == 'graph':
        abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
        sim.capture_graph(abuf)
    n_occ = n_contact = 0
    for t in range(T):
        act = random_actions(rng, N, A)
        act[:, :, 1] = rng.uniform(0, 4, (N, A))        # slow enough to meet the boxes rather than fly past them
        if drive == 'graph':
            abuf.copy_(torch.from_numpy(act.reshape(N * A, 2)))
            sim.replay()
        elif drive == 'tick':
            sim.tick(act, env_level=False)
        else:
            sim.step(act)
        torch.cuda.synchronize()
        oracle.step_batch(osims, np.concatenate([act, np.zeros((N, K, 2))], axis=1))
        where = (drive, A, K, t)
        got = cpu(sim.scans).reshape(N, A, -1)
        fin, pre = oracle.gather(osims, 'scans')[:, :A], oracle.gather(osims, 'scans_pre')[:, :A]
        occ = fin < pre
        assert not ((~occ) & (got != fin.astype(np.float32))).any(), (where, 'scan')
        assert np.where(occ, np.abs(got - fin), 0.0).max() <= TOL_OCCLUDED, (where, 'occluded beams')
        n_occ += int(occ.sum())
        col, cidx = oracle.gather(osims, 'collisions')[:, :A], oracle.gather(osims, 'collision_idx')[:, :A]
        assert np.array_equal(cpu(sim.collisions).reshape(N, A), col), (where, 'collisions')
        assert np.array_equal(cpu(sim.collision_idx).reshape(N, A).astype(np.float64), cidx), (where, 'collision_idx')
        n_contact += int((cidx >= A).sum())
        st = cpu(sim.state).reshape(7, N, A).transpose(1, 2, 0)
        assert np.abs(st - oracle.gather(osims, 'state')[:, :A]).max() <= TOL_STATE, (where, 'state')
        # the parked agents of the oracle never move
        assert np.array_equal(oracle.gather(osims, 'state')[:, A:][:, :, [0, 1, 4]], boxes[:, :, :3]), (where, 'parked')
    print('occluded beams', n_occ, 'box contacts', n_contact)
    assert n_occ > 0 and n_contact > 0


# ----------------------------------------------------------------------------- 2. other sizes
def test_other_sizes_against_plain_run_and_oracle(f110, dev, example_map):
    import oracle
    N, A, K, T = 12, 2, 4, 120
    rng = np.random.default_rng(7)
    poses, boxes = raceline_setup(f110, rng, N, A, K)
    boxes[:, :, 3] = rng.uniform(0.2, 2.5, (N, K))
    boxes[:, :, 4] = rng.uniform(0.1, 1.2, (N, K))
    boxes[:, :, 2] += rng.uniform(-1.0, 1.0, (N, K))
    active = rng.random((N, K)) < 0.8
    plain = make_sim(f110, dev, example_map, poses)
    obst = make_sim(f110, dev, example_map, poses)
    obst.set_obstacles(boxes, active)
    angles = cpu(plain.beams.scan_angles)
    L, W = CAR
    n_occ = n_contact = 0
    for t in range(T):
        act = random_actions(rng, N, A)
        act[:, :, 1] = rng.uniform(0, 4, (N, A))
        plain.tick(act, env_level=False)
        obst.tick(act, env_level=False)
        torch.cuda.synchronize()
        for name in ('state', 'agent_poses', 'wall_flag', 'steer_buf'):
            assert torch.equal(getattr(plain, name), getattr(obst, name)), (t, name)
        ps, gs = cpu(plain.scans).reshape(N, A, -1), cpu(obst.scans).reshape(N, A, -1)
        pc, gc = cpu(plain.collisions).reshape(N, A), cpu(obst.collisions).reshape(N, A)
        pi, gi = cpu(plain.collision_idx).reshape(N, A), cpu(obst.collision_idx).reshape(N, A)
        hit = cpu(obst.obstacle_hit).reshape(N, A)
        ap, wall = cpu(plain.agent_poses).reshape(N, A, 5), cpu(plain.wall_flag).reshape(N, A)
        for e in range(N):
            for i in range(A):
                pose = np.array([ap[e, i, 0], ap[e, i, 1], 0.0 if wall[e, i] else ap[e, i, 2]])
                want = ps[e, i].copy()
                top = -1
                va = oracle.get_vertices(ap[e, i, :3], L, W)
                for k in range(K):
                    if not active[e, k]:
                        continue
                    vb = oracle.get_vertices(boxes[e, k, :3], boxes[e, k, 3], boxes[e, k, 4])
                    r = oracle.ray_cast(pose, np.full(want.shape, np.inf), angles, vb).astype(np.float32)
                    want = np.minimum(want, r)
                    if oracle.collision(va, vb):
                        top = k
                # (a beam that grazes a box edge may fall either side of it: the tolerance of the opponent ray-cast)
                assert np.abs(gs[e, i].astype(np.float64) - want).max() <= TOL_OCCLUDED, (t, e, i, 'scan')
                assert (gs[e, i] <= ps[e, i]).all(), (t, e, i, 'a box lengthened a beam')
                n_occ += int((want < ps[e, i]).sum())
                assert hit[e, i] == top, (t, e, i, 'hit')
                assert gc[e, i] == (1.0 if (pc[e, i] or top >= 0) else 0.0), (t, e, i, 'collisions')
                assert gi[e, i] == (max(pi[e, i], A + top) if top >= 0 else pi[e, i]), (t, e, i, 'collision_idx')
                n_contact += int(top >= 0)
    print('clipped beams', n_occ, 'contacts', n_contact)
    assert n_occ > 0 and n_contact > 0


# ----------------------------------------------------------------------------- 3. absent = off
BUFFERS = ('state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'wall_flag', 'collisions', 'collision_idx', 'scans',
           'current_time', 'lap_times', 'lap_counts', 'toggle_list', 'near_starts', 'start_xs', 'start_ys', 'start_thetas',
           'start_rot', 'done', 'checkpoint_done', 'tick_counter')


def absent_boxes(rng, N, K, poses):
    """Boxes right on the agents that must count as absent: every env's slots inactive, non-finite or of size <= 0."""
    b = np.zeros((N, K, 5))
    b[:, :, :3] = poses[:, :1, :]
    b[:, :, 3:] = CAR
    active = np.ones((N, K), bool)
    kind = np.arange(N * K).reshape(N, K) % 6
    active[kind == 0] = False
    b[kind == 1, 0] = np.nan
    b[kind == 2, 2] = np.inf
    b[kind == 3, 3] = 0.0
    b[kind == 4, 4] = -0.3
    b[kind == 5, 3] = np.nan
    return b, active


@pytest.mark.parametrize('stack', [False, True])
@pytest.mark.parametrize('drive', ['tick', 'graph'])
def test_absent_slots_equal_the_plain_tick(f110, dev, example_map, stack, drive):
    from test_gpu_multimap import TRACKS, mixed_population, start_table
    N, A, K, T = 48, 2, 6, 80
    rng = np.random.default_rng(11)
    if stack:
        maps = [f110.DeviceMap.from_yaml(os.path.join(MAPS, n + '.yaml'), e, dev) for n, e in TRACKS]
        dmap = f110.DeviceMap.stack(maps)
        ids = np.arange(N) % len(maps)
        poses = mixed_population([m.host for m in maps], ids, rng, A)
        tabs = [torch.from_numpy(np.ascontiguousarray(start_table(m.host, rng))).to(dev) for m in maps]
    else:
        dmap, ids = example_map, None
        poses, _ = raceline_setup(f110, rng, N, A, 1)
        tabs = torch.from_numpy(f110.maps.load_waypoints()).to(dev)
    a = make_sim(f110, dev, dmap, poses, ids)
    b = make_sim(f110, dev, dmap, poses, ids)
    bx, act_mask = absent_boxes(rng, N, K, poses)
    b.set_obstacles(bx, act_mask)
    if drive == 'graph':
        bufs = [torch.zeros((N * A, 2), dtype=torch.float64, device=dev) for _ in range(2)]
        a.capture_graph(bufs[0], autoreset_poses=tabs, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True)
        b.capture_graph(bufs[1], autoreset_poses=tabs, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True)
    resets = 0
    for t in range(T):
        act = random_actions(rng, N, A)
        if drive == 'graph':
            for buf in bufs:
                buf.copy_(torch.from_numpy(act.reshape(N * A, 2)))
            a.replay(), b.replay()
        else:
            a.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
            b.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        for name in BUFFERS:
            assert torch.equal(getattr(a, name), getattr(b, name)), (t, name)
        assert (b.obstacle_hit == -1).all()
        resets += int(a.done.sum())
    assert resets > 0


# ----------------------------------------------------------------------------- 4. respawn
@pytest.mark.parametrize('layers', [1, 2])
def test_respawn_under_graph_matches_numpy_draw(f110, dev, example_map, layers):
    from f1tenth_gym_b200.obstacles import respawn_draw
    N, A, K, T = 64, 2, 6, 150
    COUNT, CLR, SEED = (1, 5), 1.5, 99
    rng = np.random.default_rng(21 + layers)
    wp = f110.maps.load_waypoints()
    if layers == 1:
        dmap, ids = example_map, None
        cands = [f110.obstacle_candidates(wp[:, :2], 200, lateral=(-0.6, 0.6), seed=5)]
    else:
        dmap = f110.DeviceMap.stack([example_map, f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', dev)])
        ids = np.arange(N) % 2
        cands = [f110.obstacle_candidates(wp[:, :2], 200, lateral=(-0.6, 0.6), seed=5),
                 f110.obstacle_candidates(wp[:, :2], 77, lateral=(-1.0, 0.2), size=(0.4, 0.4), seed=6)]
    poses, boxes = raceline_setup(f110, rng, N, A, K)
    sim = make_sim(f110, dev, dmap, poses, ids)
    sim.set_obstacles(boxes)
    sim.set_obstacle_draw(cands if layers > 1 else cands[0], count=COUNT, clearance=CLR, seed=SEED)
    tab = torch.from_numpy(wp).to(dev)
    abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
    sim.capture_graph(abuf, autoreset_poses=[tab] * layers if layers > 1 else tab, pose_gap=POSE_GAP,
                      autoreset_seed=AR_SEED, env_level=True)
    layer = np.zeros(N, int) if ids is None else ids
    resets = inactive_by_clearance = 0
    for t in range(T):
        before_b, before_a = cpu(sim.obstacle_boxes), cpu(sim.obstacle_active)
        abuf.copy_(torch.from_numpy(random_actions(rng, N, A).reshape(N * A, 2)))
        sim.replay()
        tick = int(sim.tick_counter.item())
        reset = cpu(sim.collisions).reshape(N, A)[:, 0] != 0
        bx, ac = cpu(sim.obstacle_boxes), cpu(sim.obstacle_active)
        xy = cpu(sim.state).reshape(7, N, A)[[0, 1]].transpose(1, 2, 0)
        assert np.array_equal(bx[~reset], before_b[~reset]) and np.array_equal(ac[~reset], before_a[~reset]), t
        for e in np.flatnonzero(reset):
            wb, wa = respawn_draw(cands[layer[e]], xy[e], K, COUNT, CLR, SEED, tick, int(e))
            assert np.array_equal(bx[e], wb) and np.array_equal(ac[e], wa), (t, e)
            d2 = ((bx[e, :, None, :2] - xy[e][None]) ** 2).sum(-1)
            assert (d2[ac[e].astype(bool)] >= CLR * CLR).all(), (t, e)
            inactive_by_clearance += int((d2.min(1) < CLR * CLR).sum())
        resets += int(reset.sum())
    print('resets', resets, 'slots kept inactive by the clearance', inactive_by_clearance)
    assert resets > 0


def test_host_respawn(f110, dev, example_map):
    from f1tenth_gym_b200.obstacles import respawn_draw
    N, A, K = 16, 1, 4
    rng = np.random.default_rng(3)
    poses, boxes = raceline_setup(f110, rng, N, A, K)
    sim = make_sim(f110, dev, example_map, poses)
    sim.set_obstacles(boxes)
    cand = f110.obstacle_candidates(f110.maps.load_waypoints()[:, :2], 50, seed=1)
    sim.set_obstacle_draw(cand, count=(2, 4), clearance=0.8, seed=4)
    mask = np.arange(N) % 2 == 0
    sim.respawn_obstacles(mask)
    bx, ac = cpu(sim.obstacle_boxes), cpu(sim.obstacle_active)
    for e in range(N):
        if mask[e]:
            wb, wa = respawn_draw(cand, poses[e, :, :2], K, (2, 4), 0.8, 4, 0, e)
            assert np.array_equal(bx[e], wb) and np.array_equal(ac[e], wa)
        else:
            assert np.array_equal(bx[e], boxes[e]) and ac[e].all()


# ----------------------------------------------------------------------------- 5. repeat
def test_repeat_equals_obstacle_ticks(f110, dev, example_map):
    N, A, K, R, STEPS = 64, 2, 4, 4, 60
    rng = np.random.default_rng(5)
    poses, boxes = raceline_setup(f110, rng, N, A, K)
    cand = f110.obstacle_candidates(f110.maps.load_waypoints()[:, :2], 100, seed=2)
    sims = [make_sim(f110, dev, example_map, poses) for _ in range(2)]
    for s in sims:
        s.set_obstacles(boxes)
        s.set_obstacle_draw(cand, count=(1, 4), clearance=1.0, seed=8)
    a, b = sims
    tab = torch.from_numpy(f110.maps.load_waypoints()).to(dev)
    contacts = 0
    for step in range(STEPS):
        act = torch.from_numpy(random_actions(rng, N, A)).to(dev)
        obs = a.tick_repeat(act, R, autoreset_poses=tab, pose_gap=POSE_GAP, seed=AR_SEED)
        dones = []
        for _ in range(R):
            b.tick(act, autoreset_poses=tab, pose_gap=POSE_GAP, seed=AR_SEED)
            dones.append(b.done.clone())
            contacts += int((b.collision_idx >= A).sum())
        for name in BUFFERS + ('obstacle_boxes', 'obstacle_active', 'obstacle_hit'):
            assert torch.equal(getattr(a, name), getattr(b, name)), (name, step)
        d = torch.stack(dones).bool()
        first = torch.where(d.any(0), d.int().argmax(0), torch.full((N,), -1, device=dev)).int()
        assert torch.equal(obs['done_any'].bool(), d.any(0)) and torch.equal(obs['done_tick'], first), step
    assert contacts > 0


# ----------------------------------------------------------------------------- 6. errors
def test_rejected_structs_enqueue_nothing(f110, dev, example_map):
    from test_obstacles_host import obstacle_struct_cases
    nat = f110._native
    L = nat.lib()
    N, A = 4, 2
    poses, boxes = raceline_setup(f110, np.random.default_rng(0), N, A, 2)
    sim = make_sim(f110, dev, example_map, poses)
    sim.set_obstacles(boxes)
    p = nat.ptr(sim.obstacle_boxes)
    offs_buf = (ctypes.c_int32 * 3)(0, 3, 9)
    a = nat.ptr(sim._actions_dev)
    before = {n: getattr(sim, n).clone() for n in BUFFERS}
    cases = obstacle_struct_cases(nat, p, ctypes.addressof(offs_buf))
    # per-layer tables on a single map
    cases.append(('tables vs layers', nat.F110Obstacles(4, p, p, None, p, ctypes.addressof(offs_buf), 9, 2, 0, 1, 0.0, 0)))
    sim.c.env_layer = nat.ptr(sim.steer_cnt)       # (any device buffer: the check fires before it is read)
    for name, o in cases:
        args = (ctypes.byref(sim.c), ctypes.byref(sim._map_struct), ctypes.byref(sim._march_tables), ctypes.byref(sim.beams.c), a)
        assert L.f110_step_obst(*args, ctypes.byref(o), None) == -1, name
        assert L.f110_tick_obst(*args, 1, None, 0, 0, 0, ctypes.byref(o), None) == -1, name
        assert L.f110_tick_repeat_ticks_obst(*args, 2, 0, 2, ctypes.byref(sim._repeat_struct()), 1, None, 0, 0, 0,
                                             ctypes.byref(o), None) == -1, name
    sim.c.env_layer = None
    torch.cuda.synchronize()
    for n in BUFFERS:
        assert torch.equal(before[n], getattr(sim, n)), n
    # positive control: the same arguments with the simulator's own (valid) struct run
    args = (ctypes.byref(sim.c), ctypes.byref(sim._map_struct), ctypes.byref(sim._march_tables), ctypes.byref(sim.beams.c), a)
    ok = ctypes.byref(sim._obst)
    assert L.f110_step_obst(*args, ok, None) == 0
    assert L.f110_tick_obst(*args, 1, None, 0, 0, 0, ok, None) == 0
    assert L.f110_tick_repeat_ticks_obst(*args, 2, 0, 2, ctypes.byref(sim._repeat_struct()), 1, None, 0, 0, 0, ok, None) == 0
    ids = torch.arange(N * A, dtype=torch.int32, device=dev)
    out = torch.empty((N * A, 8, 8), dtype=torch.uint8, device=dev)
    for name, o in cases[:-1]:
        assert L.f110_render_views_obst(ctypes.byref(sim.c), ctypes.byref(sim._map_struct), ctypes.byref(o), nat.ptr(ids), N * A,
                                        8, 8, 0.1, 0.0, 0, nat.ptr(out), None) == -1, name
    assert L.f110_render_views_obst(ctypes.byref(sim.c), ctypes.byref(sim._map_struct), ok, nat.ptr(ids), N * A, 8, 8, 0.1, 0.0,
                                    0, nat.ptr(out), None) == 0
    torch.cuda.synchronize()
    assert int(sim.tick_counter.item()) == int(before['tick_counter'].item()) + 4
    # the host-buffer and profiling paths refuse obstacles
    with pytest.raises(ValueError):
        sim.step_host(sim.make_host_io())
    with pytest.raises(ValueError):
        sim.step_profile(np.zeros((N, A, 2)))
    with pytest.raises(ValueError):
        sim.step_host_async(sim.make_host_pipeline(1)[0])
    sim.clear_obstacles()
    sim.step_profile(np.zeros((N, A, 2)))


def test_simulator_argument_validation(f110, dev, example_map):
    N, A = 3, 1
    poses, boxes = raceline_setup(f110, np.random.default_rng(0), N, A, 2)
    sim = make_sim(f110, dev, example_map, poses)
    for bad in (np.zeros((0, 5)), np.zeros((17, 5)), np.zeros((2, 4)), np.zeros((N + 1, 2, 5))):
        with pytest.raises(ValueError):
            sim.set_obstacles(bad)
    with pytest.raises(ValueError):
        sim.set_obstacles(boxes, active=np.ones(3, bool))
    with pytest.raises(ValueError):
        sim.set_obstacle_draw(np.zeros((3, 5)))              # before set_obstacles
    with pytest.raises(ValueError):
        sim.respawn_obstacles()
    sim.set_obstacles(boxes)
    cand = np.tile(np.array([[0.0, 0.0, 0.0, 0.58, 0.31]]), (3, 1))
    for kw in (dict(count=(2, 1)), dict(count=(0, 3)), dict(count=(-1, 1)), dict(clearance=-1.0), dict(clearance=np.inf)):
        with pytest.raises(ValueError):
            sim.set_obstacle_draw(cand, **kw)
    for bad in (np.zeros((0, 5)), np.full((2, 5), np.nan), [cand, cand]):       # a list needs a stacked map
        with pytest.raises(ValueError):
            sim.set_obstacle_draw(bad)
    sim.set_obstacle_draw(cand, count=(0, 2))
    assert sim.obstacle_boxes.shape == (N, 2, 5) and sim.obstacle_active.shape == (N, 2) and sim.obstacle_hit.shape == (N * A,)


# ----------------------------------------------------------------------------- 7. views and F110Env
def near_boxes(rng, poses, K):
    """K boxes 0.8-2.5 m around agent 0 of each env, random yaw and size."""
    N = poses.shape[0]
    r, th = rng.uniform(0.8, 2.5, (N, K)), rng.uniform(0, 2 * np.pi, (N, K))
    return np.stack([poses[:, :1, 0] + r * np.cos(th), poses[:, :1, 1] + r * np.sin(th), rng.uniform(-4, 4, (N, K)),
                     rng.uniform(0.2, 1.0, (N, K)), rng.uniform(0.1, 0.6, (N, K))], axis=2)


def test_views_draw_obstacles(f110, dev, example_map):
    import oracle
    from test_views_host import in_car, pixel_centres
    N, A, K, H, W, S = 6, 2, 5, 96, 96, 0.05
    rng = np.random.default_rng(9)
    poses, _ = raceline_setup(f110, rng, N, A, 1)
    boxes = near_boxes(rng, poses, K)
    active = np.ones((N, K), bool)
    active[:, 1] = False
    boxes[::2, 2, 0] = np.nan                                           # absent: not finite
    sim = make_sim(f110, dev, example_map, poses)
    ref = cpu(sim.render_views(None, (H, W), S, 0.0, heading_up=False))
    sim.set_obstacles(boxes, np.zeros((N, K), bool))
    assert np.array_equal(cpu(sim.render_views(None, (H, W), S, 0.0, heading_up=False)), ref)     # no box present: unchanged
    sim.set_obstacles(boxes, active)
    for heading_up in (False, True):
        sim.obstacle_active.zero_()
        ref = cpu(sim.render_views(None, (H, W), S, 0.3, heading_up=heading_up))
        sim.obstacle_active.copy_(torch.from_numpy(active.astype(np.uint8)))
        got = cpu(sim.render_views(None, (H, W), S, 0.3, heading_up=heading_up))
        st = cpu(sim.state).reshape(7, N * A)
        n5 = 0
        for v in range(N * A):
            e = v // A
            yaw = st[4, v]
            px, py = pixel_centres(st[0, v], st[1, v], np.cos(yaw), np.sin(yaw), H, W, S, 0.3, heading_up)
            # (pixels within 1e-9 of a box edge may fall either side: the vertices and the heading-up pixel centres come from
            # numpy's cos / sin here and the device's sincos there)
            inside, near = np.zeros((H, W), bool), np.zeros((H, W), bool)
            for k in range(K):
                b = boxes[e, k]
                if not (active[e, k] and np.isfinite(b).all()):
                    continue
                vb = oracle.get_vertices(b[:3], b[3], b[4])
                inside |= in_car(px, py, vb)
                for q in range(4):
                    a0, a1 = vb[q], vb[(q + 1) % 4]
                    near |= np.abs((a1[0] - a0[0]) * (py - a0[1]) - (a1[1] - a0[1]) * (px - a0[0])) < 1e-9
            car = (got[v] == 3) | (got[v] == 4)
            ok = ((got[v] == 5) == (inside & ~car)) | near
            assert ok.all(), (heading_up, v, np.argwhere(~ok)[:5])
            assert np.array_equal(got[v][got[v] != 5], ref[v][got[v] != 5]), (heading_up, v)
            assert not ((got[v] == 5) & (ref[v] >= 3)).any()             # a car wins over a box
            n5 += int((got[v] == 5).sum())
        assert n5 > 0, heading_up


def test_env_obstacles(f110, dev, example_map):
    from f1tenth_gym_b200.env import RENDER_PALETTE
    from f1tenth_gym_b200.obstacles import respawn_draw
    N, A, K = 4, 2, 3
    rng = np.random.default_rng(4)
    poses, _ = raceline_setup(f110, rng, N, A, 1)
    cand = near_boxes(rng, poses[:1], 12)[0]
    cfg = {'candidates': cand, 'count': (2, K), 'clearance': 0.7, 'seed': 31}
    env = f110.F110Env(map='example_map', map_ext='.png', num_agents=A, num_envs=N, scan_noise_std=0.0,
                       obstacles=cfg, device=dev)
    obs, _, _, _ = env.reset(poses)
    assert obs['obstacles'].data_ptr() == env.sim.obstacle_boxes.data_ptr() and obs['obstacles'].shape == (N, K, 5)
    assert obs['obstacle_active'].shape == (N, K)
    for e in range(N):
        wb, wa = respawn_draw(cand, poses[e, :, :2], K, (2, K), 0.7, 31, 0, e)
        assert np.array_equal(cpu(obs['obstacles'][e]), wb) and np.array_equal(cpu(obs['obstacle_active'][e]), wa), e
    obs, _, _, _ = env.step(np.zeros((N, A, 2)))
    assert 'obstacles' in obs and 'obstacle_active' in obs
    before = cpu(env.sim.obstacle_boxes).copy()
    tick = int(env.sim.tick_counter.item())
    mask = np.array([False, True, False, True])
    env.reset_envs(mask, poses)
    bx, ac = cpu(env.sim.obstacle_boxes), cpu(env.sim.obstacle_active)
    for e in range(N):
        if mask[e]:
            wb, wa = respawn_draw(cand, poses[e, :, :2], K, (2, K), 0.7, 31, tick, e)
            assert np.array_equal(bx[e], wb) and np.array_equal(ac[e], wa), e
        else:
            assert np.array_equal(bx[e], before[e]), e
    # rgb_array applies the palette to the class view, class 5 included
    rgb = env.render('rgb_array', env_ids=[0, 1, 2, 3], size=(160, 160), metres_per_pixel=0.05)
    cls = env.sim.render_views(torch.arange(N, dtype=torch.int32, device=dev) * A, (160, 160), 0.05, 0.0, heading_up=False)
    assert (cls == 5).any()
    assert np.array_equal(cpu(rgb), RENDER_PALETTE[cpu(cls)])
    assert tuple(RENDER_PALETTE[5]) != tuple(RENDER_PALETTE[1])
