"""k_render_views (f110_render_views, csrc/render.cuh) on the H100: every view equals the numpy model of
tests/test_views_host.py byte for byte, fed with the device state, the device's cos / sin of the yaw and car quads from
f110_get_vertices.

  * each bundled map alone; a same-size stack, the berlin / vegas / skirk / levine canvas, the six-map mixed-resolution stack, a
    rotated single map, the rot4 stack and generated tracks with berlin; heading-up and world-aligned, forward offsets, odd
    sizes and 1 x 1 views;
  * the state after 50 pure-pursuit ticks with two agents, two cars overlapping;
  * 1 x 1 views (pixel centre = the agent's (x, y)) at the boundary builders, agents placed there with Simulator.reset;
  * invalid views (bad ids, bad layers, NaN poses: all 255) and poses at 1e12 (no map cell);
  * ticks interleaved with views equal ticks without them; a CUDA graph of render_views(out=...) equals eager calls;
  * F110Env: rgb_array is the palette applied to the classes, local_map equals render_views, render('human') raises.
"""
import os

import numpy as np
import pytest
import torch

from test_multimap_host import MAPS, TRACKS
from test_rotated_host import rotated_probe_points
from test_views_host import SIX, layer_tables, model_flat, agrees, oracle_cells, views_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def load(f110, dev, name, ext, yaw=None):
    m = f110.DeviceMap.from_yaml(os.path.join(MAPS, name + '.yaml'), ext, dev)
    if yaw is None:
        return m
    h = m.host
    return f110.DeviceMap(f110.maps.HostMap(h.dt, h.resolution, (h.orig_x, h.orig_y, yaw)), dev)


@pytest.fixture(scope='module')
def six(f110, dev):
    return [load(f110, dev, n, e) for n, e in SIX]


def make_sim(f110, dev, dmap, N, A, ids=None):
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 7, num_envs=N, device=dev, noise_std=0.0)
    sim.set_device_map(dmap, env_map_ids=ids)
    return sim


def on_map_poses(hosts, layer_of_env, A, rng, spread=0.0):
    """(N, A, 3) poses: free cells of each env's own map (and a few walls and off-map points), random yaws."""
    N = len(layer_of_env)
    out = np.empty((N, A, 3))
    for e in range(N):
        h = hosts[layer_of_env[e]]
        for a in range(A):
            u = rng.random()
            if u < 0.7:
                r, c = np.argwhere(h.dt > 0.3)[rng.integers(0, int((h.dt > 0.3).sum()))]
            elif u < 0.85:
                r, c = np.argwhere(h.dt == 0)[rng.integers(0, int((h.dt == 0).sum()))]
            else:
                r, c = rng.integers(-20, h.height + 20), rng.integers(-20, h.width + 20)
            x, y = (c + rng.random()) * h.resolution, (r + rng.random()) * h.resolution
            cs, sn = h.orig_c, h.orig_s
            out[e, a] = (h.orig_x + cs * x - sn * y, h.orig_y + sn * x + cs * y, rng.uniform(-np.pi, np.pi))
    return out


def model_of(f110, sim, agent_ids, size, s, f, heading_up):
    """views_model on the simulator's device state."""
    NA = sim.num_envs * sim.num_agents
    st = sim.state
    cos_sin = torch.stack([torch.cos(st[4]), torch.sin(st[4])], dim=1).cpu().numpy()
    poses = torch.stack([st[0], st[1], st[4]], dim=1).contiguous()
    verts = f110.kernels.get_vertices(poses, sim.c.sim_length, sim.c.sim_width).cpu().numpy()
    env_layer = sim.env_layer.cpu().numpy() if sim.env_layer is not None else None
    ids = np.arange(NA) if agent_ids is None else np.asarray(agent_ids)
    return views_model(layer_tables(sim.map), st.cpu().numpy(), cos_sin, verts, env_layer, sim.num_agents, ids, size[0],
                       size[1], s, f, heading_up)


SETTINGS = [((64, 64), 0.1, 0.0, True), ((37, 53), 0.05, 1.5, False), ((31, 20), 0.25, -2.0, True), ((1, 1), 0.1, 0.0, True),
            ((128, 96), 0.5, 3.0, False)]


def check_all_settings(f110, sim, ids=None):
    torch.cuda.synchronize()
    for size, s, f, hu in SETTINGS:
        got = sim.render_views(ids, size, s, f, hu).cpu().numpy()
        want = model_of(f110, sim, ids, size, s, f, hu)
        bad = np.argwhere(got != want)
        assert bad.size == 0, (size, s, f, hu, bad[:5], got[tuple(bad[0])], want[tuple(bad[0])])
        assert set(np.unique(got)) - {0, 1, 2, 3, 4} == set()


@pytest.mark.parametrize('k', range(6))
def test_each_bundled_map(f110, dev, six, k):
    N, A = 6, 2
    sim = make_sim(f110, dev, six[k], N, A)
    sim.reset(on_map_poses([six[k].host], [0] * N, A, np.random.default_rng(10 + k)))
    check_all_settings(f110, sim)


@pytest.fixture(scope='module')
def stacks(f110, dev, six):
    from f1tenth_gym_b200 import trackgen as tg
    b = six[0].host
    flipped = f110.DeviceMap(f110.maps.HostMap(np.ascontiguousarray(b.dt[::-1, ::-1]), b.resolution,
                                               (b.orig_x, b.orig_y, 0.0)), dev)
    rot4 = [load(f110, dev, n, e, yaw) for (n, e), yaw in zip(TRACKS, (0.35, -0.8, 1.9, 3.0))]
    gen = [tg.device_map(t, dev) for t in tg.random_tracks(5, 2)]
    gen_hosts = [f110.maps.HostMap(m.dt.cpu().numpy(), m.host.resolution, (m.host.orig_x, m.host.orig_y, 0.0)) for m in gen]
    rot_single = load(f110, dev, 'berlin', '.png', 0.35)
    return {'same_size': (f110.DeviceMap.stack([six[0], flipped]), [b, flipped.host]),
            'canvas4': (f110.DeviceMap.stack(six[:4]), [m.host for m in six[:4]]),
            'mixres6': (f110.DeviceMap.stack(six, mixed_resolution=True), [m.host for m in six]),
            'rot_single': (rot_single, [rot_single.host]),
            'rot4': (f110.DeviceMap.stack(rot4, rotated_origins=True), [m.host for m in rot4]),
            'trackgen_berlin': (f110.DeviceMap.stack(gen + [six[0]], mixed_resolution=True), gen_hosts + [b])}


@pytest.mark.parametrize('kind', ['same_size', 'canvas4', 'mixres6', 'rot_single', 'rot4', 'trackgen_berlin'])
def test_stacks_and_rotated_maps(f110, dev, stacks, kind):
    dmap, hosts = stacks[kind]
    L = len(hosts)
    N, A = 3 * L, 2
    ids = np.arange(N) % L
    sim = make_sim(f110, dev, dmap, N, A, ids if L > 1 else None)
    sim.reset(on_map_poses(hosts, ids, A, np.random.default_rng(20)))
    check_all_settings(f110, sim)
    # a subset of views in any order, with repeats
    sub = [5, 0, 5, N * A - 1, 2]
    got = sim.render_views(sub, (16, 24), 0.2, 0.5, True).cpu().numpy()
    assert np.array_equal(got, model_of(f110, sim, sub, (16, 24), 0.2, 0.5, True))


def test_after_pure_pursuit_ticks_with_overlapping_cars(f110, dev, six):
    """50 ticks of pure pursuit on example_map, 2 agents; in env 0 the two cars start 0.1 m apart (overlapping)."""
    em = six[5]
    N, A = 8, 2
    wp = f110.maps.load_waypoints()
    rng = np.random.default_rng(30)
    ks = rng.integers(0, wp.shape[0], N)
    poses = np.stack([np.stack([wp[k], wp[(k - 23) % len(wp)]]) for k in ks])
    poses[0, 1] = poses[0, 0] + np.array([0.1, 0.05, 0.3])
    sim = make_sim(f110, dev, em, N, A)
    sim.reset(poses)
    pl = f110.PurePursuitPlanner(device=dev)
    obs = sim.observations()
    for _ in range(50):
        obs = sim.step(pl.plan_actions(obs, 0.8, 1.0))
    torch.cuda.synchronize()
    # the device's cos / sin the model uses are the tick's own sincos (k_dynamics' pose snapshot)
    st = sim.state
    ap = sim.agent_poses
    same = ap[:, 2] == st[4]                  # not zeroed by a wall hit after the snapshot
    assert int(same.sum()) >= 8
    assert torch.equal(ap[same, 3], torch.cos(st[4][same])) and torch.equal(ap[same, 4], torch.sin(st[4][same]))
    check_all_settings(f110, sim)
    v = sim.render_views([0, 1], (64, 64), 0.02, 0.0, True).cpu().numpy()
    assert np.array_equal(v, model_of(f110, sim, [0, 1], (64, 64), 0.02, 0.0, True))
    assert (v[0] == 3).sum() > 0 and (v[1] == 3).sum() > 0 and (v[0] == 4).sum() > 0


@pytest.mark.parametrize('kind', ['canvas4', 'rot4', 'mixres6'])
def test_one_pixel_views_at_the_boundary_builders(f110, dev, stacks, kind):
    """Agents placed with Simulator.reset at the cell-edge, just-below / at-extent, tiny-negative and -0.0 builders of each
    layer; a 1 x 1 view's one pixel centre is the agent's (x, y).  The car size is NaN in the struct, so no car is drawn and the
    pixel shows the map class: off the map exactly where the oracle's xy_2_rc is, and equal to the model."""
    dmap, hosts = stacks[kind]
    L = len(hosts)
    geom, res, rot, dt = layer_tables(dmap)
    rng = np.random.default_rng(40)
    for l, h in enumerate(hosts):
        x, y, bands = rotated_probe_points(h, rng, 2000)
        pick = np.concatenate([v for k, v in bands.items() if k not in ('uniform', 'far')])
        pick = rng.choice(pick, min(4096, pick.size), replace=False)
        x, y = x[pick], y[pick]                          # the builders
        n = x.size
        sim = make_sim(f110, dev, dmap, n, 1, np.full(n, l) if L > 1 else None)
        sim.c.sim_length = sim.c.sim_width = float('nan')
        sim.reset(np.stack([x, y, rng.uniform(-np.pi, np.pi, n)], axis=1)[:, None, :])
        flat = model_flat(h, geom[l], res[l], rot[l], x, y)
        assert agrees(h, flat, oracle_cells(h, x, y)).all()
        assert (flat < 0).sum() > 0 and (flat >= 0).sum() > 0
        for hu in (True, False):
            got = sim.render_views(None, (1, 1), 0.1, 0.0, hu).cpu().numpy()[:, 0, 0]
            want = model_of(f110, sim, None, (1, 1), 0.1, 0.0, hu)[:, 0, 0]
            assert np.array_equal(got, want), (kind, l)
            assert np.array_equal(got == 0, flat < 0), (kind, l)
            cells = dt[l].reshape(-1)[np.where(flat >= 0, (flat // h.width) * dt.shape[2] + flat % h.width, 0)]
            assert np.array_equal(got[flat >= 0] == 2, cells[flat >= 0] == 0), (kind, l)


def test_invalid_views(f110, dev, stacks):
    dmap, hosts = stacks['canvas4']
    N, A = 8, 2
    ids = np.arange(N) % 4
    sim = make_sim(f110, dev, dmap, N, A, ids)
    poses = on_map_poses(hosts, ids, A, np.random.default_rng(50))
    poses[1, 0, 0] = np.nan                       # agent 2: NaN pose
    poses[2, 1, 2] = np.inf                       # agent 5: infinite yaw
    poses[3, 0, :2] = 1e12                        # agent 6: far off every map
    sim.reset(poses)
    sim.env_layer[5] = 4                          # env 5 on a layer the map does not have
    sim.env_layer[6] = -1
    bad_ids = torch.tensor([0, -1, N * A, 2, 5, 6, 10, 12, 2 ** 31 - 1, 1], dtype=torch.int32, device=dev)
    got = sim.render_views(bad_ids, (33, 17), 0.1, 0.0, True).cpu().numpy()
    want = model_of(f110, sim, bad_ids.cpu().numpy(), (33, 17), 0.1, 0.0, True)
    assert np.array_equal(got, want)
    for k in (1, 2, 3, 4, 6, 7, 8):
        assert np.all(got[k] == 255), k
    assert not np.any(got[[0, 9]] == 255)
    assert set(np.unique(got[5])) <= {0, 4}                 # 1e12: no map cell, only the car itself
    far = sim.render_views([6], (8, 8), 2.0, 0.0, False).cpu().numpy()
    assert np.all(far == 0)


def test_views_leave_the_simulation_unchanged(f110, dev, six):
    N, A = 64, 2
    poses = on_map_poses([six[0].host], [0] * N, A, np.random.default_rng(60))
    acts = np.random.default_rng(61).uniform([-0.3, 0.0], [0.3, 6.0], (30, N, A, 2))
    outs = []
    for render in (False, True):
        sim = make_sim(f110, dev, six[0], N, A)
        sim.set_noise(0.01, 5)
        sim.reset(poses)
        for t in range(30):
            sim.tick(acts[t])
            if render:
                sim.render_views(None, (32, 32), 0.1, 0.0, t % 2 == 0)
        torch.cuda.synchronize()
        outs.append([sim.state.clone(), sim.scans.clone(), sim.collisions.clone(), sim.lap_counts.clone(),
                     sim.tick_counter.clone()])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_graph_capture_equals_eager(f110, dev, stacks):
    dmap, hosts = stacks['rot4']
    N, A = 16, 2
    ids = np.arange(N) % 4
    sim = make_sim(f110, dev, dmap, N, A, ids)
    sim.reset(on_map_poses(hosts, ids, A, np.random.default_rng(70)))
    out = torch.empty((N * A, 48, 40), dtype=torch.uint8, device=dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        sim.render_views(None, (48, 40), 0.1, 1.0, True, out=out)      # warm-up: module load, the cached id table
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    eager = out.clone()
    out.fill_(77)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        sim.render_views(None, (48, 40), 0.1, 1.0, True, out=out)
    assert g.replay() is None
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    # new poses, same graph: the replay reads the current state
    sim.reset(on_map_poses(hosts, ids, A, np.random.default_rng(71)))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, sim.render_views(None, (48, 40), 0.1, 1.0, True))


def test_f110env_rgb_array_and_local_map(f110, dev):
    from f1tenth_gym_b200.env import RENDER_PALETTE
    pal = torch.from_numpy(RENDER_PALETTE).to(dev)
    lm = {'size': (40, 24), 'metres_per_pixel': 0.1, 'forward_offset': 1.0}
    env = f110.F110Env(map='berlin', num_agents=2, num_envs=6, device=dev, scan_noise_std=0.0, local_map=lm)
    assert 'rgb_array' in env.metadata['render.modes']
    h = env.sim.map.host
    poses = on_map_poses([h], [0] * 6, 2, np.random.default_rng(80))
    obs, _, _, _ = env.reset(poses)
    for _ in range(3):
        obs, _, _, _ = env.step(torch.zeros((6, 2, 2), dtype=torch.float64, device=dev))
    buf = obs['local_map']
    assert tuple(buf.shape) == (6, 2, 40, 24) and buf.dtype == torch.uint8 and buf.is_cuda
    ref = env.sim.render_views(None, (40, 24), 0.1, 1.0, True).view(6, 2, 40, 24)
    assert torch.equal(buf, ref)
    obs2, _, _, _ = env.step(torch.zeros((6, 2, 2), dtype=torch.float64, device=dev))
    assert obs2['local_map'].data_ptr() == buf.data_ptr()            # one persistent buffer
    rgb = env.render(mode='rgb_array', env_ids=[0, 3, 5], size=(60, 80), metres_per_pixel=0.05)
    cls = env.sim.render_views([0, 6, 10], (60, 80), 0.05, 0.0, False)
    assert tuple(rgb.shape) == (3, 60, 80, 3) and rgb.is_cuda and torch.equal(rgb, pal[cls.long()])
    assert tuple(env.render(mode='rgb_array').shape) == (1, 800, 1000, 3)
    for mode in ('human', 'human_fast'):
        with pytest.raises(NotImplementedError):
            env.render(mode=mode)
    # single-env mode: numpy
    one = f110.F110Env(map='vegas', num_agents=2, device=dev, scan_noise_std=0.0, local_map=lm)
    hv = one.sim.map.host
    obs, _, _, _ = one.reset(on_map_poses([hv], [0], 2, np.random.default_rng(81))[0])
    assert isinstance(obs['local_map'], np.ndarray) and obs['local_map'].shape == (2, 40, 24)
    assert np.array_equal(obs['local_map'], one.sim.render_views(None, (40, 24), 0.1, 1.0, True).cpu().numpy())
    img = one.render(mode='rgb_array', size=(50, 70), metres_per_pixel=0.05)
    assert isinstance(img, np.ndarray) and img.shape == (50, 70, 3) and img.dtype == np.uint8
    cls = one.sim.render_views([0], (50, 70), 0.05, 0.0, False)
    assert np.array_equal(img, pal[cls.long()][0].cpu().numpy())
    plain = f110.F110Env(map='vegas', num_agents=2, num_envs=2, device=dev, scan_noise_std=0.0)
    obs, _, _, _ = plain.reset(on_map_poses([hv], [0, 0], 2, np.random.default_rng(82)))
    assert 'local_map' not in obs


def test_device_without_an_index(f110, dev):
    """device='cuda' (no index): render_views(out=...) and F110Env's local_map buffer are on that device."""
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 2, 7, num_envs=4, device='cuda', noise_std=0.0)
    berlin = f110.DeviceMap.from_yaml(os.path.join(MAPS, 'berlin.yaml'), '.png', 'cuda')
    sim.set_device_map(berlin)
    sim.reset(on_map_poses([berlin.host], [0] * 4, 2, np.random.default_rng(90)))
    out = torch.empty((8, 12, 10), dtype=torch.uint8, device='cuda')
    assert sim.render_views(None, (12, 10), 0.1, 0.0, True, out=out) is out
    assert torch.equal(out, sim.render_views(None, (12, 10), 0.1, 0.0, True))
    assert np.array_equal(out.cpu().numpy(), model_of(f110, sim, None, (12, 10), 0.1, 0.0, True))
    lm = {'size': (16, 8), 'metres_per_pixel': 0.1}
    env = f110.F110Env(map='berlin', num_agents=2, num_envs=3, device='cuda', scan_noise_std=0.0, local_map=lm)
    obs, _, _, _ = env.reset(on_map_poses([berlin.host], [0] * 3, 2, np.random.default_rng(91)))
    assert torch.equal(obs['local_map'], env.sim.render_views(None, (16, 8), 0.1, 0.0, True).view(3, 2, 16, 8))
    one = f110.F110Env(map='berlin', num_agents=2, device='cuda', scan_noise_std=0.0, local_map=lm)
    obs, _, _, _ = one.reset(on_map_poses([berlin.host], [0], 2, np.random.default_rng(92))[0])
    assert obs['local_map'].shape == (2, 16, 8)
    with pytest.raises(ValueError):
        one.render(mode='rgb_array', env_ids=[0, 0])
    with pytest.raises(ValueError):
        one.render(mode='rgb_array', env_ids=[1])


def test_device_ids_must_be_int32(f110, dev, six):
    sim = make_sim(f110, dev, six[0], 2, 2)
    sim.reset(on_map_poses([six[0].host], [0, 0], 2, np.random.default_rng(93)))
    for dt in (torch.int64, torch.int16, torch.float32):
        with pytest.raises(ValueError):
            sim.render_views(torch.tensor([2 ** 32 + 3 if dt == torch.int64 else 1], dtype=dt, device=dev), (4, 4))
    got = sim.render_views(torch.tensor([3, 4], dtype=torch.int32, device=dev), (4, 4)).cpu().numpy()
    assert np.array_equal(got, model_of(f110, sim, [3, 4], (4, 4), 0.1, 0.0, True))


def test_more_views_than_the_grid_height(f110, dev, six):
    """V > 65535: the grid's y dimension strides over the views (each block draws several)."""
    N, A = 40000, 2
    sim = make_sim(f110, dev, six[0], N, A)
    sim.reset(on_map_poses([six[0].host], [0] * 64, A, np.random.default_rng(94))[np.arange(N) % 64])
    V = N * A
    assert V > 65535
    got = sim.render_views(None, (5, 7), 0.1, 0.5, True).cpu().numpy()
    # envs e and e + 64 hold the same poses: their views are equal, and env e's equal the model
    want = model_of(f110, sim, np.arange(64 * A), (5, 7), 0.1, 0.5, True)
    assert np.array_equal(got[:64 * A], want)
    assert np.array_equal(got.reshape(N // 64, 64 * A, 5, 7), np.broadcast_to(want, (N // 64, 64 * A, 5, 7)))
    ids = torch.arange(V, dtype=torch.int32, device=dev).flip(0)
    assert np.array_equal(sim.render_views(ids, (5, 7), 0.1, 0.5, True).cpu().numpy(), got[::-1])
