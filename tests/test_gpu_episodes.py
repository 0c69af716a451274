"""Episode mode (Simulator.set_episodes, C ABI f110_tick_episodes) on the GPU.

Twin simulators: before every tick every buffer of A is copied into B, then A runs the episode tick and B the plain tick
(env_level, no auto-reset).  Envs that did not end are bit-identical on every buffer, scans included; for ended envs the final_*
buffers equal B's buffers, the flags and lengths equal a numpy restatement from B's done and the counters, and the start poses
and boxes equal the host restatements of the draws.  Each restarted env then equals a fresh simulator C that env_reset places
at A's drawn start poses, with its tick counter at (t | 2^63) - 1, after step(zeros) and env_post_step, on every buffer but
done, tick_counter and the march queue.  A in {1, 2, 3, 4}; five map kinds; noise on and off; boxes with a redraw table; a lidar
mask; the time limit, lap completion and collisions each fire.  Then a captured graph against eager ticks and F110Env.
"""
import numpy as np
import pytest
import torch

from test_gpu_repeat import dev, f110, kinds, make_sim, population, same_bits, tables_of  # noqa: F401 (fixtures)
from test_gpu_scale import AR_SEED, POSE_GAP, autoreset_poses, random_actions

pytestmark = pytest.mark.gpu

N = 64
BUFFERS = ('state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'march_rec', 'wall_flag', 'collisions', 'collision_idx',
           'current_time', 'lap_times', 'lap_counts', 'toggle_list', 'near_starts', 'start_xs', 'start_ys', 'start_thetas',
           'start_rot', 'done', 'checkpoint_done', 'tick_counter', 'scans')
COPIED = BUFFERS + ('march_cost', 'march_order', 'march_count', 'obstacle_boxes', 'obstacle_active', 'obstacle_hit', 'ep_ticks',
                    'track_seg', 'track_s', 'track_d', 'track_heading_error', 'track_progress', 'track_delta')
FINAL = (('final_state', 'state'), ('final_collisions', 'collisions'), ('final_collision_idx', 'collision_idx'),
         ('final_lap_times', 'lap_times'), ('final_lap_counts', 'lap_counts'))


def rows(t, N, A, envs, per_agent):
    """The rows of `envs` of a buffer laid out [.., N*A(, B)] or [N(, k)]."""
    if t.dim() == 2 and t.shape[0] in (2, 7) and t.shape[1] == N * A:      # state [7][N*A], steer_buf [2][N*A]
        return t.view(t.shape[0], N, A)[:, envs]
    if t.shape[0] == N * A and per_agent:
        return t.view(N, A, *t.shape[1:])[envs]
    if t.shape[0] == N:
        return t[envs]
    return t


def check_rows(x, y, envs, names, N, A, what):
    for n in names:
        tx, ty = getattr(x, n), getattr(y, n)
        if tx is None or n == 'tick_counter':
            continue
        assert same_bits(rows(tx, N, A, envs, True), rows(ty, N, A, envs, True)), (what, n)


def u64_as_i64(v):
    return int(np.array([v], dtype=np.uint64).view(np.int64)[0])


def episode_run(f110, dev, case, A, steps, max_ticks, seed=5, noise=0.0, obstacles=False, lidar=None, toggles=False):
    dmap, hosts, kind, _ = case
    rng = np.random.default_rng(seed)
    ids = np.arange(N) % len(hosts)
    poses = population(kind, hosts, ids, rng, A)
    tabs = tables_of(kind, hosts, rng, dev)
    a = make_sim(f110, dev, dmap, ids, poses, A, noise_std=noise)
    b = make_sim(f110, dev, dmap, ids, poses, A, noise_std=noise)
    c = make_sim(f110, dev, dmap, ids, poses, A, noise_std=noise)
    draw = None
    if obstacles:
        tab = tabs.cpu().numpy()
        cand = np.concatenate([tab, np.tile([[0.58, 0.31]], (tab.shape[0], 1))], axis=1)
        draw = dict(candidates=cand, count=(1, 3), clearance=1.0, seed=7)
        for s in (a, b, c):
            s.set_obstacles(np.zeros((N, 3, 5)), np.zeros((N, 3), bool))
        a.set_obstacle_draw(cand, count=(1, 3), clearance=1.0, seed=7)
        a.respawn_obstacles()
        b.obstacle_boxes.copy_(a.obstacle_boxes), b.obstacle_active.copy_(a.obstacle_active)
    if lidar is not None:
        for s in (a, b, c):
            s.set_lidar(lidar)
    a.set_episodes(max_ticks)
    sentinel = a.scans.clone()
    zeros = torch.zeros((N, A, 2), dtype=torch.float64, device=dev)
    ev = dict(terminated=0, truncated=0, collision=0, laps=0, restarted=0)
    for step in range(steps):
        if toggles and step % 7 == 3:
            # three toggles: the next crossing of the start zone completes the lap logic's two laps for every agent
            a.toggle_list.fill_(3.0)
        for n in COPIED:
            if getattr(a, n, None) is not None and getattr(b, n, None) is not None:
                getattr(b, n).copy_(getattr(a, n))
        prev_ticks = a.ep_ticks.cpu().numpy().copy()
        act = random_actions(rng, N, A)
        obs = a.tick(act, env_level=True, autoreset_poses=tabs)
        b.tick(act, env_level=True)
        done = b.done.cpu().numpy().astype(bool)
        t = prev_ticks + 1
        term = done
        trunc = ~term & (max_ticks > 0) & (t >= max_ticks)
        ended = term | trunc
        assert np.array_equal(obs['terminated'].cpu().numpy().astype(bool), term), step
        assert np.array_equal(obs['truncated'].cpu().numpy().astype(bool), trunc), step
        assert np.array_equal(a.episode_ticks.cpu().numpy(), np.where(ended, 0, t)), step
        assert np.array_equal(a.episode_length.cpu().numpy()[ended], t[ended]), step
        keep = np.nonzero(~ended)[0]
        check_rows(a, b, keep, BUFFERS + ('obstacle_boxes', 'obstacle_active', 'obstacle_hit'), N, A, ('not ended', step))
        envs = np.nonzero(ended)[0]
        if envs.size == 0:
            continue
        ev['terminated'] += int(term.sum()); ev['truncated'] += int(trunc.sum()); ev['restarted'] += int(envs.size)
        ev['collision'] += int((b.collisions.view(N, A)[:, 0].cpu().numpy()[envs] != 0).sum())
        ev['laps'] += int((b.checkpoint_done.view(N, A).cpu().numpy()[envs].all(1)).sum())
        for fn, bn in FINAL:
            assert same_bits(rows(getattr(a, fn), N, A, envs, True), rows(getattr(b, bn), N, A, envs, True)), (fn, step)
        slots = [i for i in range(A) if lidar is None or lidar[i]]
        fs, bs = a.final_scans.view(N, A, -1)[envs], b.scans.view(N, A, -1)[envs]
        assert same_bits(fs[:, slots], bs[:, slots]), step
        if lidar is not None and not all(lidar) and noise == 0.0:
            off = [i for i in range(A) if not lidar[i]]
            assert same_bits(a.scans.view(N, A, -1)[envs][:, off], sentinel.view(N, A, -1)[envs][:, off]), step
        # the start poses of the auto-reset's draw, and the respawn draw
        tick = int(b.tick_counter.item())
        starts = torch.stack([a.start_xs, a.start_ys, a.start_thetas], 1).view(N, A, 3).cpu().numpy()
        for e in envs:
            tab = tabs[ids[e]] if isinstance(tabs, list) else tabs
            assert np.array_equal(starts[e], autoreset_poses(tab.cpu().numpy(), AR_SEED, tick, int(e), A, POSE_GAP)), (step, e)
            if draw is not None:
                from f1tenth_gym_b200.obstacles import respawn_draw
                bx, act_ = respawn_draw(draw['candidates'], starts[e][:, :2], 3, draw['count'], draw['clearance'], draw['seed'],
                                        tick, int(e))
                assert np.array_equal(a.obstacle_boxes[e].cpu().numpy(), bx)
                assert np.array_equal(a.obstacle_active[e].cpu().numpy(), act_)
        # each restarted env is F110Env.reset of that env: a fresh placement, then one zero-action step
        mask = torch.from_numpy(ended).to(dev)
        c.env_reset(torch.from_numpy(starts).to(dev), mask)
        if obstacles:
            c.obstacle_boxes.copy_(a.obstacle_boxes), c.obstacle_active.copy_(a.obstacle_active)
        c.tick_counter.fill_(u64_as_i64((tick | (1 << 63)) - 1))
        c.step(zeros)
        c.env_post_step()
        names = tuple(n for n in BUFFERS if n != 'done') + (('obstacle_boxes', 'obstacle_active', 'obstacle_hit') if obstacles else ())
        check_rows(a, c, envs, names, N, A, ('restart', step))
    return ev


CASES = [('example_map', 1), ('example_map', 2), ('example_map', 3), ('example_map', 4), ('berlin', 2), ('tracks4', 2),
         ('mixed_resolution', 2), ('rotated', 2)]


@pytest.mark.parametrize('name,A', CASES)
@pytest.mark.parametrize('noise', [0.0, 0.01])
def test_episode_tick_is_plain_tick_plus_reset(f110, dev, kinds, name, A, noise):
    ev = episode_run(f110, dev, kinds[name], A, steps=120, max_ticks=40, noise=noise, seed=A * 11 + len(name))
    assert ev['truncated'] > 0 and ev['terminated'] > 0 and ev['collision'] > 0, ev


def test_episode_lap_completion_and_no_time_limit(f110, dev, kinds):
    ev = episode_run(f110, dev, kinds['example_map'], 2, steps=120, max_ticks=0, toggles=True)
    assert ev['truncated'] == 0 and ev['laps'] > 0, ev


def test_episode_with_obstacles_and_lidar_mask(f110, dev, kinds):
    ev = episode_run(f110, dev, kinds['example_map'], 2, steps=120, max_ticks=30, obstacles=True, lidar=[True, False])
    assert ev['restarted'] > 0, ev
    ev = episode_run(f110, dev, kinds['example_map'], 3, steps=80, max_ticks=25, obstacles=True, lidar=[False, True, True],
                     noise=0.01)
    assert ev['restarted'] > 0, ev


def test_episode_graph_equals_eager(f110, dev, kinds):
    dmap, hosts, kind, _ = kinds['example_map']
    rng = np.random.default_rng(9)
    ids = np.zeros(N, int)
    A = 2
    poses = population(kind, hosts, ids, rng, A)
    tabs = tables_of(kind, hosts, rng, dev)
    wp = f110.maps.load_waypoints()
    sims = [make_sim(f110, dev, dmap, ids, poses, A) for _ in range(2)]
    for s in sims:
        s.set_episodes(20)
        s.set_centerlines(wp[:, :2])
    act = torch.zeros((N, A, 2), dtype=torch.float64, device=dev)
    g = sims[0].capture_graph(act, autoreset_poses=tabs, env_level=True, progress=True)
    restarts = 0
    for i in range(60):
        act.copy_(torch.from_numpy(random_actions(rng, N, A)))
        g.replay()
        sims[1].tick(act, env_level=True, autoreset_poses=tabs)
        sims[1].update_progress()
        restarts += int((sims[1].terminated | sims[1].truncated).sum().item())
        for n in BUFFERS + ('ep_ticks', 'ep_terminated', 'ep_truncated', 'ep_length', 'final_state', 'final_scans', 'track_seg',
                            'track_s', 'track_progress'):
            assert same_bits(getattr(sims[0], n), getattr(sims[1], n)), (i, n)
    assert restarts > 0


def test_env_autoreset_with_pure_pursuit_opponent(f110, dev):
    wp = f110.maps.load_waypoints()
    n, A = 32, 2
    table = torch.from_numpy(np.ascontiguousarray(wp[::5])).to(dev)
    env = f110.F110Env(map='example_map', map_ext='.png', num_agents=A, num_envs=n, scan_noise_std=0.0, device=dev,
                       lidar=[True, False], autoreset={'poses': table, 'max_episode_steps': 60, 'seed': 3, 'pose_gap': 5})
    rng = np.random.default_rng(1)
    k = rng.integers(0, wp.shape[0], n)
    obs, _, _, _ = env.reset(np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1))
    pl = f110.PurePursuitPlanner(device=dev)
    seen = 0
    for step in range(150):
        act = torch.from_numpy(random_actions(rng, n, A)).to(dev)
        act[:, 1] = pl.plan_actions(obs, 0.82461887897713965, 0.90338203837889)[:, 1]
        obs, reward, done, info = env.step(act)
        assert set(info) >= {'terminated', 'truncated', 'episode_length', 'final_observation', 'checkpoint_done'}
        assert done.dtype == torch.bool and done.shape == (n,)
        assert torch.equal(done, info['terminated'] | info['truncated'])
        assert info['terminated'].dtype == torch.bool and info['episode_length'].dtype == torch.int32
        fo = info['final_observation']
        assert fo['scans'].shape == (n, A, 1080) and fo['poses_x'].shape == (n, A)
        # the restarted envs hold their new episode's first observation: at rest near the start pose, one tick in
        if done.any():
            d = done.nonzero().flatten()
            assert torch.isfinite(obs['scans'][d, 0]).all() and torch.isnan(obs['scans'][d, 1]).all()
            assert (env.sim.episode_ticks[d] == 0).all() and (env.sim.current_time[d] == env.timestep).all()
        seen += int(done.sum().item())
    assert seen > 0
