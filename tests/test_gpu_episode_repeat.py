"""Episodes under a held action (Simulator.tick_repeat in episode mode, C ABI f110_tick_repeat_episodes) on the GPU.

Twin simulators, as in test_gpu_episodes: before every call every buffer of A is copied into B; A runs one call of K ticks and
B runs K plain ticks (env_level, no auto-reset), recording every buffer after each.  The host restates each env's end tick j,
the flags, the lengths, end_tick, done_any and done_tick from B's done.  Then envs that did not end equal B after K ticks on
every buffer, scans included; the final_* buffers of an ended env equal B's record at j (final_scans included, also when j is
an intermediate tick of the short path, which computes no scans); done is B's at j; the start poses and boxes equal the host
restatements of the draws at the call's last tick; and each restarted env equals a fresh simulator C placed at the drawn poses
that steps once under zero actions.  Every case counts its events and requires terminated and truncated ends on an
intermediate tick, ends on the last tick and ends on tick 0 to fire.
"""
import types

import numpy as np
import pytest
import torch

from test_gpu_episodes import BUFFERS, CASES, COPIED, FINAL, N, check_rows, rows, u64_as_i64
from test_gpu_repeat import dev, f110, kinds, make_sim, population, same_bits, tables_of  # noqa: F401 (fixtures)
from test_gpu_scale import AR_SEED, POSE_GAP, autoreset_poses, random_actions

pytestmark = pytest.mark.gpu

OBST = ('obstacle_boxes', 'obstacle_active', 'obstacle_hit')
PROGRESS = ('track_seg', 'track_s', 'track_d', 'track_heading_error', 'track_progress', 'track_delta')


def record(sim, names):
    return types.SimpleNamespace(**{n: (getattr(sim, n).clone() if getattr(sim, n, None) is not None else None) for n in names})


def restate(done_j, prev_ticks, max_ticks):
    """The end decision of every tick of the call, from B's done after each tick: (end, term, trunc, length, ticks, done_any,
    done_tick)."""
    K = len(done_j)
    end = np.full(prev_ticks.shape, -1)
    term, trunc = np.zeros(prev_ticks.shape, bool), np.zeros(prev_ticks.shape, bool)
    length = np.zeros(prev_ticks.shape, np.int64)
    t = prev_ticks.astype(np.int64).copy()
    done_any = np.zeros(prev_ticks.shape, bool)
    done_tick = np.full(prev_ticks.shape, -1)
    for j in range(K):
        run = end < 0
        tj = t + 1
        d = done_j[j]
        done_any |= run & d
        done_tick = np.where(run & d & (done_tick < 0), j, done_tick)
        tm = d
        tr = ~tm & (max_ticks > 0) & (tj >= max_ticks)
        now = run & (tm | tr)
        end[now] = j
        term[now], trunc[now] = tm[now], tr[now]
        length[now] = tj[now]
        t = np.where(run, tj, t)
    ticks = np.where(end >= 0, 0, t)
    return end, term, trunc, length, ticks, done_any, done_tick


def repeat_run(f110, dev, case, A, K, calls, max_ticks, seed=5, noise=0.0, obstacles=False, lidar=None, toggles=False,
               progress=False):
    dmap, hosts, kind, _ = case
    rng = np.random.default_rng(seed)
    ids = np.arange(N) % len(hosts)
    poses = population(kind, hosts, ids, rng, A)
    tabs = tables_of(kind, hosts, rng, dev)
    a, b, c = (make_sim(f110, dev, dmap, ids, poses, A, noise_std=noise) for _ in range(3))
    draw = None
    if obstacles:
        tab = tabs.cpu().numpy()
        cand = np.concatenate([tab, np.tile([[0.58, 0.31]], (tab.shape[0], 1))], axis=1)
        draw = dict(candidates=cand, count=(1, 3), clearance=1.0, seed=7)
        for s in (a, b, c):
            s.set_obstacles(np.zeros((N, 3, 5)), np.zeros((N, 3), bool))
        a.set_obstacle_draw(cand, count=(1, 3), clearance=1.0, seed=7)
        a.respawn_obstacles()
    if lidar is not None:
        for s in (a, b, c):
            s.set_lidar(lidar)
    if progress:
        wp = f110.maps.load_waypoints()
        for s in (a, b):
            s.set_centerlines(wp[:, :2])
    a.set_episodes(max_ticks)
    sentinel = a.scans.clone()
    zeros = torch.zeros((N, A, 2), dtype=torch.float64, device=dev)
    names = BUFFERS + (OBST if obstacles else ()) + (PROGRESS if progress else ())
    slots = [i for i in range(A) if lidar is None or lidar[i]]
    ev = dict(term_mid=0, trunc_mid=0, last=0, first=0, restarted=0, laps=0)
    for call in range(calls):
        if toggles and call % 5 == 2:
            a.toggle_list.fill_(3.0)        # the next crossing of the start zone completes every agent's two laps
        for n in COPIED:
            if getattr(a, n, None) is not None and getattr(b, n, None) is not None:
                getattr(b, n).copy_(getattr(a, n))
        prev_ticks = a.ep_ticks.cpu().numpy().copy()
        act = torch.from_numpy(random_actions(rng, N, A)).to(dev)
        obs = a.tick_repeat(act, K, env_level=True, autoreset_poses=tabs, progress=progress)
        if call == 0:
            # the path under test: without noise the intermediate ticks take the short path, whose ends the final-scan pass
            # completes; with noise every tick is the plain tick and the pass is empty
            launch = f110._native.lib().f110_debug_last_launch().decode()
            if K > 1:
                want = ('sub=ttc', 'final_scan=k_restart_march') if noise == 0.0 else ('sub=full', 'final_scan=none')
                assert all(any(t.startswith(w) for t in launch.split()) for w in want), launch
            assert 'restart=k_episode_restart+' in launch, launch
        rec, dsum = [], None
        for j in range(K):
            b.tick(act, env_level=True)
            if progress:
                d = b.update_progress()['delta'].reshape(-1).clone()
                dsum = d if dsum is None else dsum + d
            rec.append(record(b, names))
        done_j = [r.done.cpu().numpy().astype(bool) for r in rec]
        end, term, trunc, length, ticks, done_any, done_tick = restate(done_j, prev_ticks, max_ticks)
        ended = end >= 0
        assert np.array_equal(obs['end_tick'].cpu().numpy(), end), call
        assert np.array_equal(a.end_tick.cpu().numpy(), end), call
        assert np.array_equal(obs['terminated'].cpu().numpy().astype(bool), term), call
        assert np.array_equal(obs['truncated'].cpu().numpy().astype(bool), trunc), call
        assert np.array_equal(a.episode_ticks.cpu().numpy(), ticks), call
        assert np.array_equal(a.episode_length.cpu().numpy()[ended], length[ended]), call
        assert np.array_equal(obs['done_any'].cpu().numpy().astype(bool), done_any), call
        assert np.array_equal(obs['done_tick'].cpu().numpy(), done_tick), call
        keep = np.nonzero(~ended)[0]
        check_rows(a, rec[K - 1], keep, names, N, A, ('not ended', call))
        if progress:
            assert same_bits(a.track_delta_sum.view(N, A)[keep], dsum.view(N, A)[keep]), call
        envs = np.nonzero(ended)[0]
        if envs.size == 0:
            continue
        if progress:
            assert (a.track_delta_sum.view(N, A)[envs] == 0).all(), call
        ev['restarted'] += int(envs.size)
        ev['term_mid'] += int((term & (end < K - 1)).sum())
        ev['trunc_mid'] += int((trunc & (end < K - 1)).sum())
        ev['last'] += int((end == K - 1).sum())
        ev['first'] += int((end == 0).sum())
        for j in range(K):
            at = np.nonzero(end == j)[0]
            if at.size == 0:
                continue
            ev['laps'] += int((rec[j].checkpoint_done.view(N, A).cpu().numpy()[at].all(1)).sum())
            for fn, bn in FINAL:
                assert same_bits(rows(getattr(a, fn), N, A, at, True), rows(getattr(rec[j], bn), N, A, at, True)), (fn, call, j)
            fs, bs = a.final_scans.view(N, A, -1)[at], rec[j].scans.view(N, A, -1)[at]
            assert same_bits(fs[:, slots], bs[:, slots]), ('final_scans', call, j)
            assert same_bits(a.done[at], rec[j].done[at]), ('done', call, j)
        if lidar is not None and not all(lidar) and noise == 0.0:
            off = [i for i in range(A) if not lidar[i]]
            assert same_bits(a.scans.view(N, A, -1)[envs][:, off], sentinel.view(N, A, -1)[envs][:, off]), call
            assert same_bits(a.final_scans.view(N, A, -1)[envs][:, off], torch.zeros_like(a.final_scans.view(N, A, -1)[envs][:, off]))
        # the draws at the counter of the call's last tick
        tick = int(b.tick_counter.item())
        starts = torch.stack([a.start_xs, a.start_ys, a.start_thetas], 1).view(N, A, 3).cpu().numpy()
        for e in envs:
            tab = tabs[ids[e]] if isinstance(tabs, list) else tabs
            assert np.array_equal(starts[e], autoreset_poses(tab.cpu().numpy(), AR_SEED, tick, int(e), A, POSE_GAP)), (call, e)
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
        check_rows(a, c, envs, tuple(n for n in BUFFERS if n != 'done') + (OBST if obstacles else ()), N, A, ('restart', call))
    return ev


def expect(ev, K, laps=False):
    assert ev['last'] > 0 and ev['first'] > 0, ev
    if K > 1:
        assert ev['term_mid'] > 0 and ev['trunc_mid'] > 0, ev
    if laps:
        assert ev['laps'] > 0, ev


def limit(K):
    """A time limit that is not a multiple of K: a truncation lands on tick K - 2 of a call (tick 0 for K = 2).  Long enough
    that collisions end episodes on every tick of a call too."""
    return 10 * K - 1 if K > 1 else 31


@pytest.mark.parametrize('name,A', CASES)
@pytest.mark.parametrize('noise', [0.0, 0.01])
@pytest.mark.parametrize('K', [1, 2, 4, 8])
def test_repeat_episodes_are_plain_ticks_cut_at_the_end(f110, dev, kinds, name, A, noise, K):
    ev = repeat_run(f110, dev, kinds[name], A, K, calls=max(40, 480 // K), max_ticks=limit(K), noise=noise,
                    seed=A * 11 + len(name) + K)
    expect(ev, K)


@pytest.mark.parametrize('K', [2, 4])
def test_repeat_episodes_time_limit_multiple_of_k_and_laps(f110, dev, kinds, K):
    ev = repeat_run(f110, dev, kinds['example_map'], 2, K, calls=200 // K, max_ticks=5 * K, seed=K)
    assert ev['trunc_mid'] == 0 and ev['last'] > 0, ev
    ev = repeat_run(f110, dev, kinds['example_map'], 2, K, calls=160 // K, max_ticks=0, toggles=True, seed=K + 1)
    assert ev['laps'] > 0 and ev['restarted'] > 0, ev


@pytest.mark.parametrize('K', [1, 4])
def test_repeat_episodes_with_obstacles_lidar_mask_and_progress(f110, dev, kinds, K):
    ev = repeat_run(f110, dev, kinds['example_map'], 2, K, calls=240 // K, max_ticks=limit(K), obstacles=True,
                    lidar=[True, False], progress=True)
    expect(ev, K)
    ev = repeat_run(f110, dev, kinds['example_map'], 3, K, calls=160 // K, max_ticks=limit(K), obstacles=True,
                    lidar=[False, True, True], noise=0.01, seed=8)
    assert ev['restarted'] > 0, ev


def test_k1_equals_the_episode_tick(f110, dev, kinds):
    """K = 1 through the new entry point is f110_tick_episodes bit for bit, with boxes and a lidar mask."""
    dmap, hosts, kind, _ = kinds['example_map']
    rng = np.random.default_rng(4)
    ids = np.zeros(N, int)
    A = 2
    poses = population(kind, hosts, ids, rng, A)
    tabs = tables_of(kind, hosts, rng, dev)
    sims = [make_sim(f110, dev, dmap, ids, poses, A) for _ in range(2)]
    cand = np.concatenate([tabs.cpu().numpy(), np.tile([[0.58, 0.31]], (tabs.shape[0], 1))], axis=1)
    for s in sims:
        s.set_obstacles(np.zeros((N, 2, 5)), np.zeros((N, 2), bool))
        s.set_obstacle_draw(cand, count=(0, 2), clearance=1.0, seed=3)
        s.respawn_obstacles()
        s.set_lidar([True, False])
        s.set_episodes(17)
    restarts = 0
    for i in range(80):
        act = random_actions(rng, N, A)
        obs = sims[0].tick_repeat(act, 1, env_level=True, autoreset_poses=tabs)
        sims[1].tick(act, env_level=True, autoreset_poses=tabs)
        for n in BUFFERS + OBST + ('ep_ticks', 'ep_terminated', 'ep_truncated', 'ep_length', 'final_state', 'final_scans',
                                   'final_collisions', 'final_collision_idx', 'final_lap_times', 'final_lap_counts'):
            assert same_bits(getattr(sims[0], n), getattr(sims[1], n)), (i, n)
        ended = (sims[1].terminated | sims[1].truncated).bool()
        assert torch.equal(obs['end_tick'], torch.where(ended, 0, -1).to(torch.int32)), i
        assert torch.equal(obs['done_any'], sims[1].done) and torch.equal(obs['done_tick'], torch.where(sims[1].done.bool(), 0, -1).to(torch.int32))
        restarts += int(ended.sum().item())
    assert restarts > 0


@pytest.mark.parametrize('progress', [False, True])
def test_repeat_episode_graph_equals_eager(f110, dev, kinds, progress):
    dmap, hosts, kind, _ = kinds['example_map']
    rng = np.random.default_rng(9)
    ids = np.zeros(N, int)
    A, K = 2, 4
    poses = population(kind, hosts, ids, rng, A)
    tabs = tables_of(kind, hosts, rng, dev)
    wp = f110.maps.load_waypoints()
    sims = [make_sim(f110, dev, dmap, ids, poses, A) for _ in range(2)]
    for s in sims:
        s.set_episodes(limit(K))
        s.set_centerlines(wp[:, :2])
    act = torch.zeros((N, A, 2), dtype=torch.float64, device=dev)
    g = sims[0].capture_graph(act, autoreset_poses=tabs, env_level=True, progress=progress, repeat=K)
    mid = 0
    for i in range(40):
        act.copy_(torch.from_numpy(random_actions(rng, N, A)))
        g.replay()
        sims[1].tick_repeat(act, K, env_level=True, autoreset_poses=tabs, progress=progress)
        mid += int(((sims[1].end_tick >= 0) & (sims[1].end_tick < K - 1)).sum().item())
        names = BUFFERS + ('ep_ticks', 'ep_terminated', 'ep_truncated', 'ep_length', 'final_state', 'final_scans', 'ep_end_tick',
                           'done_any', 'done_tick', 'track_seg', 'track_s', 'track_progress')
        for n in names + (('track_delta_sum',) if progress else ()):
            assert same_bits(getattr(sims[0], n), getattr(sims[1], n)), (i, n)
    assert mid > 0


def test_env_episode_repeat_with_pure_pursuit_opponent(f110, dev):
    wp = f110.maps.load_waypoints()
    n, A, K = 32, 2, 4
    table = torch.from_numpy(np.ascontiguousarray(wp[::5])).to(dev)
    env = f110.F110Env(map='example_map', map_ext='.png', num_agents=A, num_envs=n, scan_noise_std=0.0, device=dev,
                       lidar=[True, False], autoreset={'poses': table, 'max_episode_steps': 40, 'seed': 3, 'pose_gap': 5,
                                                       'action_repeat': K})
    rng = np.random.default_rng(1)
    k = rng.integers(0, wp.shape[0], n)
    obs, _, _, _ = env.reset(np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1))
    pl = f110.PurePursuitPlanner(device=dev)
    seen = mid = 0
    for step in range(120):
        act = torch.from_numpy(random_actions(rng, n, A)).to(dev)
        act[:, 1] = pl.plan_actions(obs, 0.82461887897713965, 0.90338203837889)[:, 1]
        obs, reward, done, info = env.step(act)
        assert set(info) >= {'terminated', 'truncated', 'end_tick', 'episode_length', 'final_observation', 'checkpoint_done'}
        assert done.dtype == torch.bool and done.shape == (n,)
        assert torch.equal(done, info['terminated'] | info['truncated'])
        assert torch.equal(done, info['end_tick'] >= 0)
        et = info['end_tick']
        assert torch.equal(reward, torch.where(et >= 0, et + 1, K).double() * env.timestep)
        # a time limit of 40 steps is 160 ticks, which every truncated episode ran
        assert (info['episode_length'][info['truncated']] == 40).all()
        assert info['final_observation']['scans'].shape == (n, A, 1080)
        if done.any():
            d = done.nonzero().flatten()
            assert torch.isfinite(obs['scans'][d, 0]).all() and torch.isnan(obs['scans'][d, 1]).all()
            assert (env.sim.episode_ticks[d] == 0).all() and (env.sim.current_time[d] == env.timestep).all()
        seen += int(done.sum().item())
        mid += int(((et >= 0) & (et < K - 1)).sum().item())
    assert seen > 0 and mid > 0
