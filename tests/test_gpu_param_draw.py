"""Per-episode parameter draws (Simulator.set_param_draw, C ABI f110_param_draw) on the GPU.

The numpy restatement param_draw.draw_rows is the reference throughout.
  * Host reset: redraw_params(mask) writes exactly the restated rows of the masked envs and nothing else.
  * Plain auto-reset: twin simulators from identical resets; A draws on the device, B gets the restated rows of the envs its own
    ego collision restarted through update_params(env_mask=...) after every tick.  Every buffer and the table are bit-identical
    after every tick: eager and captured ticks, A in {1, 2, 4}, boxes, a lidar mask, noise on and off.
  * Held action: tick_repeat(K) with the in-call auto-reset against K plain ticks with the restated draw after each, under the
    repeat contract (scans: the last tick's); restarts on intermediate ticks are required.
  * Episodes (K = 1 and K in {2, 4}): before every call B takes A's buffers; A runs with the draw, B without.  Envs that did not
    end are bit-identical on every buffer and row; an ended env's row is the restated draw at the call's tick counter, its
    final_observation['params'] the old row, every other buffer B's; and it equals a fresh simulator whose table holds the drawn
    row, env_reset at its start poses, then step(zeros): the zero-action tick does not depend on the drawn keys.
  * F110Env with a pure-pursuit opponent, and two envs at one pose under one action stream that diverge on their drawn mu.
"""
import numpy as np
import pytest
import torch

from test_gpu_episodes import BUFFERS, COPIED, N, check_rows, u64_as_i64
from test_gpu_repeat import dev, f110, kinds, make_sim, population, same_bits, tables_of  # noqa: F401 (fixtures)
from test_gpu_scale import AR_SEED, POSE_GAP, random_actions

pytestmark = pytest.mark.gpu

WIDE = {'mu': (0.6, 1.4), 'C_Sf': (3.5, 6.0), 'C_Sr': (4.0, 7.0), 'm': (3.0, 4.5), 'I': (0.035, 0.06), 'a_max': (6.0, 12.0),
        'v_max': (12.0, 25.0), 'sv_max': (2.0, 4.0)}
GROUPS = [['m', 'I']]


def draw_of(f110, A, per_slot):
    """The draw of a case: WIDE for every slot, or (per_slot) a list of dicts with a slot that is never drawn."""
    if not per_slot or A == 1:
        return WIDE
    out = [dict(WIDE), {}] + [{'mu': (0.8, 1.2), 'lf': (0.14, 0.17), 'v_min': (-6.0, -4.0)}] * (A - 2)
    return out[:A]


def setup(f110, dev, case, A, seed, noise=0.0, boxes=False, lidar=None, copies=2):
    dmap, hosts, kind, _ = case
    rng = np.random.default_rng(seed)
    ids = np.arange(N) % len(hosts)
    poses = population(kind, hosts, ids, rng, A)
    tabs = tables_of(kind, hosts, rng, dev)
    sims = [make_sim(f110, dev, dmap, ids, poses, A, noise_std=noise) for _ in range(copies)]
    for s in sims:
        s.update_params(f110.maps.DEFAULT_PARAMS, env_mask=np.ones(N, bool))      # per-env tables everywhere
        if boxes:
            tab = tabs.cpu().numpy()
            s.set_obstacles(np.zeros((N, 3, 5)), np.zeros((N, 3), bool))
            s.set_obstacle_draw(np.concatenate([tab, np.tile([[0.58, 0.31]], (tab.shape[0], 1))], axis=1), count=(1, 3),
                                clearance=1.0, seed=7)
            s.respawn_obstacles()
        if lidar is not None:
            s.set_lidar(lidar)
    return rng, tabs, sims


def restate(f110, sim, draw, envs, tick):
    """sim's table with the restated rows of `envs` at `tick`, written through update_params."""
    if len(envs) == 0:
        return
    new = f110.param_draw.draw_rows(sim.param_table.cpu().numpy(), draw, tick, envs)
    mask = np.zeros(N, bool)
    mask[envs] = True
    sim.update_params(torch.from_numpy(new), env_mask=mask)


def ego_crashed(sim, A):
    return np.nonzero(sim.collisions.view(N, A)[:, sim.ego_idx].cpu().numpy() != 0)[0]


def same_all(a, b, names, what):
    for n in names:
        if getattr(a, n, None) is not None:
            assert same_bits(getattr(a, n), getattr(b, n)), (what, n)


def test_redraw_params_is_the_restated_draw(f110, dev, kinds):
    for A, per_slot, per_env, groups in ((2, False, False, GROUPS), (3, True, False, None), (4, True, True, GROUPS),
                                         (1, False, True, None)):
        _, _, (a,) = setup(f110, dev, kinds['example_map'], A, seed=A, copies=1)
        a.set_param_draw(draw_of(f110, A, per_slot), groups=groups, per_env=per_env, seed=11 + A)
        a.tick_counter.fill_(1000 + A)
        before = a.param_table.cpu().numpy()
        mask = np.random.default_rng(A).random(N) < 0.5
        a.redraw_params(mask)
        want = f110.param_draw.draw_rows(before, a.param_draw, 1000 + A, np.nonzero(mask)[0])
        got = a.param_table.cpu().numpy()
        assert np.array_equal(got.view(np.int64), want.view(np.int64)), A
        assert np.array_equal(got[~mask], before[~mask]) and not np.array_equal(got[mask], before[mask])
        assert np.array_equal(got[..., 16:], before[..., 16:])            # width / length are never drawn
        if per_env and A > 1:
            assert np.array_equal(got[mask][:, 0, 0], got[mask][:, 1, 0]) or not (a.param_draw['keys'][1] & 1)
        a.redraw_params()                                                  # every env
        want = f110.param_draw.draw_rows(got, a.param_draw, 1000 + A, range(N))
        assert np.array_equal(a.param_table.cpu().numpy(), want)


@pytest.mark.parametrize('A', [1, 2, 4])
@pytest.mark.parametrize('noise', [0.0, 0.01])
@pytest.mark.parametrize('captured', [False, True])
def test_autoreset_draw_equals_restated_rows(f110, dev, kinds, A, noise, captured):
    boxes, lidar = A == 2, ([True, False] if A == 2 else None)
    rng, tabs, (a, b) = setup(f110, dev, kinds['example_map'], A, seed=A + 7, noise=noise, boxes=boxes, lidar=lidar)
    a.set_param_draw(draw_of(f110, A, True), groups=GROUPS, seed=5)
    act = torch.zeros((N, A, 2), dtype=torch.float64, device=dev)
    if captured:
        a.capture_graph(act, autoreset_poses=tabs, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True)
    restarts = 0
    for step in range(150):
        act.copy_(torch.from_numpy(random_actions(rng, N, A)))
        if captured:
            a.replay()
        else:
            a.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        b.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        envs = ego_crashed(b, A)
        restate(f110, b, a.param_draw, envs, int(b.tick_counter.item()))
        restarts += len(envs)
        same_all(a, b, BUFFERS + ('params_dev', 'obstacle_boxes', 'obstacle_active'), step)
    assert restarts > 10, restarts
    assert len(np.unique(a.param_table[:, 0, 0].cpu().numpy())) > 10


@pytest.mark.parametrize('K', [1, 3, 4])
@pytest.mark.parametrize('A', [1, 2])
def test_held_action_draws_after_every_tick(f110, dev, kinds, K, A):
    rng, tabs, (a, b) = setup(f110, dev, kinds['example_map'], A, seed=K * 3 + A, boxes=A == 2)
    a.set_param_draw(draw_of(f110, A, False), groups=GROUPS, per_env=A == 2, seed=9)
    ev = dict(mid=0, last=0)
    for step in range(600 // K):
        act = torch.from_numpy(random_actions(rng, N, A)).to(dev)
        a.tick_repeat(act, K, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        if step == 0 and K > 1:
            assert 'sub=ttc' in f110._native.lib().f110_debug_last_launch().decode()
        for j in range(K):
            b.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
            envs = ego_crashed(b, A)
            restate(f110, b, a.param_draw, envs, int(b.tick_counter.item()))
            ev['mid' if j < K - 1 else 'last'] += len(envs)
        same_all(a, b, BUFFERS + ('params_dev',), step)
    assert ev['last'] > 0 and (K == 1 or ev['mid'] > 0), ev


def episode_draw_run(f110, dev, kinds, A, K, calls, max_ticks, seed, noise=0.0, per_env=False):
    rng, tabs, (a, b, c) = setup(f110, dev, kinds['example_map'], A, seed=seed, noise=noise, copies=3)
    a.set_param_draw(draw_of(f110, A, True), groups=GROUPS, per_env=per_env, seed=21)
    for s in (a, b):
        s.set_episodes(max_ticks)
    zeros = torch.zeros((N, A, 2), dtype=torch.float64, device=dev)
    ev = dict(restarted=0, mid=0, first=0)
    for call in range(calls):
        for n in COPIED + ('params_dev', 'ep_ticks'):
            if getattr(a, n, None) is not None:
                getattr(b, n).copy_(getattr(a, n))
        act = torch.from_numpy(random_actions(rng, N, A)).to(dev)
        old = a.param_table.cpu().numpy()
        if K == 1:
            a.tick(act, env_level=True, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
            b.tick(act, env_level=True, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
        else:
            a.tick_repeat(act, K, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
            b.tick_repeat(act, K, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
            j = b.end_tick.cpu().numpy()
            ev['mid'] += int(((j >= 0) & (j < K - 1)).sum())
            ev['first'] += int((j == 0).sum())
        ended = (b.terminated | b.truncated).cpu().numpy().astype(bool)
        envs = np.nonzero(ended)[0]
        keep = np.nonzero(~ended)[0]
        names = BUFFERS + ('final_state', 'final_scans', 'ep_ticks', 'ep_length', 'ep_terminated', 'ep_truncated')
        check_rows(a, b, keep, names + ('params_dev',), N, A, ('not ended', call))
        check_rows(a, b, envs, names, N, A, ('ended', call))
        tick = int(a.tick_counter.item())
        want = f110.param_draw.draw_rows(old, a.param_draw, tick, envs)
        assert np.array_equal(a.param_table.cpu().numpy(), want), call
        fo = a.final_observation['params'].cpu().numpy()
        assert np.array_equal(fo[envs], old[envs]), call
        if envs.size == 0:
            continue
        ev['restarted'] += int(envs.size)
        # a fresh simulator that runs the new episode's car from the start: its table holds the drawn rows
        mask = torch.from_numpy(ended).to(dev)
        c.update_params(a.param_table.clone(), env_mask=ended)
        starts = torch.stack([a.start_xs, a.start_ys, a.start_thetas], 1).view(N, A, 3)
        c.env_reset(starts.clone(), mask)
        c.tick_counter.fill_(u64_as_i64((tick | (1 << 63)) - 1))
        c.step(zeros)
        c.env_post_step()
        check_rows(a, c, envs, tuple(n for n in BUFFERS if n != 'done') + ('params_dev',), N, A, ('fresh', call))
    return ev


@pytest.mark.parametrize('A', [1, 2, 4])
@pytest.mark.parametrize('noise', [0.0, 0.01])
def test_episode_tick_draw(f110, dev, kinds, A, noise):
    ev = episode_draw_run(f110, dev, kinds, A, 1, calls=120, max_ticks=30, seed=A + 31, noise=noise, per_env=A == 4)
    assert ev['restarted'] > 10, ev


@pytest.mark.parametrize('K', [2, 4])
def test_episode_repeat_draw(f110, dev, kinds, K):
    ev = episode_draw_run(f110, dev, kinds, 2, K, calls=240 // K, max_ticks=7 * K + 1, seed=K + 41)
    assert ev['restarted'] > 10 and ev['mid'] > 0 and ev['first'] > 0, ev


def test_episode_graph_with_draw_equals_eager(f110, dev, kinds):
    for K in (1, 4):
        rng, tabs, (a, b) = setup(f110, dev, kinds['example_map'], 2, seed=K + 61)
        for s in (a, b):
            s.set_param_draw(WIDE, groups=GROUPS, seed=4)
            s.set_episodes(9)
        act = torch.zeros((N, 2, 2), dtype=torch.float64, device=dev)
        a.capture_graph(act, autoreset_poses=tabs, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True, repeat=K)
        restarts = 0
        for i in range(40):
            act.copy_(torch.from_numpy(random_actions(rng, N, 2)))
            a.replay()
            if K == 1:
                b.tick(act, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
            else:
                b.tick_repeat(act, K, autoreset_poses=tabs, pose_gap=POSE_GAP, seed=AR_SEED)
            restarts += int((b.terminated | b.truncated).sum().item())
            same_all(a, b, BUFFERS + ('params_dev', 'final_params', 'final_state', 'ep_ticks'), (K, i))
        assert restarts > 0


def test_env_param_draw_with_pure_pursuit_opponent(f110, dev):
    wp = f110.maps.load_waypoints()
    n, A = 32, 2
    table = torch.from_numpy(np.ascontiguousarray(wp[::5])).to(dev)
    env = f110.F110Env(map='example_map', map_ext='.png', num_agents=A, num_envs=n, scan_noise_std=0.0, device=dev,
                       autoreset={'poses': table, 'max_episode_steps': 40, 'seed': 3, 'pose_gap': 5},
                       param_draw={'ranges': [WIDE, {}], 'groups': GROUPS, 'seed': 8})
    rng = np.random.default_rng(2)
    k = rng.integers(0, wp.shape[0], n)
    obs, _, _, info = env.reset(np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1))
    mu = f110.maps.PARAM_KEYS.index('mu')
    p0 = info['params'].clone()
    assert len(torch.unique(p0[:, 0, mu])) == n and (p0[:, 1] == p0[0, 1]).all()       # slot 1 is never drawn
    pl = f110.PurePursuitPlanner(device=dev)
    seen = 0
    for step in range(120):
        before = env.sim.param_table.clone()
        act = torch.from_numpy(random_actions(rng, n, A)).to(dev)
        act[:, 1] = pl.plan_actions(obs, 0.82461887897713965, 0.90338203837889)[:, 1]
        obs, reward, done, info = env.step(act)
        assert info['params'].shape == (n, A, 18)
        assert torch.equal(info['final_observation']['params'][done], before[done])
        assert torch.equal(info['params'][~done], before[~done])
        if done.any():
            assert not torch.equal(info['params'][done, 0, mu], before[done, 0, mu])
        seen += int(done.sum().item())
    assert seen > 0
    # the draw is keyed on the tick counter: after one more step, reset_envs draws cars no earlier draw gave
    env.step(act)
    mask = torch.zeros(n, dtype=torch.bool)
    mask[:5] = True
    before = env.sim.param_table.clone()
    env.reset_envs(mask, torch.from_numpy(np.stack([wp[(k - POSE_GAP * i) % wp.shape[0]] for i in range(A)], axis=1)))
    after = env.sim.param_table
    assert torch.equal(after[5:], before[5:]) and not torch.equal(after[:5, 0], before[:5, 0])


def test_drawn_mu_makes_twin_envs_diverge(f110, dev):
    """Two envs at one pose under one action stream: their drawn mu (and only it) differ, and so do their trajectories."""
    wp = f110.maps.load_waypoints()
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, AR_SEED, num_envs=2, device=dev)
    sim.set_map(f110.maps.resolve_map_path('example_map'), '.png')
    sim.env_reset(np.tile(wp[100][None, None], (2, 1, 1)))
    sim.set_param_draw({'mu': (0.3, 1.5)}, seed=1)
    sim.redraw_params()
    p = sim.param_table.cpu().numpy()
    assert p[0, 0, 0] != p[1, 0, 0] and np.array_equal(p[0, 0, 1:], p[1, 0, 1:])
    gap = 0.0
    for _ in range(150):
        sim.step(np.tile([[[0.3, 7.0]]], (2, 1, 1)))
        st = sim.state.cpu().numpy()
        gap = max(gap, float(np.abs(st[:, 0] - st[:, 1]).max()))
    assert gap > 1e-3, gap
