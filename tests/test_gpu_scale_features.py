"""Boxes, lidar masks, held actions and episodes against the CPU oracle at benchmark batch sizes.

test_gpu_scale checks the plain tick at the sizes bench.py runs.  The features added since then launch kernels of their own,
and at those sizes they take paths a small batch never reaches: the fixed-grid loops of k_march_ttc and k_restart_march run
more than one item per warp, k_ttc_select's atomics span many blocks, the march is planned on the masked (shorter) queue, k_tail2
runs without its env level before k_obstacles and k_env_tail_obst, and thousands of envs restart on one tick.  Every case is
sized from the SM count, drives the simulator as the matching tools/bench_*.py does, asserts on its first call through
f110_debug_last_launch that it reached the path it covers, and compares EVERY env with the oracle (oracle.step_batch) after
every call, with the tolerances of test_gpu_scale.run_vs_oracle:

  state <= 1e-9; collisions, collision_idx, wall flags, done, toggles and lap counts exact; lap times <= 1e-9;
  beams the opponent ray-cast did not shorten == fp32(oracle) (one fp32 ulp with noise); occluded beams <= 4e-6.

Boxes are parked agents of the oracle (the rule of test_gpu_obstacles.test_parked_car_parity): car-sized, yaw in [0, 2 pi), at
rest under the action (0, 0), an inactive slot far off the map, and toggles at 4 so that they never hold back all_done.  The
oracle restates the device's auto-reset (start-pose draw and respawn draw), the intermediate ticks of tick_repeat, and the
episode restart (the start-pose draw, then one zero-action tick of the ended envs alone, with the noise of counter t | 2^63).
Each case counts its events and asserts that each one it covers fired, and that the loops it covers ran more items than the
grid has warps.
"""
import functools
import os

import numpy as np
import pytest
import torch

import philox_ref
import test_gpu_rotated as rotated
from test_gpu_lidar import check_twins
from test_gpu_multimap import TRACKS, mixed_population, start_table
from test_gpu_scale import (AR_SEED, POSE_GAP, TOL_OCCLUDED, TOL_STATE, autoreset_poses, default_launch_settings, dev,  # noqa: F401
                            example_map, expect_path, f110, omap_of, raceline_population, random_actions, sms)

pytestmark = pytest.mark.gpu

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
T = 12                     # physics ticks per case
K_BOX = 4                  # boxes per env
BOX_DRAW = dict(count=(K_BOX, K_BOX), clearance=0.5, seed=7)
FAR = 1.0e4                # where the oracle parks the agent of an inactive box slot: off the map, out of every scan's reach
TTC_WARPS = 8              # warps per block of k_march_ttc and k_restart_march (F110_TTC_THREADS = 256)
REC_BYTES = 448            # g_launch_rec (csrc/f110_b200.cu): a record of REC_BYTES - 1 characters was cut short


def cpu(t):
    return t.detach().cpu().numpy()


def record(f110):
    """The launch record as a dict (tokens without '=' skipped, a repeated key keeps its last value), after checking that it
    was not cut short."""
    rec = f110._native.lib().f110_debug_last_launch().decode()
    print('launch record (%d chars): %s' % (len(rec), rec))
    assert len(rec) < REC_BYTES - 1, ('launch record cut short', rec)
    return dict(kv.split('=', 1) for kv in rec.split() if '=' in kv)


# ----------------------------------------------------------------------------- the oracle side
class World(object):
    """One OracleSim per env on its layer's map; with boxes, K parked agents after the A cars (slots A .. A+K-1)."""

    def __init__(self, omaps, ids, poses, boxes=None, active=None):
        import oracle
        self.oracle = oracle
        N, A = poses.shape[:2]
        self.N, self.A = N, A
        self.K = 0 if boxes is None else boxes.shape[1]
        self.boxes = None if boxes is None else boxes.copy()
        self.active = None if active is None else active.astype(np.uint8).copy()
        self.sims = [oracle.OracleSim(omaps[ids[e]], num_agents=A + self.K) for e in range(N)]
        for e in range(N):
            self.restart(e, poses[e], None if boxes is None else boxes[e], None if active is None else active[e])

    @staticmethod
    def parked(boxes, active):
        """(K, 3) poses of the parked agents: an active slot's box pose, an inactive slot far off the map."""
        p = np.asarray(boxes, dtype=np.float64)[:, :3].copy()
        off = np.flatnonzero(np.asarray(active) == 0)
        p[off] = np.stack([FAR + 10.0 * off, np.full(off.size, FAR), np.zeros(off.size)], axis=1)
        return p

    def restart(self, e, poses, boxes=None, active=None):
        """orc_env_restart of env e at poses (A, 3), its parked agents moved to boxes (K, 5) / active (K,)."""
        p = np.asarray(poses, dtype=np.float64)
        if self.K:
            self.boxes[e], self.active[e] = boxes, active
            p = np.concatenate([p, self.parked(boxes, active)])
        self.sims[e].env_restart(p)
        if self.K:
            self.sims[e].toggle_list[self.A:] = 4.0

    def step(self, act, noise=None, envs=None):
        """One step with the lap logic of every env (or of `envs`); the parked agents get the action (0, 0)."""
        sims = self.sims if envs is None else [self.sims[e] for e in envs]
        if self.K:
            assert noise is None
            act = np.concatenate([act, np.zeros((act.shape[0], self.K, 2))], axis=1)
        self.oracle.step_batch(sims, act, noise=noise, env_level=True)

    def gather(self, field, envs=None, chunk=2048):
        """oracle.gather of the cars (slots 0 .. A-1), in chunks of envs."""
        sims = self.sims if envs is None else [self.sims[e] for e in envs]
        out = []
        for i in range(0, len(sims), chunk):
            g = self.oracle.gather(sims[i:i + chunk], field)
            out.append(g[:, :self.A] if g.ndim > 1 else g)
        return np.concatenate(out) if out else np.zeros((0,))


def check_scans(got, fin, pre, noise, where):
    """got (fp32) against the oracle's scans fin and its scans before the opponent ray-cast pre; returns occluded beams."""
    occ = fin < pre
    want32 = fin.astype(np.float32)
    if noise:
        bad = (~occ) & (np.abs(got - want32) > np.spacing(np.abs(want32)))
    else:
        bad = (~occ) & (got != want32)
    assert not bad.any(), (where, 'scan', [(tuple(i), float(got[tuple(i)]), fin[tuple(i)]) for i in np.argwhere(bad)[:5]])
    d = np.where(occ, np.abs(got.astype(np.float64) - fin), 0.0)
    assert d.max(initial=0.0) <= TOL_OCCLUDED, (where, 'occluded beams', d.max(), np.unravel_index(np.argmax(d), d.shape))
    return int(occ.sum())


def compare(sim, world, where, done=None, skip_wall=None, noise=False):
    """Every env of sim against world: scans of the slots that have a lidar (the others NaN), collisions, collision_idx, wall
    flags (but for the envs in skip_wall: an auto-reset clears them), done (the oracle's, or `done`), lap counts and times,
    state, toggles and env time.  Returns the tick's event counts."""
    N, A, B = sim.num_envs, sim.num_agents, sim.num_beams
    on = [i for i in range(A) if sim.lidar[i]]
    off = [i for i in range(A) if not sim.lidar[i]]
    got = cpu(sim.scans).reshape(N, A, B)
    ev = dict(occluded=0)
    if off:
        assert np.isnan(got[:, off]).all(), (where, 'sensorless rows')
    if on:
        fin, pre = world.gather('scans'), world.gather('scans_pre')
        ev['occluded'] = check_scans(got[:, on], fin[:, on], pre[:, on], noise, where)
        del fin, pre
    del got
    col, cidx, wall = world.gather('collisions'), world.gather('collision_idx'), world.gather('in_collision')
    assert np.array_equal(cpu(sim.collisions).reshape(N, A), col), (where, 'collisions')
    gi = cpu(sim.collision_idx).reshape(N, A).astype(np.float64)
    assert np.array_equal(gi, cidx), (where, 'collision_idx', np.argwhere(gi != cidx)[:5])
    keep = np.ones(N, bool) if skip_wall is None else ~skip_wall
    gw = cpu(sim.wall_flag).reshape(N, A)
    assert np.array_equal(gw[keep], wall[keep]), (where, 'wall flags', np.argwhere(gw[keep] != wall[keep])[:5])
    want_done = world.gather('done') if done is None else done
    assert np.array_equal(cpu(sim.done).astype(np.float64), want_done), (where, 'done')
    assert np.array_equal(cpu(sim.lap_counts).reshape(N, A), world.gather('lap_counts')), (where, 'lap_counts')
    dl = np.abs(cpu(sim.lap_times).reshape(N, A) - world.gather('lap_times')).max()
    assert dl <= 1e-9, (where, 'lap_times', dl)
    st = cpu(sim.state).reshape(7, N, A).transpose(1, 2, 0)
    ds = np.abs(st - world.gather('state'))
    assert ds.max() <= TOL_STATE, (where, 'state', ds.max(), np.unravel_index(np.argmax(ds), ds.shape))
    assert np.array_equal(cpu(sim.toggle_list).reshape(N, A), world.gather('toggle_list')), (where, 'toggles')
    assert np.abs(cpu(sim.current_time) - world.gather('current_time')).max() <= 1e-12, (where, 'env time')
    if world.K:
        assert np.array_equal(cpu(sim.obstacle_boxes), world.boxes), (where, 'boxes')
        assert np.array_equal(cpu(sim.obstacle_active), world.active), (where, 'active slots')
    ev['gjk'] = int(((cidx >= 0) & (cidx < A)).sum())
    ev['box'] = int((cidx >= A).sum())
    ev['wall'] = int(wall.sum())
    ev['wall_sensorless'] = int(wall[:, off].sum()) if off else 0
    return ev


def add(total, ev):
    for k, v in ev.items():
        total[k] = total.get(k, 0) + v


def assert_events(ev, *names):
    print('events:', ev)
    for k in names:
        assert ev.get(k, 0) > 0, ('no %s within the run' % k, ev)


# ----------------------------------------------------------------------------- setups
def example_case(f110, example_map, n, seed):
    """example_map, raceline population (bench starts, close trains, cars facing a wall), the waypoint start table."""
    wp = f110.maps.load_waypoints()
    poses = raceline_population(f110, example_map.host, np.random.default_rng(seed), n, 2)
    return example_map, [example_map.host], np.zeros(n, int), poses, [wp]


@functools.lru_cache(maxsize=1)
def _box_candidates():
    import f1tenth_gym_b200 as f110
    wp = f110.maps.load_waypoints()
    cand = f110.obstacle_candidates(wp[:, :2], 4096, lateral=(-0.8, 0.8), seed=AR_SEED)
    cand[:, 2] = np.where(cand[:, 2] < 0, cand[:, 2] + 2 * np.pi, cand[:, 2])
    return cand


def box_candidates(f110):
    """Car-sized boxes along the waypoints, yaws wrapped into [0, 2 pi) as the dynamics' single-shot wrap leaves a parked
    agent's yaw (so that the box and the oracle's parked car have the same vertices)."""
    return _box_candidates()


def make_sim(f110, dev, dmap, ids, poses, noise=0.0, boxes=False, mask=None, max_ticks=None):
    N, A = poses.shape[:2]
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=N, device=dev, noise_std=noise)
    layers = getattr(dmap, 'layers', [])
    sim.set_device_map(dmap, env_map_ids=ids if len(layers) > 1 else None)
    sim.env_reset(poses)
    if boxes:
        # as tools/bench_obstacles.py: empty slots, the draw, a first respawn around the start poses
        sim.set_obstacles(np.zeros((K_BOX, 5)), np.zeros(K_BOX, bool))
        sim.set_obstacle_draw(box_candidates(f110), **BOX_DRAW)
        sim.respawn_obstacles()
    if mask is not None:
        sim.set_lidar(mask)
    if max_ticks is not None:
        sim.set_episodes(max_ticks)
    return sim


def make_world(f110, hosts, ids, poses, sim, rotated_maps=False):
    omaps = [(rotated.omap_of if rotated_maps else omap_of)(h) for h in hosts]
    if sim.obstacle_boxes is None:
        return World(omaps, ids, poses)
    return World(omaps, ids, poses, cpu(sim.obstacle_boxes), cpu(sim.obstacle_active))


def restart_env(f110, world, tables, ids, tick, e):
    """The device's restart of env e at tick counter `tick`: the start-pose draw from its layer's table and, with boxes, the
    respawn draw around the new positions."""
    from f1tenth_gym_b200.obstacles import respawn_draw
    p = autoreset_poses(tables[ids[e]], AR_SEED, tick, int(e), world.A, POSE_GAP)
    if world.K:
        bx, ac = respawn_draw(box_candidates(f110), p[:, :2], world.K, BOX_DRAW['count'], BOX_DRAW['clearance'],
                              BOX_DRAW['seed'], tick, int(e))
        world.restart(e, p, bx, ac)
    else:
        world.restart(e, p)


# ----------------------------------------------------------------------------- the drivers
def run_autoreset(f110, dev, case, sim, world, drive, ticks=T, repeat=1, seed=1, on_first=None, twin=None, per_call=None):
    """`ticks` physics ticks with lap logic and auto-reset: drive 'graph' (a captured graph of one call, tick_repeat(repeat)
    when repeat > 1) or 'tick'.  The oracle steps every tick, restarts the envs whose ego collided at the device's draw, and is
    compared with the device after every call; with repeat > 1 done_any / done_tick against the oracle's per-tick done.  twin:
    a simulator without the lidar mask, ticked alike and compared bit for bit.  per_call(call): extra checks after a call."""
    dmap, hosts, ids, poses, tables = case
    N, A = poses.shape[:2]
    rng = np.random.default_rng(seed)
    tab_dev = torch.from_numpy(np.ascontiguousarray(tables[0])).to(dev)
    if drive == 'graph':
        abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
        sim.capture_graph(abuf, autoreset_poses=tab_dev, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True,
                          repeat=repeat)
        if on_first:
            on_first()
    ev = dict(resets=0, mid_call_done=0)
    counter = 0
    for call in range(ticks // repeat):
        act = random_actions(rng, N, A)
        if drive == 'graph':
            abuf.copy_(torch.from_numpy(act.reshape(N * A, 2)))
            sim.replay()
        else:
            sim.tick(act, autoreset_poses=tab_dev, pose_gap=POSE_GAP, seed=AR_SEED)
            if call == 0 and on_first:
                on_first()
            if twin is not None:
                twin.tick(act, autoreset_poses=tab_dev, pose_gap=POSE_GAP, seed=AR_SEED)
        torch.cuda.synchronize()
        assert int(sim.tick_counter.item()) == counter + repeat, call
        if twin is not None:
            check_twins(sim, twin, sim.lidar, call)
        dones = []
        for j in range(repeat):
            counter += 1
            world.step(act)
            dones.append(world.gather('done') != 0)
            if j < repeat - 1:      # the intermediate ticks' events (the last tick's come from compare)
                cidx, wall = world.gather('collision_idx'), world.gather('in_collision')
                add(ev, dict(gjk=int(((cidx >= 0) & (cidx < A)).sum()), box=int((cidx >= A).sum()), wall=int(wall.sum())))
            reset = world.gather('collisions')[:, 0] != 0
            for e in np.flatnonzero(reset):
                restart_env(f110, world, tables, ids, counter, e)
            ev['resets'] += int(reset.sum())
        where = 'call %d' % call
        add(ev, compare(sim, world, where, skip_wall=reset))
        if repeat > 1:
            d = np.stack(dones)
            first = np.where(d.any(0), d.argmax(0), -1)
            assert np.array_equal(cpu(sim.done_any) != 0, d.any(0)), (where, 'done_any')
            assert np.array_equal(cpu(sim.done_tick), first), (where, 'done_tick')
            ev['mid_call_done'] += int(((first >= 0) & (first < repeat - 1)).sum())
        if per_call is not None:
            per_call(call)
    return ev


def run_episodes(f110, dev, case, sim, world, max_ticks, ticks=T, seed=1, noise=0.0, on_first=None, laps_at=3,
                 rotated_maps=False):
    """`ticks` episode ticks through a captured graph against the oracle episode driver: an env ends when the oracle says done
    (terminated) or its own tick count reaches max_ticks (truncated); terminated, truncated, episode_length and every final_*
    buffer are compared with the oracle before the restart; the env then restarts at the restated draw and takes one
    zero-action step alone (noise of counter t | 2^63); done stays the plain tick's.  At call laps_at every fifth env's toggles
    are set to 4 on both sides: from a start pose a car cannot leave the start zone within the run, so its lap logic
    completes there and the env ends on all_done."""
    dmap, hosts, ids, poses, tables = case
    N, A, B = sim.num_envs, sim.num_agents, sim.num_beams
    ipa = (B + 31) // 32
    rng = np.random.default_rng(seed)
    tab_dev = [torch.from_numpy(np.ascontiguousarray(t)).to(dev) for t in tables]
    abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
    sim.capture_graph(abuf, autoreset_poses=tab_dev if len(tab_dev) > 1 else tab_dev[0], pose_gap=POSE_GAP,
                      autoreset_seed=AR_SEED, env_level=True)
    d = record(f110)
    if on_first:
        on_first(d)
    restart_warps = int(d['restart_grid']) * TTC_WARPS
    on = [i for i in range(A) if sim.lidar[i]]
    ep_t = np.zeros(N, np.int64)
    ev = dict(terminated=0, truncated=0, collided=0, laps=0, restarted=0, bulk=0, max_listed=0, gjk_tick=0, box_tick=0)
    for call in range(ticks):
        if call == laps_at:
            lap_envs = np.arange(0, N, 5)
            sim.toggle_list.view(N, A)[torch.from_numpy(lap_envs).to(dev)] = 4.0
            for e in lap_envs:
                world.sims[e].toggle_list[:A] = 4.0
        act = random_actions(rng, N, A)
        abuf.copy_(torch.from_numpy(act.reshape(N * A, 2)))
        sim.replay()
        torch.cuda.synchronize()
        tick = int(sim.tick_counter.item())
        assert tick == call + 1, call
        where = 'tick %d' % call
        # the plain tick
        nz = philox_ref.tick_noise(sim.c.noise_seed, tick, N * A, B, noise).reshape(N, A, B) if noise > 0 else None
        world.step(act, noise=nz)
        del nz
        # contacts of the plain tick (an ego contact ends the episode: after the restart it is gone)
        cidx = world.gather('collision_idx')
        ev['gjk_tick'] += int(((cidx >= 0) & (cidx < A)).sum())
        ev['box_tick'] += int((cidx >= A).sum())
        done = world.gather('done')
        ep_t += 1
        term = done != 0
        trunc = ~term & (ep_t >= max_ticks)
        ended = np.flatnonzero(term | trunc)
        assert np.array_equal(cpu(sim.terminated) != 0, term), (where, 'terminated')
        assert np.array_equal(cpu(sim.truncated) != 0, trunc), (where, 'truncated')
        assert np.array_equal(cpu(sim.episode_length)[ended], ep_t[ended]), (where, 'episode_length')
        listed = int(sim.ep_list_count.item())
        assert listed == ended.size, (where, 'restart list', listed, ended.size)
        ev['max_listed'] = max(ev['max_listed'], listed)
        if listed * A * ipa > restart_warps:
            ev['bulk'] += 1
        # the final observation: what the plain tick left, before the restart
        if ended.size:
            fs = cpu(sim.final_state).reshape(7, N, A)[:, ended].transpose(1, 2, 0)
            assert np.abs(fs - world.gather('state', ended)).max() <= TOL_STATE, (where, 'final_state')
            col = world.gather('collisions', ended)
            assert np.array_equal(cpu(sim.final_collisions).reshape(N, A)[ended], col), (where, 'final_collisions')
            assert np.array_equal(cpu(sim.final_collision_idx).reshape(N, A)[ended].astype(np.float64),
                                  world.gather('collision_idx', ended)), (where, 'final_collision_idx')
            assert np.array_equal(cpu(sim.final_lap_counts).reshape(N, A)[ended], world.gather('lap_counts', ended)), \
                (where, 'final_lap_counts')
            assert np.abs(cpu(sim.final_lap_times).reshape(N, A)[ended] - world.gather('lap_times', ended)).max() <= 1e-9, \
                (where, 'final_lap_times')
            if on:
                fsc = cpu(sim.final_scans).reshape(N, A, B)[ended][:, on]
                check_scans(fsc, world.gather('scans', ended)[:, on], world.gather('scans_pre', ended)[:, on], noise > 0,
                            (where, 'final_scans'))
            ev['collided'] += int((col[:, 0] != 0).sum())
            ev['laps'] += int((world.gather('toggle_list', ended) >= 4).all(1).sum())
        ev['terminated'] += int(term.sum())
        ev['truncated'] += int(trunc.sum())
        ev['restarted'] += int(ended.size)
        # the restart: the draw, then one zero-action step of the ended envs alone
        for e in ended:
            restart_env(f110, world, tables, ids, tick, e)
        if ended.size:
            rz = None
            if noise > 0:
                idx = ((ended[:, None, None] * A + np.arange(A)[None, :, None]) * B + np.arange(B)[None, None, :])
                rz = noise * philox_ref.normal_sample(sim.c.noise_seed, tick | (1 << 63), idx.astype(np.uint64))
            world.step(np.zeros((ended.size, A, 2)), noise=rz, envs=ended)
        ep_t[ended] = 0
        assert np.array_equal(cpu(sim.episode_ticks), ep_t), (where, 'episode_ticks')
        add(ev, compare(sim, world, where, done=done, noise=noise > 0))
    print('restart list: up to %d envs, %d ticks with more items than the %d warps of the restart grid'
          % (ev['max_listed'], ev['bulk'], restart_warps))
    assert ev['bulk'] > 0, ('the restart march never ran more items than its grid has warps', ev, restart_warps)
    return ev


def is_lean_dyn(d, ipt):
    return d.get('march') == 'lean' and d.get('DYN') == '1' and d.get('IPT') == str(ipt)


# ----------------------------------------------------------------------------- 1. boxes
def test_boxes_graph_with_autoreset_and_respawn(f110, dev, sms, example_map):
    """16384 x 2 (on 132 SMs), four car-sized boxes per env redrawn at every auto-reset, a captured graph with the lap logic:
    the lean DYN kernel with four entries per ticket, k_tail2 without its env level (several envs per block, a partial last
    block), then k_obstacles and k_env_tail_obst with the respawn draw."""
    n = int(16384 * sms / 132)
    case = example_case(f110, example_map, n, 201)
    sim = make_sim(f110, dev, example_map, case[2], case[3], boxes=True)
    world = make_world(f110, case[1], case[2], case[3], sim)

    def first():
        d = expect_path(f110, {'march': 'lean', 'CELLS': 1, 'DYN': 1, 'IPT': 4, 'tail': 'k_tail2', 'obst': K_BOX})
        epb = int(d['epb'])
        assert epb > 1 and n % epb != 0 and int(d['tail_grid']) == -(-n // epb), d
    ev = run_autoreset(f110, dev, case, sim, world, 'graph', seed=202, on_first=first)
    assert_events(ev, 'gjk', 'occluded', 'wall', 'resets', 'box')


# ----------------------------------------------------------------------------- 2. lidar masks
@pytest.mark.parametrize('mask', ['ego', 'none', 'alternating'])
def test_lidar_mask_tick_with_autoreset(f110, dev, sms, example_map, mask):
    """f110_tick with a lidar mask and auto-reset: [True, False] at 16384 x 2 (the DYN kernel planned on the masked queue,
    built by k_lidar_order), [False, False] at 4096 x 2 (no march at all) and [True, False, True, False] at 4096 x 4.
    Against the oracle, against an unmasked twin bit for bit, and with more k_march_ttc items than its grid has warps."""
    A = 4 if mask == 'alternating' else 2
    m = {'ego': [True, False], 'none': [False, False], 'alternating': [True, False, True, False]}[mask]
    n = int((16384 if mask == 'ego' else 4096) * sms / 132)
    wp = f110.maps.load_waypoints()
    poses = raceline_population(f110, example_map.host, np.random.default_rng(300 + A), n, A)
    case = (example_map, [example_map.host], np.zeros(n, int), poses, [wp])
    sim = make_sim(f110, dev, example_map, case[2], poses, mask=m)
    twin = make_sim(f110, dev, example_map, case[2], poses)
    world = make_world(f110, case[1], case[2], poses, sim)
    S = sum(m)
    ipa = (sim.num_beams + 31) // 32
    grid = {}

    def first():
        if S:
            want = {'march': 'lean', 'DYN': 1, 'tail': 'k_lidar_cast+k_tail_noscan', 'lidar': '%d/%d' % (S, A)}
            if mask == 'ego':
                want['IPT'] = 2
            d = expect_path(f110, want)
        else:
            d = expect_path(f110, {'march': 'none', 'tail': 'k_tail_noscan', 'lidar': '0/%d' % A})
        record(f110)
        grid['warps'] = int(d['grid']) * TTC_WARPS       # the last grid= of the record: k_march_ttc's
        grid['listed'] = []

    def listed(call):
        grid['listed'].append(int(sim.lidar_list_count.item()))
    ev = run_autoreset(f110, dev, case, sim, world, 'tick', seed=310 + A, on_first=first, twin=twin, per_call=listed)
    most = max(grid['listed'])
    print('listed sensorless agents per tick', grid['listed'], 'k_march_ttc warps', grid['warps'])
    assert most * ipa > grid['warps'], (most, ipa, grid['warps'])
    assert_events(ev, 'gjk', 'wall_sensorless', 'resets', *(('occluded',) if S else ()))


# ----------------------------------------------------------------------------- 3. tick_repeat
@pytest.mark.parametrize('variant', ['plain', 'boxes', 'mask'])
def test_repeat_graph_at_bench_size(f110, dev, sms, example_map, variant):
    """A captured tick_repeat(a, 4) at 16384 x 2: plain, with four boxes, and with the mask [True, False].  Every call is four
    oracle ticks; done_any / done_tick against the oracle's per-tick done; more k_march_ttc items than its grid has warps on
    the intermediate ticks."""
    R = 4
    n = int(16384 * sms / 132)
    case = example_case(f110, example_map, n, 400 + len(variant))
    sim = make_sim(f110, dev, example_map, case[2], case[3], boxes=variant == 'boxes',
                   mask=[True, False] if variant == 'mask' else None)
    world = make_world(f110, case[1], case[2], case[3], sim)
    ipa = (sim.num_beams + 31) // 32
    grid = {}

    def first():
        want = {'repeat': R, 'sub': 'ttc', 'UNITS': 'cells'}
        if variant == 'boxes':
            want['obst'] = K_BOX
        if variant == 'mask':
            want['lidar'] = '1/2'
        d = expect_path(f110, want)
        record(f110)
        grid['warps'] = int(d['grid']) * TTC_WARPS
        grid['listed'] = []

    def listed(call):
        grid['listed'].append(int(cpu(sim.repeat_list_count)[:R - 1].max()))
    ev = run_autoreset(f110, dev, case, sim, world, 'graph', repeat=R, seed=410 + len(variant), on_first=first, per_call=listed)
    print('most agents listed on an intermediate tick, per call', grid['listed'], 'k_march_ttc warps', grid['warps'])
    assert max(grid['listed']) * ipa > grid['warps'], (grid, ipa)
    assert_events(ev, 'gjk', 'occluded', 'wall', 'resets', 'mid_call_done', *(('box',) if variant == 'boxes' else ()))


# ----------------------------------------------------------------------------- 4. episodes
RESTART = 'k_episode_end+k_episode_dyn+k_restart_march+k_episode_cast+k_episode_tail'


@pytest.mark.parametrize('variant', ['noise', 'mask_boxes', 'tracks4', 'rotated'])
def test_episodes_graph_with_bulk_restarts(f110, dev, sms, example_map, variant):
    """A captured episode tick with max_ticks = 6 over 12 ticks: the time limit truncates most envs on ticks 6 and 12 together,
    walls and collisions terminate others, and the lap logic completes for some.  example_map at 16384 x 2 with scan noise (the
    full path) and with the mask [True, False] plus boxes with their redraw (the combination of tools/bench_episodes.py's
    record); the metre-unit stack of four tracks with per-layer start tables and a rotated map at 4096 x 2."""
    A, MAX_TICKS = 2, 6
    rng = np.random.default_rng(500 + len(variant))
    rot = variant == 'rotated'
    if variant in ('noise', 'mask_boxes'):
        case = example_case(f110, example_map, int(16384 * sms / 132), 510 + len(variant))
    else:
        n = int(4096 * sms / 132)
        if rot:
            maps = [rotated.load(f110, dev, 'berlin', '.png', rotated.YAWS['berlin'])]
            dmap = maps[0]
        else:
            maps = [f110.DeviceMap.from_yaml(os.path.join(MAPS, name + '.yaml'), ext, dev) for name, ext in TRACKS]
            dmap = f110.DeviceMap.stack(maps)
        hosts = [m.host for m in maps]
        ids = np.arange(n) % len(hosts)
        poses = (rotated.population if rot else mixed_population)(hosts, ids, rng, A)
        tables = [(rotated.start_table if rot else start_table)(h, rng) for h in hosts]
        case = (dmap, hosts, ids, poses, tables)
    noise = 0.01 if variant == 'noise' else 0.0
    boxes = variant == 'mask_boxes'
    sim = make_sim(f110, dev, case[0], case[2], case[3], noise=noise, boxes=boxes,
                   mask=[True, False] if boxes else None, max_ticks=MAX_TICKS)
    world = make_world(f110, case[1], case[2], case[3], sim, rotated_maps=rot)

    def first(d):
        want = {'restart': RESTART + ('+k_episode_obstacles' if boxes else '')}
        if variant == 'noise':
            want.update({'march': 'lean', 'DYN': '1', 'IPT': '4', 'NOISE': '1', 'tail': 'k_tail2'})
        elif boxes:
            want.update({'march': 'lean', 'DYN': '1', 'tail': 'k_lidar_cast+k_tail_noscan', 'obst': str(K_BOX), 'lidar': '1/2'})
        elif rot:
            want.update({'march': 'lean-rot', 'ROT': '1'})
        else:
            want.update({'march': 'lean-het', 'HET': '1', 'layers': '4', 'CELLS': '0'})
        for k, v in want.items():
            assert d.get(k) == v, ('launch record does not show %s=%s' % (k, v), d)
    ev = run_episodes(f110, dev, case, sim, world, MAX_TICKS, seed=520 + len(variant), noise=noise, on_first=first,
                      rotated_maps=rot)
    assert_events(ev, 'terminated', 'truncated', 'collided', 'laps', 'wall', 'gjk_tick', 'occluded',
                  *(('box_tick', 'wall_sensorless') if boxes else ()))
