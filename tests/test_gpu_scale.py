"""The CUDA tick against the CPU oracle at benchmark batch sizes, on every kernel the launch logic of step_impl picks there.

step_impl (csrc/f110_b200.cu) chooses its kernels from the batch size: the dynamic queue tail of the lean march kernel
once every block has `dyn_ahead` static runs, two or four queue entries per ticket from the queue entries per warp, 2 x
1024-thread blocks for long non-dynamic queues (stacked maps), the envs per block of k_tail2 from the occupancy query, and
the fused tail by agents per env.  The small-batch parity tests never reach most of these paths.  Every case here is sized
from the SM count, asserts through f110_debug_last_launch that it reached the path it covers (and fails with the record
if not), and compares EVERY env with the oracle (oracle.step_batch, threaded) at every tick:

  state <= 1e-9; collisions, collision_idx, wall flags, done, toggles and lap counts exact; lap times <= 1e-9;
  beams the opponent ray-cast did not shorten == fp32(oracle); occluded beams <= 4e-6;
  with scan noise: within one fp32 ulp of fp32(oracle + numpy noise) (tests/philox_ref.py), wall flags exact.

Cases with auto-reset restate the device's draw (mix64 over seed, tick, env; tick = the device tick counter after the
tick), check that every collided env sits exactly on its drawn start poses, and restart the oracle env there
(orc_env_restart).  Populations mix bench starts (gap 23), close trains (gap 3-5) and cars facing a wall from a few
centimetres, so that GJK contacts, opponent occlusion, iTTC wall hits and auto-resets all happen within the ticks.
"""
import os

import numpy as np
import pytest
import torch

import philox_ref

pytestmark = pytest.mark.gpu

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
TOL_STATE = 1e-9
TOL_OCCLUDED = 4e-6
T = 12                    # > 1: later ticks run on a queue ordered by the previous tick's costs
POSE_GAP = 23
AR_SEED = 12345           # bench.py SEED (rank 0)
M64 = (1 << 64) - 1


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
def example_map(f110, dev):
    return f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', dev)


@pytest.fixture(autouse=True)
def default_launch_settings(f110):
    """Every case runs the production launch logic; the debug switches are put back to their defaults before and after."""
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


def cpu(t):
    return t.detach().cpu().numpy()


# ----------------------------------------------------------------------------- sizing (step_impl's thresholds)
def envs_for_per_warp(per_warp, A, B, sms):
    """Envs whose queue gives `per_warp` entries per warp of the default 4 x 512-thread launch (items / (16 * 4 * SMs))."""
    ipa = (B + 31) // 32
    return -(-per_warp * 16 * 4 * sms // (ipa * A))


def last_launch(f110):
    rec = f110._native.lib().f110_debug_last_launch().decode()
    print('launch record:', rec)
    return rec, dict(kv.split('=', 1) for kv in rec.split())


def expect_path(f110, want, check=None):
    """Asserts the launch record of the last tick: `want` maps keys to values; `check(rec dict)` extra conditions."""
    rec, d = last_launch(f110)
    for k, v in want.items():
        assert d.get(k) == str(v), 'launch record does not show %s=%s: %s' % (k, v, rec)
    if check is not None:
        assert check(d), 'launch record: %s' % rec
    return d


# ----------------------------------------------------------------------------- populations
def near_wall_poses(h, rng, n):
    """Poses a few centimetres (0.18-0.21 m of distance transform: the front bumper is 0.165 m ahead of the centre) from a
    wall, heading into it: the iTTC check fires within a few ticks of throttle."""
    gy, gx = np.gradient(h.dt)
    cells = np.argwhere((h.dt >= 0.18) & (h.dt <= 0.21) & (np.hypot(gx, gy) > 0))
    sel = cells[rng.choice(cells.shape[0], n, replace=n > cells.shape[0])]
    r, c = sel[:, 0], sel[:, 1]
    yaw = np.arctan2(-gy[r, c], -gx[r, c]) + rng.uniform(-0.2, 0.2, n)
    return np.stack([(c + 0.5) * h.resolution + h.orig_x, (r + 0.5) * h.resolution + h.orig_y,
                     np.mod(yaw, 2 * np.pi)], axis=1)


def raceline_population(f110, h, rng, N, A):
    """Envs in thirds: bench starts (gap 23), close trains (gap 3-5), every car facing a wall from a few centimetres."""
    wp = f110.maps.load_waypoints()
    k = rng.integers(0, wp.shape[0], N)
    gap = np.where(np.arange(N) % 3 == 0, POSE_GAP, 3 + (np.arange(N) // 3) % 3)
    poses = np.stack([wp[(k - gap * i) % wp.shape[0]] for i in range(A)], axis=1)
    wall = np.arange(N) % 3 == 2
    poses[wall] = near_wall_poses(h, rng, int(wall.sum()) * A).reshape(-1, A, 3)
    return poses


def free_space_population(h, rng, N, A):
    """Metre maps (no raceline): as test_rollout_other_maps_vs_oracle, a car in free space with the others 0.45 m
    ahead-left of it; every third env faces a wall from a few centimetres instead."""
    free = np.argwhere(h.dt > 0.6)
    sel = free[rng.choice(free.shape[0], N, replace=False)]
    poses = np.zeros((N, A, 3))
    poses[:, 0, 0] = sel[:, 1] * h.resolution + h.orig_x + 0.011
    poses[:, 0, 1] = sel[:, 0] * h.resolution + h.orig_y + 0.017
    poses[:, 0, 2] = rng.uniform(0, 2 * np.pi, N)
    for i in range(1, A):
        poses[:, i] = poses[:, 0] + np.array([0.45, 0.1, 0.3]) * i
    wall = np.arange(N) % 3 == 2
    poses[wall] = near_wall_poses(h, rng, int(wall.sum()) * A).reshape(-1, A, 3)
    return poses


def random_actions(rng, N, A):
    return np.stack([rng.uniform(-0.4189, 0.4189, (N, A)), rng.uniform(0, 8, (N, A))], axis=2)


# ----------------------------------------------------------------------------- the device auto-reset, restated
def mix64(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def autoreset_poses(wp, seed, tick, env, A, gap):
    """autoreset_one (csrc/f110_b200.cu): k = floor(u * K) with u from mix64(seed, tick, env); agent i -> wp[k - gap * i]."""
    K = wp.shape[0]
    h = mix64((seed + 0x9E3779B97F4A7C15 * (tick + 1) + 0xD1B54A32D192ED03 * (env + 1)) & M64)
    k = min(int(float(h >> 11) * (1.0 / 9007199254740992.0) * K), K - 1)
    return np.stack([wp[(k - gap * i) % K] for i in range(A)])


# ----------------------------------------------------------------------------- the comparison
def omap_of(h):
    import oracle
    return oracle.OracleMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.0))


def run_vs_oracle(f110, dev, dmap, omaps, poses, drive, B=1080, env_map_ids=None, autoreset=False, env_level=False,
                  noise_std=0.0, count=False, seed=1, on_first_tick=None, fov=4.7, params=None, time_step=0.01,
                  integrator=1, lidar_dist=0.0, ego_idx=0, march_item_beams=32, ticks=T):
    """Runs T ticks of the CUDA path (drive: 'graph' = a CUDA graph captured as bench.measure_workload does, 'tick' =
    f110_tick, 'step' = f110_step) and of one oracle sim per env; compares every env at every tick.  fov, params (body size
    included), time_step, integrator (1 RK4, 2 Euler), lidar_dist and ego_idx go to both sides alike (ticks: how many); the simulator takes
    the map's theta_dis, eps and max_range (the oracle maps must be built with the same).  Returns counts of GJK contacts,
    occluded beams, wall hits and auto-resets, and of the ticks where only the ego (when it is not agent 0) or only agent 0
    collided in an env."""
    import oracle
    N, A = poses.shape[:2]
    NA = N * A
    rng = np.random.default_rng(seed)
    params = f110.maps.DEFAULT_PARAMS if params is None else params
    sim = f110.Simulator(params, A, AR_SEED, time_step=time_step, ego_idx=ego_idx, integrator=integrator,
                         lidar_dist=lidar_dist, num_envs=N, num_beams=B, fov=fov, device=dev, noise_std=noise_std,
                         count_lookups=count, march_item_beams=march_item_beams, theta_dis=int(dmap.c.theta_dis))
    sim.set_device_map(dmap, env_map_ids=env_map_ids)
    sim.env_reset(poses)
    ids = np.zeros(N, int) if env_map_ids is None else np.asarray(env_map_ids)
    osims = [oracle.OracleSim(omaps[ids[e]], params=params, num_agents=A, num_beams=B, fov=fov, timestep=time_step,
                              integrator=integrator, lidar_dist=lidar_dist, ego_idx=ego_idx) for e in range(N)]
    for e in range(N):
        osims[e].env_restart(poses[e])
    wp_np = f110.maps.load_waypoints()
    wp = torch.from_numpy(wp_np).to(dev) if autoreset else None
    if drive == 'graph':
        abuf = torch.zeros((NA, 2), dtype=torch.float64, device=dev)
        sim.capture_graph(abuf, autoreset_poses=wp, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=env_level)
        if on_first_tick:
            on_first_tick()
    n_gjk = n_occ = n_wall = n_reset = n_ego_only = n_zero_only = 0
    for t in range(ticks):
        act = random_actions(rng, N, A)
        if drive == 'graph':
            abuf.copy_(torch.from_numpy(act.reshape(NA, 2)))
            sim.replay()
        elif drive == 'tick':
            sim.tick(act, env_level=env_level, autoreset_poses=wp, pose_gap=POSE_GAP, seed=AR_SEED)
        else:
            sim.step(act)
        torch.cuda.synchronize()
        if t == 0 and on_first_tick and drive != 'graph':
            on_first_tick()
        tick = int(sim.tick_counter.item())
        noise = philox_ref.tick_noise(sim.c.noise_seed, tick, NA, B, noise_std).reshape(N, A, B) if noise_std > 0 else None
        oracle.step_batch(osims, act, noise=noise, env_level=env_level)
        where = 'tick %d' % t
        # ---- scans: beams the opponent ray-cast did not shorten are fp32(oracle) (one ulp with noise), the others 4e-6
        got = cpu(sim.scans).reshape(N, A, B)
        fin, pre = oracle.gather(osims, 'scans'), oracle.gather(osims, 'scans_pre')
        occ = fin < pre
        want32 = fin.astype(np.float32)
        if noise is None:
            bad = (~occ) & (got != want32)
        else:
            bad = (~occ) & (np.abs(got - want32) > np.spacing(np.abs(want32)))
        assert not bad.any(), (where, 'scan', [(tuple(i), float(got[tuple(i)]), fin[tuple(i)]) for i in np.argwhere(bad)[:5]])
        d_all = np.where(occ, np.abs(got.astype(np.float64) - fin), 0.0)
        if d_all.max() > TOL_OCCLUDED:
            e, i, b = np.unravel_index(np.argmax(d_all), d_all.shape)
            st_e = oracle.gather(osims, 'state')[e]
            pytest.fail(str((where, 'occluded beams', d_all.max(), 'env %d agent %d beam %d: got %r oracle %r before the '
                             'ray-cast %r' % (e, i, b, float(got[e, i, b]), fin[e, i, b], pre[e, i, b]), 'oracle state',
                             st_e.tolist(), 'wall', oracle.gather(osims, 'in_collision')[e].tolist(), 'beams off',
                             int((d_all > TOL_OCCLUDED).sum()))))
        n_occ += int(occ.sum())
        # ---- collisions, wall flags, env level (before the auto-reset touches anything)
        col = oracle.gather(osims, 'collisions')
        assert np.array_equal(cpu(sim.collisions).reshape(N, A), col), (where, 'collisions', np.argwhere(cpu(sim.collisions).reshape(N, A) != col)[:5])
        cidx = oracle.gather(osims, 'collision_idx')
        assert np.array_equal(cpu(sim.collision_idx).reshape(N, A).astype(np.float64), cidx), (where, 'collision_idx')
        n_gjk += int((cidx >= 0).sum())
        wall = oracle.gather(osims, 'in_collision')
        n_wall += int(wall.sum())
        if env_level:
            assert np.array_equal(cpu(sim.done).astype(np.float64), oracle.gather(osims, 'done')), (where, 'done')
            assert np.array_equal(cpu(sim.lap_counts).reshape(N, A), oracle.gather(osims, 'lap_counts')), (where, 'lap_counts')
            dl = np.abs(cpu(sim.lap_times).reshape(N, A) - oracle.gather(osims, 'lap_times')).max()
            assert dl <= 1e-9, (where, 'lap_times', dl)
        if ego_idx != 0:
            n_ego_only += int(((col[:, ego_idx] != 0) & (col[:, 0] == 0)).sum())
            n_zero_only += int(((col[:, 0] != 0) & (col[:, ego_idx] == 0)).sum())
        # ---- auto-reset: the envs whose ego collided sit exactly on the restated draw; the oracle env restarts there (an
        # env where only another agent collided goes on, and the state comparison below holds it to that)
        reset = np.zeros(N, bool)
        if autoreset:
            reset = col[:, ego_idx] != 0
            st = cpu(sim.state).reshape(7, N, A)
            for e in np.flatnonzero(reset):
                p = autoreset_poses(wp_np, AR_SEED, tick, int(e), A, POSE_GAP)
                assert np.array_equal(st[[0, 1, 4], e].T, p) and not st[[2, 3, 5, 6], e].any(), (where, 'auto-reset pose', e)
                osims[e].env_restart(p)
            n_reset += int(reset.sum())
        assert np.array_equal(cpu(sim.wall_flag).reshape(N, A)[~reset], wall[~reset]), (where, 'wall flags')
        # ---- state, toggles, env time (after the auto-reset)
        st = cpu(sim.state).reshape(7, N, A).transpose(1, 2, 0)
        ds = np.abs(st - oracle.gather(osims, 'state')).max()
        assert ds <= TOL_STATE, (where, 'state', ds, np.unravel_index(np.argmax(np.abs(st - oracle.gather(osims, 'state'))), st.shape))
        if env_level:
            assert np.array_equal(cpu(sim.toggle_list).reshape(N, A), oracle.gather(osims, 'toggle_list')), (where, 'toggles')
            assert np.abs(cpu(sim.current_time) - oracle.gather(osims, 'current_time')).max() <= 1e-12, (where, 'env time')
    if count:
        assert sim.lookups() == int(oracle.gather(osims, 'nlook').sum())
    return dict(gjk=n_gjk, occluded=n_occ, wall=n_wall, resets=n_reset, ego_only=n_ego_only, agent0_only=n_zero_only)


def assert_events(n, gjk=True, occluded=True, wall=True, resets=True):
    print('events:', n)
    for k, on in (('gjk', gjk), ('occluded', occluded), ('wall', wall), ('resets', resets)):
        if on:
            assert n[k] > 0, ('no %s within %d ticks' % (k, T), n)


def is_lean(d, cells=1, layered=0, dyn=1):
    return d.get('march') == 'lean' and d.get('CELLS') == str(cells) and d.get('LAYERED') == str(layered) and \
        d.get('DYN') == str(dyn)


# ----------------------------------------------------------------------------- the cases
def test_cfg3_graph_with_autoreset(f110, dev, sms, example_map):
    """The flagship workload as bench.py times it (16384 x 2 on 132 SMs): a captured CUDA graph with env-level logic and
    auto-reset.  Lean DYN kernel with four entries per ticket and the st.release / ld.acquire ring; k_tail2 with several
    envs per block and a partial last block."""
    A = 2
    n = int(16384 * sms / 132)
    assert (n * A * 34) // (16 * 4 * sms) >= 80                # four entries per ticket from 72 per warp, with margin
    poses = raceline_population(f110, example_map.host, np.random.default_rng(11), n, A)

    def check():
        d = expect_path(f110, {'march': 'lean', 'CELLS': 1, 'LAYERED': 0, 'DYN': 1, 'IPT': 4, 'RING': 2, 'PT': 512,
                               'tail': 'k_tail2'})
        epb = int(d['epb'])
        assert epb > 1 and n % epb != 0 and int(d['tail_grid']) == -(-n // epb), d
    ev = run_vs_oracle(f110, dev, example_map, [omap_of(example_map.host)], poses, 'graph', autoreset=True, env_level=True,
                       seed=20, on_first_tick=check)
    assert_events(ev)


def test_cfg2x2_tick_with_autoreset(f110, dev, sms, example_map):
    """4096 x 2: two entries per ticket (27..72 per warp) and k_tail2."""
    A = 2
    n = int(4096 * sms / 132)
    pw = (n * A * 34) // (16 * 4 * sms)
    assert 30 <= pw <= 60, pw
    poses = raceline_population(f110, example_map.host, np.random.default_rng(12), n, A)
    check = lambda: expect_path(f110, {'march': 'lean', 'DYN': 1, 'IPT': 2, 'RING': 2, 'tail': 'k_tail2'})  # noqa: E731
    assert_events(run_vs_oracle(f110, dev, example_map, [omap_of(example_map.host)], poses, 'tick', autoreset=True,
                                env_level=True, seed=21, on_first_tick=check))


def test_cfg2_tick_with_autoreset(f110, dev, sms, example_map):
    """4096 x 1: ticket size by run class (fewer than 27 entries per warp) on the DYN kernel; k_tail<128,8>, 4 envs per
    block."""
    n = int(4096 * sms / 132)
    assert (n * 34) // (16 * 4 * sms) < 24
    poses = raceline_population(f110, example_map.host, np.random.default_rng(13), n, 1)
    check = lambda: expect_path(f110, {'march': 'lean', 'DYN': 1, 'IPT': 0, 'tail': 'k_tail<128,8>', 'epb': 4},  # noqa: E731
                                lambda d: int(d['static_runs']) >= 6)
    assert_events(run_vs_oracle(f110, dev, example_map, [omap_of(example_map.host)], poses, 'tick', autoreset=True,
                                env_level=True, seed=22, on_first_tick=check), gjk=False, occluded=False)


@pytest.mark.parametrize('A,N', [(3, 4096), (4, 2048)])
def test_tail2_three_and_four_agents(f110, dev, example_map, A, N):
    """k_tail2 with several envs per block: its shared-memory task table grows as A (A - 1) per env."""
    poses = raceline_population(f110, example_map.host, np.random.default_rng(14 + A), N, A)
    check = lambda: expect_path(f110, {'tail': 'k_tail2'}, lambda d: int(d['epb']) > 1 and  # noqa: E731
                                int(d['smem']) == int(d['epb']) * A * (A - 1) * 120)
    assert_events(run_vs_oracle(f110, dev, example_map, [omap_of(example_map.host)], poses, 'tick', env_level=True,
                                seed=30 + A, on_first_tick=check), resets=False)


@pytest.mark.parametrize('A,N', [(8, 1024), (32, 64)])
def test_fused_tail_many_agents_with_autoreset(f110, dev, example_map, A, N):
    """k_tail<1024,1> (5 <= A <= 32: one env per block of 32 A threads), auto-reset included; at A = 32 the staging array
    of the auto-reset's start poses is full."""
    poses = raceline_population(f110, example_map.host, np.random.default_rng(40 + A), N, A)
    check = lambda: expect_path(f110, {'tail': 'k_tail<1024,1>', 'epb': 1, 'threads': 32 * A, 'tail_grid': N})  # noqa: E731
    assert_events(run_vs_oracle(f110, dev, example_map, [omap_of(example_map.host)], poses, 'tick', autoreset=True,
                                env_level=True, seed=50 + A, on_first_tick=check))


@pytest.mark.parametrize('B', [270, 2160])
def test_beam_sweep_dynamic_queue(f110, dev, sms, example_map, B):
    """Beam sweep (9 and 68 items per agent) on the DYN kernel: 270 beams with the ticket size by run class (about 15000
    envs on 132 SMs), 2160 beams with two entries per ticket (about 3900 envs)."""
    ipa = (B + 31) // 32
    n = envs_for_per_warp(16 if B == 270 else 31, 1, B, sms)
    pw = (n * ipa) // (16 * 4 * sms)
    ipt = 4 if pw >= 72 else 2 if pw >= 27 else 0
    assert ipt == (0 if B == 270 else 2), pw
    poses = raceline_population(f110, example_map.host, np.random.default_rng(60 + B), n, 1)
    check = lambda: expect_path(f110, {'march': 'lean', 'DYN': 1, 'IPT': ipt, 'per_warp': pw},  # noqa: E731
                                lambda d: int(d['static_runs']) >= 6)
    assert_events(run_vs_oracle(f110, dev, example_map, [omap_of(example_map.host)], poses, 'tick', B=B, seed=70 + B,
                                on_first_tick=check), gjk=False, occluded=False, resets=False)


@pytest.mark.parametrize('name', ['vegas', 'berlin'])
def test_metre_maps_dynamic_kernel(f110, dev, name):
    """0.05 m maps at 2048 x 2: the metre-unit DYN lean kernel (every large run on vegas, the reference's default map)."""
    dmap = f110.DeviceMap.from_yaml(os.path.join(MAPS, name + '.yaml'), '.png', dev)
    assert dmap.host.fast_path == 0
    poses = free_space_population(dmap.host, np.random.default_rng(80), 2048, 2)
    check = lambda: expect_path(f110, {'march': 'lean', 'CELLS': 0, 'LAYERED': 0, 'DYN': 1},  # noqa: E731
                                lambda d: int(d['static_runs']) >= 6)
    assert_events(run_vs_oracle(f110, dev, dmap, [omap_of(dmap.host)], poses, 'tick', env_level=True, seed=81,
                                on_first_tick=check), resets=False)


def _flipped(f110, dev, dmap):
    h = dmap.host
    flipped = f110.maps.HostMap(np.ascontiguousarray(h.dt[::-1, ::-1]), h.resolution, (h.orig_x, h.orig_y, 0.0))
    return f110.DeviceMap(flipped, dev), flipped


def _mirror(h, poses, ids):
    cx, cy = h.orig_x + 0.5 * h.width * h.resolution, h.orig_y + 0.5 * h.height * h.resolution
    out = poses.copy()
    m = ids == 1
    out[m, :, 0] = 2 * cx - poses[m, :, 0]
    out[m, :, 1] = 2 * cy - poses[m, :, 1]
    out[m, :, 2] = np.mod(poses[m, :, 2] + np.pi, 2 * np.pi)
    return out


@pytest.mark.parametrize('name', ['example_map', 'berlin'])
def test_stacked_maps_big_blocks(f110, dev, sms, example_map, name):
    """A map stacked with its 180-degree flip, 4096 x 2 through f110_step: the layered lean kernel with 2 x 1024-thread
    blocks (cell units on example_map, metre units on berlin)."""
    import oracle
    A = 2
    n = int(4096 * sms / 132)
    assert n * A * 34 >= 1.3 * 700 * 2 * sms
    dmap = example_map if name == 'example_map' else f110.DeviceMap.from_yaml(os.path.join(MAPS, name + '.yaml'), '.png', dev)
    h = dmap.host
    dm2, flipped = _flipped(f110, dev, dmap)
    stacked = f110.DeviceMap.stack([dmap, dm2])
    ids = np.arange(n) % 2
    rng = np.random.default_rng(90)
    base = raceline_population(f110, h, rng, n, A) if name == 'example_map' else free_space_population(h, rng, n, A)
    # mirrored envs start at the mirrored pose: the flipped map is the original rotated by pi about the canvas centre
    poses = _mirror(h, base, ids)
    omaps = [omap_of(h), oracle.OracleMap(flipped.dt, h.resolution, (h.orig_x, h.orig_y, 0.0))]
    check = lambda: expect_path(f110, {'march': 'lean', 'CELLS': 1 if name == 'example_map' else 0, 'LAYERED': 1,  # noqa: E731
                                       'DYN': 0, 'PT': 1024, 'MINB': 2, 'grid': 2 * sms})
    assert_events(run_vs_oracle(f110, dev, stacked, omaps, poses, 'step', env_map_ids=ids, seed=91, on_first_tick=check),
                  resets=False)


def test_cfg3_scan_noise(f110, dev, sms, example_map):
    """Default F110Env noise (std 0.01) on the four-entries-per-ticket DYN kernel: the NOISE build, keyed by (seed, tick,
    a B + i); the oracle adds the numpy draw before check_ttc and the opponent ray-cast.  An odd batch: k_tail2's last block
    (env-level phase included) is partial."""
    A = 2
    n = envs_for_per_warp(80, A, 1080, sms) | 1
    poses = raceline_population(f110, example_map.host, np.random.default_rng(100), n, A)
    check = lambda: expect_path(f110, {'march': 'lean', 'DYN': 1, 'IPT': 4, 'NOISE': 1, 'COUNT': 0, 'tail': 'k_tail2'},  # noqa: E731
                                lambda d: int(d['epb']) > 1 and n % int(d['epb']) != 0)
    assert_events(run_vs_oracle(f110, dev, example_map, [omap_of(example_map.host)], poses, 'tick', env_level=True,
                                noise_std=0.01, seed=101, on_first_tick=check), resets=False)


def test_cfg3_lookup_count(f110, dev, sms, example_map):
    """The COUNT build of the four-entries-per-ticket DYN kernel: total DT lookups equal the oracle's."""
    A = 2
    n = envs_for_per_warp(80, A, 1080, sms) | 1
    poses = raceline_population(f110, example_map.host, np.random.default_rng(110), n, A)
    check = lambda: expect_path(f110, {'march': 'lean', 'DYN': 1, 'IPT': 4, 'NOISE': 0, 'COUNT': 1})  # noqa: E731
    assert_events(run_vs_oracle(f110, dev, example_map, [omap_of(example_map.host)], poses, 'step', count=True, seed=111,
                                on_first_tick=check), resets=False)
