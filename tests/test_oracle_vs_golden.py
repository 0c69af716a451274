"""Pins the CPU oracle (oracle/f110_oracle.c) against the reference's own known-answer vectors and
against golden outputs of the unmodified reference numba path (tests/golden/make_golden.py).

Tolerances: dynamics / state / un-occluded scans are BIT-EXACT (the oracle restates the same fp64
operation order with the same libm); opponent ray-cast and vertices may differ in the last bits
because the reference routes 2-element dot products through BLAS (tolerance 1e-9 m).
"""
import os

import numpy as np
import pytest

import oracle

G = os.path.join(os.path.dirname(__file__), 'golden')
MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')


def g(name):
    return np.load(os.path.join(G, name))


@pytest.fixture(scope='module')
def example_map():
    return oracle.OracleMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png')


def test_reference_dynamics_kat():
    k = g('kat_reference_tests.npz')
    f_ks = oracle.vehicle_dynamics_ks(k['x_ks'], k['u'], k['pvec'])
    f_st = oracle.vehicle_dynamics_st(k['x_st'], k['u'], k['pvec'])
    # dynamic_models.py:277-278 assertAlmostEqual (7 places)
    assert np.max(np.abs(k['f_ks_gt'] - f_ks)) < 5e-8
    assert np.max(np.abs(k['f_st_gt'] - f_st)) < 5e-8


def test_reference_collision_kat():
    k = g('kat_reference_tests.npz')
    col, idx = oracle.collision_multiple(k['multi_vertices'])
    assert np.array_equal(col, k['multi_collisions'])      # [1,1,1,1,1,1,0]
    assert np.array_equal(idx, k['multi_collision_idx'])   # [5,5,5,5,5,4,-1] last writer wins
    for p in k['jitter_pairs']:
        assert oracle.collision(p[0], p[1])


def test_kernel_kats():
    k = g('kat_kernels.npz')
    F = np.stack([oracle.vehicle_dynamics_st(x, u, k['pvec']) for x, u in zip(k['X'], k['U'])])
    assert np.array_equal(F, k['F'])
    pv = k['pvec']
    out = np.array([oracle.pid(r[0], r[1], r[2], r[3], pv[11], pv[13], pv[15], pv[14]) for r in k['pid_in']])
    assert np.array_equal(out, k['pid_out'])
    va = np.stack([oracle.get_vertices(p, 0.58, 0.31) for p in k['pose_a']])
    assert np.max(np.abs(va - k['verts_a'])) < 1e-12
    hit = np.array([oracle.collision(a, b) for a, b in zip(k['verts_a'], k['verts_b'])])
    assert np.array_equal(hit, k['gjk'])
    sa = k['scan_angles']
    for i in range(k['rc_ego'].shape[0]):
        lo, hi = oracle.blocked_view_indices(k['rc_ego'][i], k['rc_opp_verts'][i], sa)
        assert (lo, hi) == tuple(k['rc_window'][i])
        out = oracle.ray_cast(k['rc_ego'][i], k['rc_scan_in'][i].astype(np.float64), sa, k['rc_opp_verts'][i])
        assert np.max(np.abs(out - k['rc_scan_out'][i])) < 1e-9
    ttc = np.array([oracle.check_ttc(s.astype(np.float64), v, k['cosines'], k['side_distances'])
                    for s, v in zip(k['ttc_scan'], k['ttc_vel'])])
    assert np.array_equal(ttc, k['ttc'])
    assert ttc.any() and not ttc.all()


def test_beam_tables_match_reference():
    k = g('kat_kernels.npz')
    sa, co, sd = oracle.beam_tables(1080, 4.7, oracle.DEFAULT_PARAMS)
    assert np.array_equal(sa, k['scan_angles']) and np.array_equal(co, k['cosines'])
    assert np.array_equal(sd, k['side_distances'])


def test_scans_example_map(example_map):
    k = g('scans_example_map.npz')
    for B in (270, 540, 1080, 2160):
        for p, ref in zip(k['poses'], k['scan_%d' % B]):
            assert np.array_equal(oracle.get_scan(example_map, p, B, 4.7), ref)


@pytest.mark.parametrize('name', ['berlin', 'skirk', 'vegas', 'stata_basement'])
def test_scans_other_maps(name):
    k = g('scans_%s.npz' % name)
    m = oracle.OracleMap.from_yaml(os.path.join(MAPS, name + '.yaml'), '.png')
    for p, ref in zip(k['poses'], k['scan_1080']):
        assert np.array_equal(oracle.get_scan(m, p, 1080, 4.7), ref)


@pytest.mark.parametrize('name', ['example_map', 'berlin', 'skirk', 'vegas', 'stata_basement', 'levine'])
def test_scans_wide(name):
    """208 reference scans per map (tests/golden/make_golden_scans_wide.py): on-track, free space, inside walls, hugging the
    map border from both sides, far outside and absurd coordinates."""
    k = g('scans_wide_%s.npz' % name)
    m = oracle.OracleMap.from_yaml(os.path.join(MAPS, name + '.yaml'), '.pgm' if name == 'levine' else '.png')
    assert k['poses'].shape == (208, 3)
    for j, p in enumerate(k['poses']):
        s = oracle.get_scan(m, p, 1080, 4.7)
        if name == 'example_map':
            assert np.array_equal(s, k['scan_1080'][j]), j
        else:
            assert np.array_equal(s[k['beam_idx'][j]], k['scan_1080_sub'][j]), j
    if name == 'example_map':
        for B in (270, 2160):
            for p, ref in zip(k['poses'][:48], k['scan_%d' % B]):
                assert np.array_equal(oracle.get_scan(m, p, B, 4.7), ref)


@pytest.mark.parametrize('name', ['traj_a1_random', 'traj_a2_random', 'traj_a2_close', 'traj_a3_euler', 'traj_a4_train'])
def test_trajectories(example_map, name):
    k = g(name + '.npz')
    E, T, A = k['actions'].shape[:3]
    sim = oracle.OracleSim(example_map, num_agents=A, integrator=int(k['integrator']),
                           lidar_dist=float(k['lidar_dist']))
    ticks = {(int(e), int(t)): i for i, (e, t) in enumerate(k['scan_ticks'])}
    n_col = 0
    for e in range(E):
        sim.reset(k['poses0'][e])
        for t in range(T):
            sim.step(k['actions'][e, t])
            assert np.array_equal(sim.state, k['states'][e, t]), (e, t)
            assert np.array_equal(sim.collisions, k['collisions'][e, t]), (e, t)
            assert np.array_equal(sim.collision_idx, k['collision_idx'][e, t]), (e, t)
            n_col += int(sim.collisions.sum())
            if (e, t) in ticks:
                assert np.max(np.abs(sim.scans - k['scans'][ticks[(e, t)]])) < 1e-9, (e, t)
    if name in ('traj_a2_close', 'traj_a4_train'):      # (a4: four cars nose to tail, make_golden_a4.py)
        assert n_col > 0


@pytest.mark.parametrize('name', ['traj_a1_random', 'traj_a2_random', 'traj_a2_close', 'traj_a3_euler', 'traj_a4_train'])
def test_step_batch_equals_per_sim_step(example_map, name):
    """orc_step_batch (the threaded batch driver of the large-batch GPU tests) over the golden trajectories: every field of
    every env equals the one-sim-at-a-time step, bit for bit, with and without the env-level logic; the optional noise is
    added to the scan before the opponent ray-cast."""
    k = g(name + '.npz')
    E, T, A = k['actions'].shape[:3]
    kw = dict(num_agents=A, integrator=int(k['integrator']), lidar_dist=float(k['lidar_dist']))
    one = [oracle.OracleSim(example_map, **kw) for _ in range(E)]
    bat = [oracle.OracleSim(example_map, **kw) for _ in range(E)]
    for e in range(E):
        one[e].env_reset(k['poses0'][e])
        bat[e].env_reset(k['poses0'][e])
    for t in range(T):
        env_level = t % 2 == 1
        done = []
        for e in range(E):
            one[e].step(k['actions'][e, t])
            done.append(one[e].env_post_step() if env_level else None)
        oracle.step_batch(bat, k['actions'][:, t], env_level=env_level, num_threads=3)
        for f in ('state', 'scans', 'collisions', 'collision_idx', 'in_collision', 'lap_times', 'lap_counts', 'toggle_list'):
            got = oracle.gather(bat, f)
            want = np.stack([getattr(o, f) for o in one]).astype(np.float64)
            assert np.array_equal(got, want), (f, t)
        assert np.array_equal(oracle.gather(bat, 'current_time'), [o.current_time for o in one])
        assert np.array_equal(oracle.gather(bat, 'nlook'), [o.nlook for o in one])
        if env_level:
            assert np.array_equal(oracle.gather(bat, 'done'), np.array(done, dtype=np.float64)), t
    assert np.array_equal(oracle.gather(bat, 'scans'), oracle.gather(one, 'scans'))
    # noise: the scan check_ttc and the opponent ray-cast see is the clean one plus the noise (first tick from rest: no
    # iTTC flag can flip)
    B = 1080
    clean = [oracle.OracleSim(example_map, **kw) for _ in range(E)]
    noisy = [oracle.OracleSim(example_map, **kw) for _ in range(E)]
    for e in range(E):
        clean[e].reset(k['poses0'][e])
        noisy[e].reset(k['poses0'][e])
    nz = np.random.default_rng(1).normal(0.0, 0.01, (E, A, B))
    oracle.step_batch(clean, k['actions'][:, 0])
    oracle.step_batch(noisy, k['actions'][:, 0], noise=nz)
    assert np.array_equal(oracle.gather(noisy, 'scans_pre'), oracle.gather(clean, 'scans_pre') + nz)
    assert np.array_equal(oracle.gather(noisy, 'state'), oracle.gather(clean, 'state'))
    if A == 1:
        assert np.array_equal(oracle.gather(noisy, 'scans'), oracle.gather(noisy, 'scans_pre'))
    occl = oracle.gather(noisy, 'scans') < oracle.gather(noisy, 'scans_pre')
    assert np.array_equal(oracle.gather(noisy, 'scans')[~occl], oracle.gather(noisy, 'scans_pre')[~occl])


def test_env_restart_is_the_device_autoreset():
    """orc_env_restart: Simulator.reset + counters and start frame of F110Env.reset, no zero-action step; done and the
    collision observation of the ending tick stay."""
    m = oracle.OracleMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png')
    from f1tenth_gym_b200 import maps
    wp = maps.load_waypoints()
    s = oracle.OracleSim(m, num_agents=2)
    s.env_reset(wp[[10, 5]])
    for _ in range(5):
        s.step(np.array([[0.3, 6.0], [-0.2, 5.0]]))
        s.env_post_step()
    s.collisions[0] = 1.0
    n0 = s.nlook
    s.env_restart(wp[[40, 17]])
    assert np.array_equal(s.state[:, [0, 1, 4]], wp[[40, 17]]) and not s.state[:, [2, 3, 5, 6]].any()
    assert s.current_time == 0.0 and not s.toggle_list.any() and s.collisions[0] == 1.0
    assert not s.steer_cnt.any() and s.nlook == n0                  # nothing was stepped
    s.step(np.zeros((2, 2)))
    assert not s.env_post_step()                                    # lap logic measured from the new start frame


def test_scans_rotated_origin():
    """A map yaml whose origin has a yaw (0.35 rad): the rotation terms of xy_2_rc (laser_models.py:75-78), which none
    of the bundled maps exercises.  Golden: the reference ScanSimulator2D on example_map.png with that origin."""
    from f1tenth_gym_b200 import maps
    k = g('scans_rotated_origin.npz')
    hm = maps.load_map(os.path.join(MAPS, 'example_map.yaml'), '.png')
    om = oracle.OracleMap(hm.dt, float(k['resolution']), tuple(k['origin']))
    for p, ref in zip(k['poses'], k['scan_1080']):
        assert np.array_equal(oracle.get_scan(om, p, 1080, 4.7), ref)
    assert (k['scan_1080'][:-1] < 29.0).mean() > 0.8 and np.all(k['scan_1080'][-1] == 30.0)     # last pose is off the map


def test_trajectory_with_updated_params(example_map):
    """Simulator.update_params(p2, agent_idx=1) (base_classes.py:514-534): slot 1 integrates with its own parameters and
    ray-casts opponents with its own body size, while GJK keeps the Simulator-level length/width (:536-550) and the
    iTTC side distances stay those of the construction-time parameters."""
    from f1tenth_gym_b200 import maps
    k = g('traj_a2_params.npz')
    E, T, A = k['actions'].shape[:3]
    p2 = dict(maps.DEFAULT_PARAMS, mu=0.8, m=4.5, lf=0.17, lr=0.16, C_Sf=5.1, I=0.05, width=0.28, length=0.50, a_max=7.0)
    sim = oracle.OracleSim(example_map, num_agents=A)
    sim.params[1] = oracle.params_vector(p2)
    ticks = {(int(e), int(t)): i for i, (e, t) in enumerate(k['scan_ticks'])}
    for e in range(E):
        sim.reset(k['poses0'][e])
        for t in range(T):
            sim.step(k['actions'][e, t])
            assert np.array_equal(sim.state, k['states'][e, t]), (e, t)
            assert np.array_equal(sim.collisions, k['collisions'][e, t]), (e, t)
            if (e, t) in ticks:
                assert np.max(np.abs(sim.scans - k['scans'][ticks[(e, t)]])) < 1e-9, (e, t)
    assert k['collisions'].sum() > 0


@pytest.mark.parametrize('name', ['berlin', 'vegas'])
def test_trajectories_other_maps(name):
    """Reference Simulator trajectories on 0.05 m maps (no power-of-two resolution; vegas is the reference's default)."""
    k = g('traj_%s_a2.npz' % name)
    omap = oracle.OracleMap.from_yaml(os.path.join(MAPS, name + '.yaml'), '.png')
    E, T, A = k['actions'].shape[:3]
    sim = oracle.OracleSim(omap, num_agents=A)
    ticks = {(int(e), int(t)): i for i, (e, t) in enumerate(k['scan_ticks'])}
    n_col = n_occluded = 0
    for e in range(E):
        sim.reset(k['poses0'][e])
        for t in range(T):
            sim.step(k['actions'][e, t])
            assert np.array_equal(sim.state, k['states'][e, t]), (e, t)
            assert np.array_equal(sim.collisions, k['collisions'][e, t]), (e, t)
            assert np.array_equal(sim.collision_idx, k['collision_idx'][e, t]), (e, t)
            n_col += int(sim.collisions.sum())
            if (e, t) in ticks:
                assert np.max(np.abs(sim.scans - k['scans'][ticks[(e, t)]])) < 1e-9, (e, t)
                n_occluded += int((sim.scans[0] < 1.5).sum())
    assert n_occluded > 0


def test_env_laps(example_map):
    k = g('env_laps.npz')
    sim = oracle.OracleSim(example_map, num_agents=1)
    done = sim.env_reset(k['pose0'])
    T = k['actions'].shape[0]
    for t in range(T):
        if t > 0:
            sim.step(k['actions'][t])
            done = sim.env_post_step()
        assert np.array_equal(sim.state[0], k['states'][t]), t
        assert np.array_equal(sim.lap_times, k['lap_times'][t]), t
        assert np.array_equal(sim.lap_counts, k['lap_counts'][t]), t
        assert np.array_equal(sim.toggle_list, k['toggles'][t]), t
        assert done == bool(k['done'][t]), t
    assert done and sim.lap_counts[0] == 2.0


def test_env_race2(example_map):
    """BASELINE configs[0] (two pure-pursuit cars in the real F110Env): 2088 ticks, one lap each in the ego's start
    frame, the ego closes in on the slower car (opponent occlusion in its scan) and rams it -> done."""
    k = g('env_race2.npz')
    sim = oracle.OracleSim(example_map, num_agents=2)
    done = sim.env_reset(k['pose0'])
    T = k['actions'].shape[0]
    for t in range(T):
        if t > 0:
            sim.step(k['actions'][t])
            done = sim.env_post_step()
        assert np.array_equal(sim.state, k['states'][t]), t
        assert np.array_equal(sim.collisions, k['collisions'][t]), t
        assert np.array_equal(sim.lap_times, k['lap_times'][t]), t
        assert np.array_equal(sim.lap_counts, k['lap_counts'][t]), t
        assert np.array_equal(sim.toggle_list, k['toggles'][t]), t
        assert done == bool(k['done'][t]), t
    assert done and sim.collisions[0] == 1.0 and np.array_equal(sim.lap_counts, [1.0, 1.0])


CONFIG_MAPS = {'example_map': '.png', 'berlin': '.png'}


@pytest.mark.parametrize('name', sorted(CONFIG_MAPS))
def test_scans_off_default_config(name):
    """ScanSimulator2D(B, fov, eps=, theta_dis=, max_range=) off the defaults (tests/golden/make_golden_configs.py): theta_dis
    1000 / 4000 / 32767, max_range 5 / 40, eps 0.01, fov 0.1 / pi / 6.28 / 7.0 and B 2 / 3 / 33 / 100 / 8224, bit for bit."""
    k = g('kat_configs.npz')
    poses = k['poses_' + name]
    hits = {}
    for j, (B, fov, eps, td, mr) in enumerate(k['configs']):
        B, td = int(B), int(td)
        m = oracle.OracleMap.from_yaml(os.path.join(MAPS, name + '.yaml'), CONFIG_MAPS[name], theta_dis=td, eps=eps,
                                       max_range=mr)
        ref = k['scan_%d_%s' % (j, name)]
        for p, want in zip(poses[:ref.shape[0]], ref):
            got = oracle.get_scan(m, p, B, fov)
            assert np.array_equal(got, want), (str(k['names'][j]), p)
        hits[str(k['names'][j])] = int((ref == mr).sum())
    # the 5 m clamp is reached more often than the default 30 m one, and that more often than the 40 m one
    assert hits['mr5'] > hits['td1000'] >= hits['mr40'] and hits['mr5'] > 0, hits


def test_env_ego1(example_map):
    """F110Env(ego_idx=1) of the reference (tests/golden/env_ego1.npz): the ego's wall crash ends the episode; agent 0's
    wall crash does not, and the lap toggles of both cars run in the ego's start frame."""
    k = g('env_ego1.npz')
    for ep, ego_crash in (('ego_crash_', True), ('opp_crash_', False)):
        sim = oracle.OracleSim(example_map, num_agents=2, ego_idx=1)
        done = sim.env_reset(k[ep + 'pose0'])
        T = k[ep + 'actions'].shape[0]
        for t in range(T):
            if t > 0:
                sim.step(k[ep + 'actions'][t])
                done = sim.env_post_step()
            assert np.array_equal(sim.state, k[ep + 'states'][t]), (ep, t)
            assert np.array_equal(sim.collisions, k[ep + 'collisions'][t]), (ep, t)
            assert np.array_equal(sim.lap_times, k[ep + 'lap_times'][t]), (ep, t)
            assert np.array_equal(sim.lap_counts, k[ep + 'lap_counts'][t]), (ep, t)
            assert np.array_equal(sim.toggle_list, k[ep + 'toggles'][t]), (ep, t)
            assert done == bool(k[ep + 'done'][t]), (ep, t)
        if ego_crash:
            assert done and np.array_equal(sim.collisions, [0.0, 1.0])
        else:
            assert not done and np.array_equal(sim.collisions, [1.0, 0.0]) and sim.toggle_list.any()
    # with the default ego (agent 0) the same actions end the second episode at agent 0's crash
    sim = oracle.OracleSim(example_map, num_agents=2)
    sim.env_reset(k['opp_crash_pose0'])
    ends = []
    for t in range(1, k['opp_crash_actions'].shape[0]):
        sim.step(k['opp_crash_actions'][t])
        ends.append(sim.env_post_step())
    assert any(ends)


def test_oracle_ego_idx_range(example_map):
    with pytest.raises(ValueError):
        oracle.OracleSim(example_map, num_agents=2, ego_idx=2)
    with pytest.raises(ValueError):
        oracle.OracleSim(example_map, num_agents=2, ego_idx=-1)


def test_planner_vs_reference():
    """oracle pure pursuit == reference PurePursuitPlanner.plan (examples/waypoint_follow.py) incl. the
    re-acquire and no-waypoint branches; ulp-level slack for the BLAS dot products in the reference."""
    k = g('kat_planner.npz')
    wp = np.loadtxt(os.path.join(MAPS, 'example_waypoints.csv'), delimiter=';', skiprows=3)
    wx, wy, wv = wp[:, 1].copy(), wp[:, 2].copy(), wp[:, 5].copy()
    out = np.array([oracle.pure_pursuit(wx, wy, wv, p, float(k['tlad']), float(k['vgain']), float(k['wheelbase']))
                    for p in k['poses']])
    assert np.abs(out - k['speed_steer']).max() < 1e-12
    none = (k['speed_steer'][:, 0] == 4.0) & (k['speed_steer'][:, 1] == 0.0)
    assert 10 < none.sum() < 500
    out2 = np.array([oracle.pure_pursuit(wx, wy, wv, p, 2.5, 0.9, float(k['wheelbase'])) for p in k['poses'][:400]])
    assert np.abs(out2 - k['speed_steer_l25']).max() < 1e-12
    # the env_laps golden is the same planner in closed loop: actions[t] = plan(state[t-1])
    e = g('env_laps.npz')
    for t in range(1, 400):
        st = e['states'][t - 1]
        sp, sa = oracle.pure_pursuit(wx, wy, wv, (st[0], st[1], st[4]), 0.82461887897713965, 1.375, 0.17145 + 0.15875)
        assert abs(sa - e['actions'][t, 0, 0]) < 1e-12 and abs(sp - e['actions'][t, 0, 1]) < 1e-12
