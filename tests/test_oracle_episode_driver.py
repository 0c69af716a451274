"""The oracle episode driver of test_gpu_scale_features, on the CPU: restarting an env (World.restart, orc_env_restart) and then
one zero-action World.step of the restarted envs alone is F110Env.reset of that env (orc_env_reset), on state, scans, collisions,
toggles and the lap fields, with and without parked box agents; the envs that were not restarted do not move.  A bug in the
driver would otherwise pass as agreement between the device and the oracle."""
import os

import numpy as np
import pytest

from test_gpu_scale_features import World

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
FIELDS = ('state', 'scans', 'collisions', 'collision_idx', 'toggle_list', 'lap_times', 'lap_counts')


@pytest.mark.parametrize('K', [0, 3])
def test_restart_and_zero_step_equal_env_reset(K):
    import oracle
    from f1tenth_gym_b200 import maps
    N, A = 6, 2
    omap = oracle.OracleMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png')
    wp = maps.load_waypoints()
    rng = np.random.default_rng(3)

    def poses_at(k):
        return np.stack([wp[(k - 23 * i) % wp.shape[0]] for i in range(A)])

    def boxes_near(p):
        b = np.zeros((K, 5))
        b[:, 0] = p[0, 0] + rng.uniform(-3, 3, K)
        b[:, 1] = p[0, 1] + rng.uniform(-3, 3, K)
        b[:, 2] = rng.uniform(0, 2 * np.pi, K)
        b[:, 3:] = (0.58, 0.31)
        return b

    ks = rng.integers(0, wp.shape[0], N)
    poses = np.stack([poses_at(k) for k in ks])
    boxes = np.stack([boxes_near(p) for p in poses]) if K else None
    active = (rng.random((N, K)) < 0.7).astype(np.uint8) if K else None
    world = World([omap], np.zeros(N, int), poses, boxes, active)
    for _ in range(5):
        world.step(np.stack([rng.uniform(-0.4, 0.4, (N, A)), rng.uniform(1, 6, (N, A))], axis=2))
    ended = np.array([1, 3, 4])
    kept = np.setdiff1d(np.arange(N), ended)
    before = {f: world.gather(f, kept) for f in FIELDS + ('current_time',)}
    new = {int(e): poses_at(int(rng.integers(0, wp.shape[0]))) for e in ended}
    new_boxes = {int(e): boxes_near(new[int(e)]) for e in ended} if K else {}
    new_active = {int(e): (np.arange(K) != 1).astype(np.uint8) for e in ended} if K else {}
    for e in ended:
        world.restart(int(e), new[int(e)], new_boxes.get(int(e)), new_active.get(int(e)))
    world.step(np.zeros((ended.size, A, 2)), envs=ended)
    for f in FIELDS + ('current_time',):
        assert np.array_equal(world.gather(f, kept), before[f]), ('an env that did not restart moved', f)
    for e in ended:
        e = int(e)
        ref = oracle.OracleSim(omap, num_agents=A + K)
        ref.env_reset(np.concatenate([new[e], World.parked(new_boxes[e], new_active[e])]) if K else new[e])
        for f in FIELDS:
            got, want = world.gather(f, [e])[0], oracle.gather([ref], f)[0][:A]
            assert np.array_equal(got, want), (e, f)
        assert world.gather('current_time', [e])[0] == ref.current_time
        if K:
            # the parked agents stay where the restart put them, and their toggles never hold back all_done
            st = oracle.gather([world.sims[e]], 'state')[0][A:]
            assert np.array_equal(st[:, [0, 1, 4]], World.parked(new_boxes[e], new_active[e]))
            assert (world.sims[e].toggle_list[A:] == 4.0).all()
