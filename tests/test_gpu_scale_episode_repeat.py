"""Episodes under a held action (f110_tick_repeat_episodes) against the CPU oracle at benchmark batch size.

test_gpu_episode_repeat checks the call against the project's own plain tick at 64 envs.  Here one captured call of K = 4 ticks
runs at 16384 x 2 (on 132 SMs) with four boxes per env redrawn at every restart and the lidar mask [True, False], and every env
is compared with the oracle (oracle.step_batch, test_gpu_scale_features' World driver) after every call, at the tolerances of
test_gpu_scale.run_vs_oracle.  The oracle runs each env tick by tick and stops it at the tick its episode ends -- done
(terminated) or its tick count reaching max_ticks (truncated) -- so the final_* buffers, scans included, are compared with the
oracle's state at that tick, also when it is an intermediate tick of the short path whose scan the call computes afterwards from
its snapshot.  After the K ticks the oracle restarts the ended envs as the device does: the start-pose and box draws at the
counter of the call's last tick, then one zero-action step of those envs alone.  A time limit of 6 ticks truncates most envs on
tick 1 of the second call, so the final-scan pass and the restart run on lists of thousands of envs; the case asserts that both
marches ran more items than their fixed grid has warps, and that ends on an intermediate tick (terminated and truncated), on the
last tick and on tick 0 all fired.
"""
import numpy as np
import pytest
import torch

from test_gpu_scale import (AR_SEED, POSE_GAP, TOL_STATE, default_launch_settings, dev, example_map, f110,  # noqa: F401
                            random_actions, sms)
from test_gpu_scale_features import (K_BOX, TTC_WARPS, add, assert_events, check_scans, compare, cpu, example_case, make_sim,
                                     make_world, restart_env)

pytestmark = pytest.mark.gpu

K = 4                      # ticks per call
CALLS = 3
MAX_TICKS = 6              # not a multiple of K: the truncations land on tick 1 of the second call
REC_BYTES = 768            # g_launch_rec (csrc/f110_b200.cu): a record of REC_BYTES - 1 characters was cut short
RESTART = 'k_episode_restart+k_episode_dyn+k_restart_march+k_episode_cast+k_episode_tail+k_episode_obstacles'
FINAL_SCAN = 'k_restart_march+k_episode_cast+k_episode_obstacles'


def launch_record(f110):
    rec = f110._native.lib().f110_debug_last_launch().decode()
    print('launch record (%d chars): %s' % (len(rec), rec))
    assert len(rec) < REC_BYTES - 1, ('launch record cut short', rec)
    return dict(kv.split('=', 1) for kv in rec.split() if '=' in kv)


def test_repeat_episodes_graph_with_boxes_and_mask_at_bench_size(f110, dev, sms, example_map):
    n = int(16384 * sms / 132)
    case = example_case(f110, example_map, n, 601)
    dmap, hosts, ids, poses, tables = case
    N, A = poses.shape[:2]
    sim = make_sim(f110, dev, dmap, ids, poses, boxes=True, mask=[True, False], max_ticks=MAX_TICKS)
    world = make_world(f110, hosts, ids, poses, sim)
    B = sim.num_beams
    ipa = (B + 31) // 32
    rng = np.random.default_rng(602)
    tab_dev = torch.from_numpy(np.ascontiguousarray(tables[0])).to(dev)
    abuf = torch.zeros((N * A, 2), dtype=torch.float64, device=dev)
    sim.capture_graph(abuf, autoreset_poses=tab_dev, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True, repeat=K)
    d = launch_record(f110)
    want = {'repeat': str(K), 'sub': 'ttc', 'UNITS': 'cells', 'lidar': '1/2', 'obst': str(K_BOX), 'restart': RESTART,
            'final_scan': FINAL_SCAN}
    for k, v in want.items():
        assert d.get(k) == v, ('launch record does not show %s=%s' % (k, v), d)
    warps = int(d['restart_grid']) * TTC_WARPS       # the final-scan pass runs k_restart_march on a grid of the same size
    on, off = [0], [1]
    ep_t = np.zeros(N, np.int64)
    ev = dict(term_mid=0, trunc_mid=0, last=0, first=0, restarted=0, final_bulk=0, restart_bulk=0, gjk_tick=0, box_tick=0,
              occluded_final=0)
    counter = 0
    for call in range(CALLS):
        act = random_actions(rng, N, A)
        abuf.copy_(torch.from_numpy(act.reshape(N * A, 2)))
        sim.replay()
        torch.cuda.synchronize()
        assert int(sim.tick_counter.item()) == counter + K, call
        where = 'call %d' % call
        # the oracle: every env still in its episode steps; an env stops at the tick its episode ends
        end = np.full(N, -1)
        term, trunc = np.zeros(N, bool), np.zeros(N, bool)
        length = np.zeros(N, np.int64)
        done_any, done_tick = np.zeros(N, bool), np.full(N, -1)
        for j in range(K):
            counter += 1
            run = np.flatnonzero(end < 0)
            world.step(act[run], envs=run)
            dj = world.gather('done', run) != 0
            done_any[run] |= dj
            done_tick[run[dj & (done_tick[run] < 0)]] = j
            ep_t[run] += 1
            tr = ~dj & (ep_t[run] >= MAX_TICKS)
            now = run[dj | tr]
            end[now] = j
            term[run[dj]] = True
            trunc[run[tr]] = True
            length[now] = ep_t[now]
            cidx = world.gather('collision_idx', run)
            ev['gjk_tick'] += int(((cidx >= 0) & (cidx < A)).sum())
            ev['box_tick'] += int((cidx >= A).sum())
        ended = np.flatnonzero(end >= 0)
        assert np.array_equal(cpu(sim.end_tick), end), (where, 'end_tick')
        assert np.array_equal(cpu(sim.terminated) != 0, term), (where, 'terminated')
        assert np.array_equal(cpu(sim.truncated) != 0, trunc), (where, 'truncated')
        assert np.array_equal(cpu(sim.episode_length)[ended], length[ended]), (where, 'episode_length')
        assert np.array_equal(cpu(sim.done_any) != 0, done_any), (where, 'done_any')
        assert np.array_equal(cpu(sim.done_tick), done_tick), (where, 'done_tick')
        # the device lists: the envs whose final scan the pass computed, and the restarted envs
        mid = ended[end[ended] < K - 1]
        scan_listed, restart_listed = int(sim.ep_scan_count.item()), int(sim.ep_list_count.item())
        assert scan_listed == mid.size and restart_listed == ended.size, (where, scan_listed, mid.size, restart_listed, ended.size)
        ev['final_bulk'] += int(scan_listed * A * ipa > warps)
        ev['restart_bulk'] += int(restart_listed * A * ipa > warps)
        # the final observation: the oracle's state at each ended env's end tick (it has not stepped since)
        if ended.size:
            fs = cpu(sim.final_state).reshape(7, N, A)[:, ended].transpose(1, 2, 0)
            assert np.abs(fs - world.gather('state', ended)).max() <= TOL_STATE, (where, 'final_state')
            assert np.array_equal(cpu(sim.final_collisions).reshape(N, A)[ended], world.gather('collisions', ended)), \
                (where, 'final_collisions')
            assert np.array_equal(cpu(sim.final_collision_idx).reshape(N, A)[ended].astype(np.float64),
                                  world.gather('collision_idx', ended)), (where, 'final_collision_idx')
            assert np.array_equal(cpu(sim.final_lap_counts).reshape(N, A)[ended], world.gather('lap_counts', ended)), \
                (where, 'final_lap_counts')
            assert np.abs(cpu(sim.final_lap_times).reshape(N, A)[ended] - world.gather('lap_times', ended)).max() <= 1e-9, \
                (where, 'final_lap_times')
            fsc = cpu(sim.final_scans).reshape(N, A, B)[ended]
            ev['occluded_final'] += check_scans(fsc[:, on], world.gather('scans', ended)[:, on],
                                                world.gather('scans_pre', ended)[:, on], False, (where, 'final_scans'))
            assert (fsc[:, off] == 0).all(), (where, 'sensorless final_scans rows written')
            del fsc
        ev['term_mid'] += int((term & (end >= 0) & (end < K - 1)).sum())
        ev['trunc_mid'] += int((trunc & (end >= 0) & (end < K - 1)).sum())
        ev['last'] += int((end == K - 1).sum())
        ev['first'] += int((end == 0).sum())
        ev['restarted'] += int(ended.size)
        done = world.gather('done')       # each env's done on its last tick in the call: an ended env's at its end tick
        # the restart: the draws at the counter of the call's last tick, then one zero-action step of the ended envs alone
        for e in ended:
            restart_env(f110, world, tables, ids, counter, e)
        if ended.size:
            world.step(np.zeros((ended.size, A, 2)), envs=ended)
        ep_t[ended] = 0
        assert np.array_equal(cpu(sim.episode_ticks), ep_t), (where, 'episode_ticks')
        add(ev, compare(sim, world, where, done=done))
    print('final-scan / restart lists against the %d warps of the grid:' % warps, ev)
    assert_events(ev, 'term_mid', 'trunc_mid', 'last', 'first', 'final_bulk', 'restart_bulk', 'gjk_tick', 'box_tick', 'occluded',
                  'occluded_final', 'wall')
