"""Simulator.predict (C ABI f110_predict, csrc/predict.cuh) on the GPU.

  * Twin simulator: every sample's recorded states and final state equal, bit for bit (NaN as bits), those of a replica
    Simulator of M * K envs x 1 agent into which the source rows (state, steer FIFO, parameter row, map layer) were copied and
    which is stepped H times with actions[:, :, h]; wall_step is the first tick of the replica's wall flag.  Over every map kind
    (cell units, metres, a four-track canvas stack, a five-map mixed-resolution stack, a rotated map, a rotated mixed stack), RK4 and Euler,
    lidar_dist 0 and 0.275, 270 / 1080 / 2160 beams, per-env parameters from set_param_draw and H in {1, 7, 40}; sources with
    full FIFOs at mixed speeds near walls, freshly reset agents (steer_cnt 0 and 1) and one agent at absurd coordinates; action
    sets that drive a stated share of the samples into a wall inside the horizon; device ids out of range give NaN rows.
  * The oracle: a few hundred samples against one-agent oracle sims with state, FIFO and parameters written in: states within
    1e-9 (the last-ulp trig differences smoke() allows), equal wall steps, and clearance equal to the oracle's lookup.
  * Side effects: every Simulator buffer is unchanged by a call, two calls agree, a captured graph of step + predict replays equal
    to the eager calls.
  * Scale: M = 4096 egos of cfg3's layout, K = 256, H = 20 against a sensorless replica.
"""
import zlib

import numpy as np
import pytest
import torch

import test_gpu_rotated as rotated
from test_gpu_multimap import MAPS, TRACKS, mixed_population
from test_predict_host import oracle_dt_lookup

pytestmark = pytest.mark.gpu

BUFFERS = ('state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'march_rec', 'wall_flag', 'collisions', 'collision_idx',
           'current_time', 'lap_times', 'lap_counts', 'toggle_list', 'near_starts', 'start_xs', 'start_ys', 'start_thetas',
           'start_rot', 'done', 'checkpoint_done', 'tick_counter', 'scans', 'params_dev', 'march_cost', 'march_order', 'march_count')


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def kinds(f110, dev):
    """name -> (device map, host maps of its layers, population kind)."""
    import os

    def plain(name, ext='.png'):
        return f110.DeviceMap.from_yaml(os.path.join(MAPS, name + '.yaml'), ext, dev)
    em, be = plain('example_map'), plain('berlin')
    tr = [plain(n, e) for n, e in TRACKS]
    rb = rotated.load(f110, dev, 'berlin', '.png', rotated.YAWS['berlin'])
    rs = [rb, rotated.load(f110, dev, 'vegas', '.png'), rotated.load(f110, dev, 'skirk', '.png', rotated.YAWS['skirk']),
          rotated.load(f110, dev, 'example_map', '.png', rotated.YAWS['example_map'], 0.0625)]
    mix = [em, be, tr[1], tr[2], tr[3]]
    return {'example_map': (em, [em.host], 'plain'), 'berlin': (be, [be.host], 'plain'),
            'rotated': (rb, [rb.host], 'rot'), 'tracks4': (f110.DeviceMap.stack(tr), [m.host for m in tr], 'plain'),
            'mixres5': (f110.DeviceMap.stack(mix[:5], mixed_resolution=True), [m.host for m in mix[:5]], 'plain'),
            'rot4': (f110.DeviceMap.stack(rs, mixed_resolution=True, rotated_origins=True), [m.host for m in rs], 'rot')}


def bits(t):
    return t.view(torch.int64) if t.dtype == torch.float64 else t.view(torch.int32) if t.dtype == torch.float32 else t


def same_bits(x, y):
    return torch.equal(bits(x.contiguous()), bits(y.contiguous()))


def make_sim(f110, dev, dm, N, A, layers, beams=1080, integrator=1, lidar_dist=0.0):
    from f1tenth_gym_b200.simulator import Integrator
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 7, num_envs=N, device=dev, num_beams=beams, lidar_dist=lidar_dist,
                         integrator=Integrator.RK4 if integrator == 1 else Integrator.Euler)
    sim.set_device_map(dm, env_map_ids=layers if getattr(dm.c, 'num_layers', 1) > 1 else None)
    return sim


def source(f110, dev, kinds, name, A, rng, beams=1080, integrator=1, lidar_dist=0.0, per_env=False, ticks=30):
    """A noise-free source: random-action ticks (FIFOs full, speeds mixed, some cars at walls), then envs 0 / 1 reset (steer_cnt
    0) and env 1 ticked once more with the rest (steer_cnt 1 there), and one agent moved to absurd coordinates."""
    dm, hosts, kind = kinds[name]
    N = 12
    layers = np.arange(N) % len(hosts)
    sim = make_sim(f110, dev, dm, N, A, layers, beams, integrator, lidar_dist)
    pop = rotated.population if kind == 'rot' else mixed_population
    poses = pop(hosts, layers, rng, A)
    sim.reset(poses)
    if per_env:
        sim.set_param_draw({'mu': (0.7, 1.3), 'm': (2.8, 4.6), 'C_Sf': (4.0, 5.5), 'a_max': (7.0, 10.5)}, seed=3)
        sim.redraw_params()
    for t in range(ticks):
        sim.step(np.stack([rng.uniform(-0.4189, 0.4189, (N, A)), rng.uniform(-2, 9, (N, A))], axis=2))
    m = np.zeros(N, bool)
    m[:2] = True
    sim.reset(poses, env_mask=m)            # steer_cnt 0 in envs 0 and 1 ...
    a1 = torch.arange(A, device=dev) + A    # ... and env 1 as after one tick at rest: one command queued
    sim.steer_cnt[a1] = 1
    sim.steer_buf[0, a1] = torch.as_tensor(rng.uniform(-0.4, 0.4, A), device=dev)
    return sim, layers


def candidate_actions(rng, M, K, H):
    """A third of the samples at full speed straight on (walls within the horizon for many), a third random, a third near rest."""
    steer = rng.uniform(-0.4189, 0.4189, (M, K, H))
    speed = rng.uniform(-3, 10, (M, K, H))
    k3 = K // 3
    steer[:, :k3] = rng.uniform(-0.05, 0.05, (M, k3, 1))
    speed[:, :k3] = 20.0
    speed[:, 2 * k3:] = rng.uniform(-0.3, 0.3, (M, K - 2 * k3, H))
    return np.ascontiguousarray(np.stack([steer, speed], axis=3))


def replica(f110, dev, src, dm, layers, ids, K, beams, integrator, lidar_dist):
    """M * K envs x 1 agent with the source rows copied in."""
    M = ids.size
    A = src.num_agents
    rep = make_sim(f110, dev, dm, M * K, 1, np.repeat(layers[ids // A], K), beams, integrator, lidar_dist)
    a = torch.as_tensor(np.repeat(ids, K), device=dev, dtype=torch.long)
    rep.state.copy_(src.state[:, a])
    rep.steer_buf.copy_(src.steer_buf[:, a])
    rep.steer_cnt.copy_(src.steer_cnt[a])
    rep.update_params(src.param_table.reshape(-1, 18)[a].reshape(M * K, 1, 18))
    return rep


def run_replica(rep, actions):
    M, K, H = actions.shape[:3]
    states, walls = [], []
    for h in range(H):
        rep.step(actions[:, :, h].reshape(M * K, 1, 2))
        states.append(rep.state.t().clone())
        walls.append(rep.wall_flag.clone())
    st = torch.stack(states, 1).reshape(M, K, H, 7)
    w = torch.stack(walls, 1).reshape(M, K, H) != 0
    first = torch.where(w.any(2), w.int().argmax(2), torch.full_like(w[..., 0], -1, dtype=torch.int64))
    return st, first.int()


CASES = [('example_map', 1, 1080, 1, 0.0, False, 7), ('example_map', 2, 270, 2, 0.275, True, 40),
         ('example_map', 4, 2160, 1, 0.275, False, 1), ('berlin', 2, 1080, 1, 0.0, True, 7), ('berlin', 1, 270, 2, 0.275, False, 40),
         ('rotated', 2, 1080, 1, 0.275, False, 7), ('rotated', 4, 2160, 2, 0.0, True, 7),
         ('tracks4', 2, 1080, 1, 0.0, False, 40), ('tracks4', 4, 270, 2, 0.275, True, 1),
         ('mixres5', 2, 1080, 2, 0.275, True, 7), ('mixres5', 1, 2160, 1, 0.0, False, 40),
         ('rot4', 2, 1080, 1, 0.0, True, 40), ('rot4', 4, 270, 2, 0.275, False, 7)]


@pytest.mark.parametrize('name,A,beams,integrator,lidar_dist,per_env,H', CASES)
def test_twin_simulator(f110, dev, kinds, name, A, beams, integrator, lidar_dist, per_env, H):
    rng = np.random.default_rng(zlib.crc32(('%s %d %d %d' % (name, A, beams, H)).encode()))
    src, layers = source(f110, dev, kinds, name, A, rng, beams, integrator, lidar_dist, per_env)
    NA = src.num_envs * A
    src.state[0, NA - 1] = 3.0e12           # absurd coordinates: the literal march, in both
    src.state[1, NA - 1] = -2.0e12
    src.state[3, 2 * A::2] = 7.0            # every other agent outside envs 0 / 1 at speed: walls within reach of the horizon
    cnt = src.steer_cnt.cpu().numpy()
    assert (cnt == 0).any() and (cnt == 1).any() and (cnt == 2).any()
    K = 12
    ids = np.arange(NA)
    act = candidate_actions(rng, NA, K, H)
    out = src.predict(act, record_states=True, record_clearance=True)
    rep = replica(f110, dev, src, kinds[name][0], layers, ids, K, beams, integrator, lidar_dist)
    st, first = run_replica(rep, torch.as_tensor(act, device=dev))
    assert same_bits(out['states'], st), (name, int((bits(out['states']) != bits(st)).sum()))
    assert same_bits(out['final_state'], st[:, :, -1])
    assert torch.equal(out['wall_step'], first)
    hit = (first >= 0).float().mean().item()
    print('%s: %.3f of the samples hit a wall within %d steps' % (name, hit, H))
    assert hit < 1.0
    if H == 40:
        assert hit >= 0.01, hit             # the march path is exercised
    assert torch.isfinite(out['clearance'][:-1]).all() and (out['clearance'] >= 0).all()
    # device ids out of range: NaN states and clearance, wall_step -1; the other rows as before
    bad = torch.tensor([-1, NA, 5, 2 ** 31 - 1], dtype=torch.int32, device=dev)
    o2 = src.predict(torch.as_tensor(act[[0, 1, 5, 2]], device=dev), agent_ids=bad, record_states=True, record_clearance=True)
    for r in (0, 1, 3):
        assert torch.isnan(o2['states'][r]).all() and torch.isnan(o2['clearance'][r]).all() and (o2['wall_step'][r] == -1).all()
    assert same_bits(o2['states'][2], st[5])


def test_against_the_oracle(f110, dev, kinds):
    import oracle
    rng = np.random.default_rng(11)
    dm, hosts, _ = kinds['example_map']
    for lidar_dist, integrator in ((0.0, 1), (0.275, 2)):
        src, _ = source(f110, dev, kinds, 'example_map', 2, rng, 1080, integrator, lidar_dist, per_env=True)
        NA = src.num_envs * 2
        src.state[3, 4::2] = 7.0
        K, H = 12, 25
        act = candidate_actions(rng, NA, K, H)
        out = src.predict(act, record_states=True, record_clearance=True)
        states, walls, clear = (out['states'].cpu().numpy(), out['wall_step'].cpu().numpy(), out['clearance'].cpu().numpy())
        st0, buf0, cnt0 = src.state.cpu().numpy(), src.steer_buf.cpu().numpy(), src.steer_cnt.cpu().numpy()
        prm = src.param_table.reshape(-1, 18).cpu().numpy()
        h = hosts[0]
        om = oracle.OracleMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.0))
        hits = 0
        for a in range(NA):
            for k in range(K):
                o = oracle.OracleSim(om, num_agents=1, num_beams=1080, integrator=integrator, lidar_dist=lidar_dist)
                o.state[0] = st0[:, a]
                o.steer_buf[0] = buf0[:, a]
                o.steer_cnt[0] = cnt0[a]
                o.params[0] = prm[a]
                first = -1
                for s in range(H):
                    o.step(act[a, k, s][None])
                    # CUDA's sin / cos / tan and the host libm may differ in the last ulp (dynamics.cuh): 1e-9, as smoke()
                    assert np.abs(o.state[0] - states[a, k, s]).max() < 1e-9, (a, k, s)
                    if o.in_collision[0] and first < 0:
                        first = s
                    if lidar_dist == 0.0:       # the clearance rule at the predicted pose, exactly
                        x, y = states[a, k, s, 0], states[a, k, s, 1]
                        assert clear[a, k, s] == np.float32(oracle_dt_lookup(h, x, y)), (a, k, s)
                assert walls[a, k] == first, (a, k)
                hits += first >= 0
        assert hits > 0


def test_no_side_effects_and_graph(f110, dev, kinds):
    rng = np.random.default_rng(5)
    src, _ = source(f110, dev, kinds, 'tracks4', 2, rng, ticks=20)
    NA = src.num_envs * 2
    act = torch.as_tensor(candidate_actions(rng, NA, 16, 10), device=dev)
    before = {b: getattr(src, b).clone() for b in BUFFERS if getattr(src, b, None) is not None}
    o1 = {k: v.clone() for k, v in src.predict(act, record_states=True, record_clearance=True).items()}
    torch.cuda.synchronize()
    for b, t in before.items():
        assert same_bits(getattr(src, b), t), b
    o2 = src.predict(act, record_states=True, record_clearance=True)
    for k in o1:
        assert same_bits(o1[k], o2[k]), k
    # a captured graph of step + predict against the eager calls on a twin
    twin, _ = source(f110, dev, kinds, 'tracks4', 2, np.random.default_rng(5), ticks=20)
    step_act = torch.as_tensor(np.stack([rng.uniform(-0.4, 0.4, (src.num_envs, 2)), rng.uniform(0, 6, (src.num_envs, 2))], 2),
                               device=dev).reshape(NA, 2).contiguous()
    src.step(step_act)                     # warm-up outside the capture
    twin.step(step_act)
    src.predict(act, record_states=True)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        src.step(step_act)
        gout = src.predict(act, record_states=True)
    g.replay()
    twin.step(step_act)
    eager = twin.predict(act, record_states=True)
    torch.cuda.synchronize()
    assert same_bits(src.state, twin.state)
    for k in ('final_state', 'wall_step', 'states'):
        assert same_bits(gout[k], eager[k]), k


def test_scale_cfg3(f110, dev):
    """M = 4096 egos of cfg3's layout (16384 envs x 2 agents, example_map), K = 256, H = 20, against a sensorless replica."""
    import os
    dm = f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', dev)
    rng = np.random.default_rng(3)
    N, A, K, H = 16384, 2, 256, 20
    sim = make_sim(f110, dev, dm, N, A, None)
    sim.reset(mixed_population([dm.host], np.zeros(N, int), rng, A))
    for t in range(20):
        sim.step(np.stack([rng.uniform(-0.4189, 0.4189, (N, A)), rng.uniform(0, 8, (N, A))], axis=2))
    ids = np.sort(rng.choice(N, 4096, replace=False)) * A
    act = torch.as_tensor(candidate_actions(rng, ids.size, K, H), device=dev)
    out = sim.predict(act, agent_ids=ids)
    fs, ws = out['final_state'].clone(), out['wall_step'].clone()
    rep = replica(f110, dev, sim, dm, np.zeros(N, int), ids, K, 1080, 1, 0.0)
    rep.set_lidar([False])
    walls = []
    for h in range(H):
        rep.step(act[:, :, h].reshape(-1, 1, 2))
        walls.append(rep.wall_flag.clone())
    w = torch.stack(walls, 1).reshape(ids.size, K, H) != 0
    first = torch.where(w.any(2), w.int().argmax(2), torch.full_like(w[..., 0], -1, dtype=torch.int64)).int()
    assert same_bits(fs, rep.state.t().reshape(ids.size, K, 7))
    assert torch.equal(ws, first)
    assert (ws >= 0).any()
