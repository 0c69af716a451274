"""k_tail2's opponent ray-cast (phase 2: every task's beams in one flat list per opponent rank, cast by every thread of the block)
against k_tail, the warp-per-agent tail that casts the same beams with its own prologue: scans, state, collisions and the
collision index bit for bit, through the fused tick (lap logic + auto-reset) and through f110_step (env level off).

The population mixes, per env:
  * raceline trains 23 waypoints apart (narrow windows; some opponents out of range on the far side of the track);
  * trains 3 waypoints apart (contacts, rear windows that run from beam 0 or to beam B - 1, wide windows with a cone, and at
    A >= 3 two opponents that shorten the same beams of the ego behind them);
  * opponents at random places on the track (many beyond max_range);
  * cars side by side 0.3 m apart (closer than 1.25 half-diagonals: wide windows with cone = 4);
  * egos turned round towards the train behind them, yaw jittered.
Random actions up to 8 m/s drive some cars into the walls (iTTC hits, whose yaw the cast zeroes).  Block shapes: the default
rule, and shapes forced with f110_debug_set_tail2, down to 32 threads for 128 agents, where every thread casts several batches.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def example_map(f110, dev):
    return f110.DeviceMap.from_yaml(os.path.join(MAPS, 'example_map.yaml'), '.png', dev)


def cpu(t):
    return t.detach().cpu().numpy()


def population(f110, rng, N, A):
    wp = f110.maps.load_waypoints()
    W = wp.shape[0]
    k = rng.integers(0, W, N)
    kind = np.arange(N) % 5
    poses = np.empty((N, A, 3))
    for i in range(A):
        poses[:, i] = wp[(k - 23 * i) % W]
        tr3 = kind == 1
        poses[tr3, i] = wp[(k[tr3] - 3 * i) % W]
        far = kind == 2
        poses[far, i] = wp[rng.integers(0, W, far.sum())] if i else wp[k[far]]
        side = kind == 3
        th = wp[k[side], 2]
        poses[side, i] = wp[k[side]]
        poses[side, i, 0] -= 0.3 * i * np.sin(th)
        poses[side, i, 1] += 0.3 * i * np.cos(th)
        back = kind == 4
        poses[back, i] = wp[(k[back] - 5 * i) % W]
    back = kind == 4
    poses[back, 0, 2] += np.pi + rng.uniform(-0.3, 0.3, back.sum())
    poses[:, :, 2] += rng.uniform(-0.05, 0.05, (N, A))
    return poses


def run(f110, dev, example_map, tail, shape, N, A, seed, fused):
    L = f110._native.lib()
    rng = np.random.default_rng(seed)
    poses = population(f110, rng, N, A)
    T = 12
    acts = np.stack([rng.uniform(-0.4189, 0.4189, (T, N, A)), rng.uniform(0, 8, (T, N, A))], axis=3)
    wp = torch.from_numpy(f110.maps.load_waypoints()).to(dev)
    try:
        L.f110_debug_set_tail(tail)
        if shape is not None:
            L.f110_debug_set_tail2(*shape)
        sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 1, num_envs=N, device=dev)
        sim.set_device_map(example_map)
        sim.env_reset(poses)
        out = []
        for t in range(T):
            if fused:
                sim.tick(acts[t], env_level=True, autoreset_poses=wp, pose_gap=3)
            else:
                sim.step(acts[t])
            if t in (0, 5, T - 1):
                torch.cuda.synchronize()
                out.append([cpu(x).copy() for x in (sim.scans, sim.state, sim.collisions, sim.collision_idx)])
        return out
    finally:
        L.f110_debug_set_tail(8)
        L.f110_debug_set_tail2(256, 64)


CASES = [
    ('cfg3', 16384, None),
    ('odd', 1001, None),
    ('odd_42', 1001, (128, -42)),
    ('odd_8x256', 1001, (256, -8)),
    ('batches', 1001, (32, -128)),
]
PARAMS = [pytest.param(A, N, shape, True, id='tick-%s-A%d' % (case, A)) for case, N, shape in CASES for A in (2, 3, 4)] + \
         [pytest.param(A, 1001, None, False, id='step-odd-A%d' % A) for A in (2, 3, 4)]


@pytest.mark.parametrize('A,N,shape,fused', PARAMS)
def test_tail2_flat_cast_equals_k_tail(f110, dev, example_map, A, N, shape, fused):
    seed = 900 + 10 * A + N % 7
    got = run(f110, dev, example_map, -2, shape, N, A, seed, fused)
    ref = run(f110, dev, example_map, -1, None, N, A, seed, fused)
    for t, (g, r) in enumerate(zip(got, ref)):
        for name, x, y in zip(('scans', 'state', 'collisions', 'collision_idx'), g, r):
            assert np.array_equal(x, y), (t, name, int((x != y).sum()))
    # the population reaches what it is there for: contacts and opponent-shortened beams
    col = ref[-1][2]
    assert (col != 0).any()
