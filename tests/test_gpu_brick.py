"""The ray march on the 4 x 4-cell brick table (f110_march_tables.dt_cells_brick, k_march_lean_brick) against the same launch
on the padded row-major table (debug variant 90), on the GPU.

  * f110_map_brick builds, bit for bit, the host model maps.brick_table of the padded table;
  * at 4096 x 2 and 16384 x 2 envs, 30 ticks with auto-reset, driven as bench.py drives them (a captured CUDA graph of
    f110_tick_ex): scans, state, collisions and wall flags are bit-identical after every tick, and so are they with scan noise,
    in the lookup-counting build (whose totals must agree too), with eager f110_tick_ex ticks and through
    f110_step_host_async_ex; the launch record shows which table each run read.
"""
import hashlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')
POSE_GAP = 23
SEED = 12345
TICKS = 30
ROW_MAJOR = 90           # debug variant: the default launch on the padded row-major table


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


@pytest.fixture(autouse=True)
def default_variant(f110):
    L = f110._native.lib()
    L.f110_debug_set_variant(0)
    yield
    L.f110_debug_set_variant(0)


def test_device_brick_table_matches_the_host_model(f110, example_map):
    assert example_map.dt_cells_brick is not None
    assert example_map.march_tables.dt_cells_brick == example_map.dt_cells_brick.data_ptr()
    pad = example_map.dt_cells_pad.cpu().numpy()
    assert np.array_equal(pad.view(np.int64), f110.maps.pad_table(example_map.dt_cells.cpu().numpy()).view(np.int64))
    want = f110.maps.brick_table(pad)
    got = example_map.dt_cells_brick.cpu().numpy()
    assert got.shape == want.shape and np.array_equal(got.view(np.int64), want.view(np.int64))


def run(f110, dev, dmap, variant, N, A, drive='graph', noise_std=0.0, count=False):
    """TICKS ticks from bench-style start poses with auto-reset; returns (one digest per tick of scans, state, collisions and
    wall flags, lookup total or None, launch record of the last tick)."""
    L = f110._native.lib()
    L.f110_debug_set_variant(variant)
    NA = N * A
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, SEED, num_envs=N, device=dev, noise_std=noise_std,
                         count_lookups=count)
    sim.set_device_map(dmap)
    wp_np = f110.maps.load_waypoints()
    wp = torch.from_numpy(wp_np).to(dev)
    k = np.random.default_rng(N).integers(0, wp_np.shape[0], N)
    sim.env_reset(np.stack([wp_np[(k - POSE_GAP * i) % wp_np.shape[0]] for i in range(A)], axis=1))
    gen = torch.Generator(device=dev)
    gen.manual_seed(SEED)
    u = torch.rand((TICKS, NA, 2), generator=gen, device=dev, dtype=torch.float64)
    u[..., 0] = -0.4189 + 0.8378 * u[..., 0]
    u[..., 1] = 8.0 * u[..., 1]
    digests = []

    def digest(*arrays):
        h = hashlib.sha1()
        for a in arrays:
            h.update(a.tobytes())
        digests.append(h.hexdigest())

    if drive == 'graph':
        abuf = torch.zeros((NA, 2), dtype=torch.float64, device=dev)
        sim.capture_graph(abuf, autoreset_poses=wp, pose_gap=POSE_GAP, autoreset_seed=SEED, env_level=True)
    if drive == 'async':
        sets = sim.make_host_pipeline(depth=2)
        for t in range(TICKS):
            io = sets[t % 2]
            sim.wait_host(io)
            io['actions'].copy_(u[t].cpu())
            sim.step_host_async(io)
            sim.autoreset(wp, POSE_GAP, SEED)
            sim.wait_host(io)
            digest(io['scans'].numpy(), io['state'].numpy(), io['collisions'].numpy(), sim.wall_flag.cpu().numpy())
    else:
        for t in range(TICKS):
            if drive == 'graph':
                abuf.copy_(u[t])
                sim.replay()
            else:
                sim.tick(u[t].view(N, A, 2), env_level=True, autoreset_poses=wp, pose_gap=POSE_GAP, seed=SEED)
            digest(sim.scans.cpu().numpy(), sim.state.cpu().numpy(), sim.collisions.cpu().numpy(),
                   sim.wall_flag.cpu().numpy())
    torch.cuda.synchronize(dev)
    if drive == 'graph':
        sim.step_profile(u[0].view(N, A, 2))        # one eager step: the launch record of the path the graph replays
    rec = L.f110_debug_last_launch().decode()
    return digests, sim.lookups(), rec


def compare(f110, dev, dmap, N, A, **kw):
    b_dig, b_look, b_rec = run(f110, dev, dmap, 0, N, A, **kw)
    r_dig, r_look, r_rec = run(f110, dev, dmap, ROW_MAJOR, N, A, **kw)
    assert 'layout=brick4x4' in b_rec, b_rec
    assert 'march=lean ' in r_rec and 'layout=' not in r_rec, r_rec
    # the brick path runs the launch the row-major one does (same queue, block shape and ticket size)
    strip = lambda rec: rec.replace(' layout=brick4x4', '')
    assert strip(b_rec) == r_rec, (b_rec, r_rec)
    first = next((t for t in range(TICKS) if b_dig[t] != r_dig[t]), None)
    assert first is None, 'brick and row-major results differ from tick %s' % first
    assert b_look == r_look
    return b_look


@pytest.mark.parametrize('N', [4096, 16384])
def test_brick_equals_row_major_graph(f110, dev, example_map, N):
    compare(f110, dev, example_map, N, 2)


def test_brick_equals_row_major_counted(f110, dev, example_map):
    looks = compare(f110, dev, example_map, 4096, 2, count=True)
    assert looks and looks > 4096 * 2 * 1080 * TICKS


def test_brick_equals_row_major_noise(f110, dev, example_map):
    compare(f110, dev, example_map, 4096, 2, noise_std=0.01)


def test_brick_equals_row_major_eager_tick(f110, dev, example_map):
    compare(f110, dev, example_map, 4096, 2, drive='tick')


def test_graph_equals_eager_tick_on_the_brick(f110, dev, example_map):
    g, _, _ = run(f110, dev, example_map, 0, 4096, 2, drive='graph')
    t, _, rec = run(f110, dev, example_map, 0, 4096, 2, drive='tick')
    assert 'layout=brick4x4' in rec
    assert g == t


def test_brick_equals_row_major_host_async(f110, dev, example_map):
    compare(f110, dev, example_map, 4096, 2, drive='async')


def test_row_major_above_1080_beams(f110, dev, example_map):
    """At more than 1080 beams per scan the march reads the row-major table (measured faster there, DESIGN.md §3.2)."""
    L = f110._native.lib()
    for B, want in ((1080, True), (2160, False)):
        sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, SEED, num_envs=2048, num_beams=B, device=dev)
        sim.set_device_map(example_map)
        wp = f110.maps.load_waypoints()
        sim.env_reset(wp[np.arange(2048) % wp.shape[0]][:, None, :])
        sim.tick(np.zeros((2048, 1, 2)), env_level=True)
        torch.cuda.synchronize(dev)
        rec = L.f110_debug_last_launch().decode()
        assert ('layout=brick4x4' in rec) == want, (B, rec)
