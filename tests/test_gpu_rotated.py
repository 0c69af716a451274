"""Maps whose yaml origin has a yaw, on k_march_lean_rot: one rotated map alone, and canvas stacks that hold rotated maps
(DeviceMap.stack(maps, rotated_origins=True)), against the oracle on each env's own map.

Every case asserts its launch record (march=lean-rot ROT=1, layers, block shape, NOISE / COUNT), with the tolerances of
test_gpu_scale.py.  The same seeded runs on k_march_lean_rot and on the literal k_raymarch (debug variant 13, today's path
for a rotated map) are bit-identical, and a mixed batch equals single-map simulators bit for bit.  Poses and start tables
are built in each map's rotated frame and turned into world coordinates.
"""
import math
import os
import shutil

import numpy as np
import pytest
import torch

import test_gpu_multimap
from test_gpu_multimap import MAPS, T, _sim, run_multi
from test_gpu_scale import AR_SEED, POSE_GAP, assert_events, cpu, expect_path, free_space_population, random_actions, \
    run_vs_oracle

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), 'golden')
YAWS = {'berlin': 0.35, 'example_map': 1.9, 'skirk': -0.8}


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


@pytest.fixture(autouse=True)
def default_launch_settings(f110, monkeypatch):
    L = f110._native.lib()

    def defaults():
        L.f110_debug_set_variant(0)
        L.f110_debug_set_chunk(3)
        L.f110_debug_set_dyn(50, 4)
        L.f110_debug_set_ipt(-1, -1, -1, -1)
        L.f110_debug_set_tail(-2)
        L.f110_debug_set_tail2(256, 64)
        L.f110_debug_set_pdl(0)
    # run_multi builds one oracle map per host: give it the host's rotation
    monkeypatch.setattr(test_gpu_multimap, 'omap_of', omap_of)
    defaults()
    yield
    defaults()


def omap_of(h):
    import oracle
    om = oracle.OracleMap(h.dt, h.resolution, (h.orig_x, h.orig_y, 0.0))
    om.orig_c, om.orig_s = h.orig_c, h.orig_s
    om.c.orig_c, om.c.orig_s = h.orig_c, h.orig_s
    return om


def load(f110, dev, name, ext, yaw=0.0, res=None):
    h = f110.maps.load_map(os.path.join(MAPS, name + '.yaml'), ext)
    return f110.DeviceMap(f110.maps.HostMap(h.dt, h.resolution if res is None else res, (h.orig_x, h.orig_y, yaw)), dev)


def to_world(h, p):
    """Poses (..., 3) in the map's own frame (relative to its origin) -> world: x_rot = R(-yaw) (x - orig)."""
    c, s = h.orig_c, h.orig_s
    out = np.empty_like(p)
    out[..., 0] = h.orig_x + (c * p[..., 0] - s * p[..., 1])
    out[..., 1] = h.orig_y + (s * p[..., 0] + c * p[..., 1])
    out[..., 2] = np.mod(p[..., 2] + math.atan2(s, c), 2 * np.pi)
    return out


class _Frame(object):
    """The map's tables at origin (0, 0): the population builders of test_gpu_scale / test_gpu_multimap then return poses in
    the map's own frame."""
    def __init__(self, h):
        self.dt, self.resolution, self.height, self.width = h.dt, h.resolution, h.height, h.width
        self.orig_x = self.orig_y = 0.0


def population(hosts, ids, rng, A):
    poses = np.zeros((ids.size, A, 3))
    for l, h in enumerate(hosts):
        m = ids == l
        poses[m] = to_world(h, free_space_population(_Frame(h), rng, int(m.sum()), A))
    return poses


def start_table(h, rng, K=64):
    return to_world(h, test_gpu_multimap.start_table(_Frame(h), rng, K))


def rot_path(f110, layers, pt=None, noise=0, count=0):
    want = {'march': 'lean-rot', 'ROT': 1, 'layers': layers, 'CELLS': 0, 'NOISE': noise, 'COUNT': count}
    want.update({'HET': 1, 'RES': 1} if layers > 1 else {'HET': 0})
    if pt is not None:
        want.update(PT=pt, MINB=4 if pt == 512 else 2)
    return lambda: expect_path(f110, want)  # noqa: E731


def generated(f110, dev, seed):
    from f1tenth_gym_b200 import trackgen as tg
    m = tg.device_map(tg.random_tracks(seed, 1)[0], dev)
    return m, f110.maps.HostMap(m.dt.cpu().numpy(), m.host.resolution, (m.host.orig_x, m.host.orig_y, 0.0))


@pytest.fixture(scope='module')
def mixed(f110, dev):
    """rotated berlin, vegas, rotated example_map at 0.0625 m, rotated skirk, one generated track."""
    g, gh = generated(f110, dev, 21)
    layers = [load(f110, dev, 'berlin', '.png', YAWS['berlin']), load(f110, dev, 'vegas', '.png'),
              load(f110, dev, 'example_map', '.png', YAWS['example_map'], 0.0625),
              load(f110, dev, 'skirk', '.png', YAWS['skirk']), g]
    hosts = [m.host for m in layers[:4]] + [gh]
    return layers, hosts, f110.DeviceMap.stack(layers, mixed_resolution=True, rotated_origins=True)


# ----------------------------------------------------------------------------- 1. one rotated map, f110_tick
@pytest.mark.parametrize('name', ['example_map', 'berlin'])
@pytest.mark.parametrize('shape', ['4x512', '2x1024'])
def test_single_rotated_map_tick(f110, dev, sms, monkeypatch, name, shape):
    """f110_tick with env level and auto-reset from a start table in the map's rotated frame; sized from the SM count for
    both block shapes."""
    dm = load(f110, dev, name, '.png', YAWS[name])
    h = dm.host
    A = 2
    n = 8 * sms if shape == '4x512' else 24 * sms
    rng = np.random.default_rng(500)
    table = start_table(h, rng)
    monkeypatch.setattr(f110.maps, 'load_waypoints', lambda: table)     # run_vs_oracle's auto-reset table
    poses = population([h], np.zeros(n, int), rng, A)
    ev = run_vs_oracle(f110, dev, dm, [omap_of(h)], poses, 'tick', autoreset=True, env_level=True, seed=501,
                       on_first_tick=rot_path(f110, 1, 512 if shape == '4x512' else 1024))
    assert_events(ev)


# ----------------------------------------------------------------------------- 2. lean-rot == k_raymarch
def _drive(f110, dev, dm, poses, acts, table, variant, count):
    L = f110._native.lib()
    L.f110_debug_set_variant(variant)
    N, A = poses.shape[:2]
    s = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=N, device=dev, noise_std=0.0, count_lookups=count)
    s.set_device_map(dm)
    s.env_reset(poses)
    out = []
    for a in acts:
        if count:
            s.step(a)
        else:
            s.tick(a, autoreset_poses=table, pose_gap=POSE_GAP, seed=AR_SEED)
        rec = L.f110_debug_last_launch().decode()
        assert ('march=lean-rot ROT=1' in rec) == (variant == 0) and ('march=literal' in rec) == (variant == 13), rec
        out.append({f: cpu(getattr(s, f)).copy() for f in ('scans', 'state', 'collisions', 'collision_idx', 'done',
                                                            'lap_times', 'lap_counts', 'toggle_list')})
    return out, (s.lookups() if count else None)


@pytest.mark.parametrize('name', ['example_map', 'berlin'])
def test_lean_rot_equals_raymarch(f110, dev, sms, name):
    dm = load(f110, dev, name, '.png', YAWS[name])
    h = dm.host
    A, n = 2, 4 * sms
    rng = np.random.default_rng(510)
    table = torch.from_numpy(start_table(h, rng)).to(dev)
    poses = population([h], np.zeros(n, int), rng, A)
    acts = [random_actions(rng, n, A) for _ in range(T)]
    resets = 0
    for count in (False, True):
        lean, nl = _drive(f110, dev, dm, poses, acts, table, 0, count)
        lit, nr = _drive(f110, dev, dm, poses, acts, table, 13, count)
        for t, (a, b) in enumerate(zip(lean, lit)):
            for f in a:
                assert np.array_equal(a[f], b[f]), (count, 'tick %d' % t, f)
            resets += int(a['collisions'].reshape(n, A)[:, 0].astype(bool).sum())
        assert nl == nr and (nl is None or nl > 0), (nl, nr)
    assert resets > 0


# ----------------------------------------------------------------------------- 3. the reference golden
def test_golden_rotated_origin_on_the_tick(f110, dev):
    """scans_rotated_origin.npz: the reference's scans at its poses on example_map with a yawed origin.  Cars at rest through
    f110_step, one per env: every beam equals fp32(golden)."""
    k = np.load(os.path.join(G, 'scans_rotated_origin.npz'))
    hm0 = f110.maps.load_map(os.path.join(MAPS, 'example_map.yaml'), '.png')
    dm = f110.DeviceMap(f110.maps.HostMap(hm0.dt, float(k['resolution']), tuple(k['origin'])), dev)
    # (k_dynamics wraps a yaw outside [0, 2 pi] into it, and the scan then starts from the wrapped yaw: those poses are left out)
    keep = (k['poses'][:, 2] >= 0) & (k['poses'][:, 2] <= 2 * np.pi)
    assert keep.sum() >= 5
    poses = np.asarray(k['poses'], dtype=np.float64)[keep]
    want = np.asarray(k['scan_1080'])[keep]
    N = poses.shape[0]
    s = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 3, num_envs=N, device=dev, noise_std=0.0)
    s.set_device_map(dm)
    s.reset(poses[:, None, :])
    s.step(np.zeros((N, 1, 2)))
    expect_path(f110, {'march': 'lean-rot', 'ROT': 1, 'layers': 1})
    st = cpu(s.state).reshape(7, N)
    assert np.array_equal(st[[0, 1, 4]].T, poses)
    assert np.array_equal(cpu(s.scans).reshape(N, -1), want.astype(np.float32))


# ----------------------------------------------------------------------------- 4. guard bands, absurd coordinates
def test_guard_bands_on_every_layer(f110, dev, mixed):
    """The CPU builders of test_rotated_host (x_rot / y_rot within 8 ulps of a cell edge, just below or at W_l res_l and
    H_l res_l, tiny negative, -0.0) on every layer of the mixed stack, cars at rest (f110_step): every beam equals
    fp32(oracle)."""
    from test_rotated_host import rotated_probe_points
    layers, hosts, st = mixed
    rng = np.random.default_rng(520)
    xs, ids = [], []
    for l, h in enumerate(hosts):
        x, y, bands = rotated_probe_points(h, rng, 1000)
        pick = np.concatenate([rng.permutation(v)[:48] for k, v in bands.items() if k not in ('uniform', 'far')])
        xs.append(np.stack([x[pick], y[pick], rng.uniform(0, 2 * np.pi, pick.size)], axis=1))
        ids.append(np.full(pick.size, l))
    poses = np.concatenate(xs)[:, None, :]
    ids = np.concatenate(ids)
    zero = lambda t, N, A: np.zeros((N, A, 2))  # noqa: E731
    run_multi(f110, dev, st, hosts, ids, poses, 'step', env_level=False, seed=521, ticks=2, actions=zero,
              check=rot_path(f110, len(layers)))


@pytest.mark.parametrize('stacked', [False, True])
def test_absurd_coordinates(f110, dev, mixed, stacked):
    """Scan poses at |x| + |y| >= 1e9 cells (k_dynamics marks them absurd): march_generic_rot, the literal arithmetic."""
    layers, hosts, st = mixed
    rng = np.random.default_rng(530)
    n = 40
    ids = np.arange(n) % len(layers) if stacked else np.zeros(n, int)
    big = np.array([6e7, -6e7, 3e9, -3e9, 1e15])
    xy = np.stack([rng.choice(big, n), rng.choice(big, n)], axis=1) * rng.uniform(0.9, 1.1, (n, 2))
    near = population(hosts if stacked else hosts[:1], ids, rng, 1)[:, 0, :2]
    xy[::4] = near[::4] + np.array([4e7, 0.0])
    poses = np.concatenate([xy, rng.uniform(0, 2 * np.pi, (n, 1))], axis=1)[:, None, :]
    zero = lambda t, N, A: np.zeros((N, A, 2))  # noqa: E731
    run_multi(f110, dev, st if stacked else layers[0], hosts if stacked else hosts[:1], ids, poses, 'step',
              env_level=False, seed=531, ticks=2, actions=zero, check=rot_path(f110, len(layers) if stacked else 1))


# ----------------------------------------------------------------------------- 5. the mixed stack
@pytest.mark.parametrize('shape', ['4x512', '2x1024'])
def test_mixed_stack_tick_with_per_layer_autoreset(f110, dev, sms, mixed, shape):
    layers, hosts, st = mixed
    A = 2
    n = 8 * sms if shape == '4x512' else 24 * sms
    ids = np.arange(n) % len(layers)
    rng = np.random.default_rng(540)
    tables = [start_table(h, rng) for h in hosts]
    poses = population(hosts, ids, rng, A)
    ev = run_multi(f110, dev, st, hosts, ids, poses, 'tick', tables=tables, seed=541,
                   check=rot_path(f110, len(layers), 512 if shape == '4x512' else 1024))
    assert_events(ev)


def test_mixed_stack_noise_build(f110, dev, sms, mixed):
    layers, hosts, st = mixed
    A, n = 2, 8 * sms | 1
    ids = np.arange(n) % len(layers)
    poses = population(hosts, ids, np.random.default_rng(550), A)
    ev = run_multi(f110, dev, st, hosts, ids, poses, 'tick', noise_std=0.01, seed=551,
                   check=rot_path(f110, len(layers), 512, noise=1))
    assert_events(ev, resets=False)


def test_mixed_stack_count_build(f110, dev, sms, mixed):
    layers, hosts, st = mixed
    A, n = 2, 8 * sms
    ids = np.arange(n) % len(layers)
    poses = population(hosts, ids, np.random.default_rng(560), A)
    run_multi(f110, dev, st, hosts, ids, poses, 'step', env_level=False, count=True, seed=561,
              check=rot_path(f110, len(layers), 512, count=1))


# ----------------------------------------------------------------------------- 6. batch == separate runs
def test_batch_equals_separate_runs(f110, dev, sms, mixed):
    """Each layer's envs in the mixed batch equal, bit for bit, a single-map Simulator over all N envs (rotated maps on
    k_march_lean_rot, the unrotated ones on their own default kernels): scans, state, collisions, done, laps, and lookup
    counts in a counting run."""
    layers, hosts, st = mixed
    A, n = 2, 4 * sms
    L = len(layers)
    ids = np.arange(n) % L
    rng = np.random.default_rng(570)
    tables = [torch.from_numpy(start_table(h, rng)).to(dev) for h in hosts]
    poses = population(hosts, ids, rng, A)
    acts = [random_actions(rng, n, A) for _ in range(T)]
    lib = f110._native.lib()
    batch = _sim(f110, dev, n, A, 0.01)
    batch.set_device_map(st, env_map_ids=ids)
    batch.env_reset(poses)
    singles = []
    for m in layers:
        s = _sim(f110, dev, n, A, 0.01)
        s.set_device_map(m)
        s.env_reset(poses)
        singles.append(s)
    fields = ('scans', 'state', 'collisions', 'collision_idx', 'done', 'lap_times', 'lap_counts', 'toggle_list')
    resets = 0
    for t in range(T):
        batch.tick(acts[t], autoreset_poses=tables, seed=AR_SEED)
        assert 'march=lean-rot ROT=1 layers=%d HET=1 RES=1' % L in lib.f110_debug_last_launch().decode()
        resets += int(cpu(batch.collisions).reshape(n, A)[:, 0].astype(bool).sum())
        for l, s in enumerate(singles):
            s.tick(acts[t], autoreset_poses=tables[l], seed=AR_SEED)
            rec = lib.f110_debug_last_launch().decode()
            rotated = hosts[l].orig_s != 0.0
            assert ('ROT=1' in rec) == rotated and 'HET=0' in rec, rec
            envs = np.flatnonzero(ids == l)
            for f in fields:
                a, b = cpu(getattr(batch, f)), cpu(getattr(s, f))
                if f == 'state':
                    a, b = a.reshape(7, n, A)[:, envs], b.reshape(7, n, A)[:, envs]
                elif f == 'done':
                    a, b = a[envs], b[envs]
                else:
                    a, b = a.reshape(n, A, -1)[envs], b.reshape(n, A, -1)[envs]
                assert np.array_equal(a, b), ('tick %d' % t, f, l)
    assert resets > 0
    for l, m in enumerate(layers):
        envs = np.flatnonzero(ids == l)
        counted = []
        for dmap, eids in ((st, ids[envs]), (m, None)):
            s = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, AR_SEED, num_envs=envs.size, device=dev, noise_std=0.0,
                               count_lookups=True)
            s.set_device_map(dmap, env_map_ids=eids) if eids is not None else s.set_device_map(dmap)
            s.env_reset(poses[envs])
            for t in range(3):
                s.step(acts[t][envs])
            counted.append(s.lookups())
        assert counted[0] == counted[1] > 0, (l, counted)


# ----------------------------------------------------------------------------- 7. CUDA graph == eager
def test_graph_equals_eager_tick(f110, dev, sms, mixed):
    layers, hosts, st = mixed
    A, n = 2, 4 * sms
    ids = np.arange(n) % len(layers)
    rng = np.random.default_rng(580)
    tables = [torch.from_numpy(start_table(h, rng)).to(dev) for h in hosts]
    poses = population(hosts, ids, rng, A)
    g, e = _sim(f110, dev, n, A, 0.01), _sim(f110, dev, n, A, 0.01)
    for s in (g, e):
        s.set_device_map(st, env_map_ids=ids)
        s.env_reset(poses)
    abuf = torch.zeros((n * A, 2), dtype=torch.float64, device=dev)
    g.capture_graph(abuf, autoreset_poses=tables, pose_gap=POSE_GAP, autoreset_seed=AR_SEED, env_level=True)
    resets = 0
    for t in range(T):
        act = random_actions(rng, n, A)
        abuf.copy_(torch.from_numpy(act.reshape(-1, 2)))
        g.replay()
        e.tick(act, env_level=True, autoreset_poses=tables, pose_gap=POSE_GAP, seed=AR_SEED)
        resets += int(cpu(e.collisions).reshape(n, A)[:, 0].astype(bool).sum())
        for f in ('scans', 'state', 'collisions', 'done', 'lap_counts', 'lap_times', 'tick_counter'):
            assert np.array_equal(cpu(getattr(g, f)), cpu(getattr(e, f))), ('tick %d' % t, f)
    assert resets > 0
    assert 'ROT=1' in f110._native.lib().f110_debug_last_launch().decode()


# ----------------------------------------------------------------------------- 8. F110Env, invalid arguments
def test_f110env_with_rotated_maps(f110, dev, tmp_path):
    """A map list whose yaml origins have a yaw (copies of the bundled maps): rotated_origins=True is needed, and the env
    steps what a Simulator on the same stack steps."""
    import yaml
    names, exts = [], []
    for name, ext, yaw in (('berlin', '.png', YAWS['berlin']), ('vegas', '.png', None), ('skirk', '.png', YAWS['skirk'])):
        with open(os.path.join(MAPS, name + '.yaml')) as f:
            meta = yaml.safe_load(f)
        if yaw is not None:
            meta['origin'] = [meta['origin'][0], meta['origin'][1], yaw]
        with open(str(tmp_path / (name + '.yaml')), 'w') as f:
            yaml.safe_dump(meta, f)
        shutil.copy(os.path.join(MAPS, name + ext), str(tmp_path / (name + ext)))
        names.append(str(tmp_path / name))                  # F110Env(map=...) adds '.yaml' to a path
        exts.append(ext)
    N, A = 9, 2
    with pytest.raises(ValueError):
        f110.F110Env(map=names, map_ext=exts, num_envs=N, num_agents=A)
    env = f110.F110Env(map=names, map_ext=exts, num_envs=N, num_agents=A, scan_noise_std=0.0, rotated_origins=True)
    layers = [f110.DeviceMap.from_yaml(p + '.yaml', e, dev) for p, e in zip(names, exts)]
    assert [m.host.orig_s != 0.0 for m in layers] == [True, False, True]
    ids = np.arange(N) % 3
    poses = population([m.host for m in layers], ids, np.random.default_rng(590), A)
    ref = _sim(f110, dev, N, A, 0.0)
    ref.set_device_map(f110.DeviceMap.stack(layers, rotated_origins=True), env_map_ids=ids)
    obs, _, done, _ = env.reset(poses)
    ref.env_reset(poses)
    ref.step(np.zeros((N, A, 2)))
    ref.env_post_step()
    for t in range(5):
        act = random_actions(np.random.default_rng(t), N, A)
        obs, _, done, _ = env.step(act)
        want = ref.step(act)
        ref.env_post_step()
        for k in ('scans', 'poses_x', 'poses_y', 'poses_theta', 'collisions'):
            assert torch.equal(obs[k], want[k]), (t, k)
        assert torch.equal(done, ref.done.bool())
    assert 'march=lean-rot ROT=1 layers=3' in f110._native.lib().f110_debug_last_launch().decode()
    env.update_map([names[1] + '.yaml'] * 2, exts[1:2] * 2, env_map_ids=np.zeros(N, int), rotated_origins=False)
    env.step(np.zeros((N, A, 2)))
    assert 'ROT=0' in f110._native.lib().f110_debug_last_launch().decode()


def test_layer_rot_invalid_arguments(f110, dev, mixed):
    """layer_rot without layer_res, without layer_geom, with fast_path, or on another march path (round-1 kernels: variant
    1; the literal kernel: variant 13) returns F110_ERR_INVALID before anything is enqueued; the unmodified stack then
    steps.  f110_scan refuses it."""
    layers, hosts, st = mixed
    N, A = 10, 2
    ids = np.arange(N) % len(layers)
    sim = _sim(f110, dev, N, A, 0.0)
    sim.set_device_map(st, env_map_ids=ids)
    sim.env_reset(population(hosts, ids, np.random.default_rng(600), A))
    good = sim._map_struct
    bads = []
    for field, value in (('layer_res', None), ('layer_geom', None), ('fast_path', 1)):
        b = type(good).from_buffer_copy(good)
        setattr(b, field, value)
        bads.append(b)
    single = type(good).from_buffer_copy(layers[0].c)      # one rotated map with a layer_rot table
    single.layer_rot = good.layer_rot
    zero = np.zeros((N, A, 2))
    lib = f110._native.lib()
    try:
        for bad in bads:
            sim._map_struct = bad
            with pytest.raises(f110._native.F110Error):
                sim.step(zero)
        sim._map_struct = good
        for v in (1, 13):
            lib.f110_debug_set_variant(v)
            with pytest.raises(f110._native.F110Error):
                sim.step(zero)
        lib.f110_debug_set_variant(0)
        s1 = _sim(f110, dev, N, A, 0.0)
        s1.set_device_map(layers[0])
        s1.env_reset(population(hosts[:1], np.zeros(N, int), np.random.default_rng(601), A))
        s1._map_struct = single
        with pytest.raises(f110._native.F110Error):
            s1.step(zero)
    finally:
        sim._map_struct = good
        lib.f110_debug_set_variant(0)
    sim.step(zero)
    expect_path(f110, {'march': 'lean-rot', 'ROT': 1, 'layers': len(layers)})
    ss = f110.ScanSimulator2D(1080, 4.7, device=dev)
    ss.set_device_map(st)
    with pytest.raises(f110._native.F110Error):
        ss.scan(np.zeros((1, 3)))
