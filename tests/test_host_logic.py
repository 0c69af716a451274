"""CPU-only tests (no GPU): host-side tables vs the reference goldens, the C-ABI library loads and
exports every symbol include/f110_b200.h declares, the ctypes struct mirrors match the C layout, the
product fails loudly without its CUDA library, env sharding + the optional observation all-gather
(gloo, world_size 2)."""
import ctypes
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
HEADER = os.path.join(ROOT, 'include', 'f110_b200.h')


def test_beam_tables_and_lut_match_reference():
    from f1tenth_gym_b200 import maps
    k = np.load(os.path.join(G, 'kat_kernels.npz'))
    sa, co, sd = maps.beam_tables(1080, 4.7, maps.DEFAULT_PARAMS)
    assert np.array_equal(sa, k['scan_angles'])
    assert np.array_equal(co, k['cosines'])
    assert np.array_equal(sd, k['side_distances'])
    assert maps.theta_index_increment(1080, 4.7) == 1.3865212836550662    # SURVEY appendix A
    s, c = maps.angle_lut(2000)
    assert s.shape == (2000,) and abs(s[-1]) < 1e-15 and c[-1] == 1.0      # linspace includes 2*pi
    assert np.array_equal(maps.params_vector(maps.DEFAULT_PARAMS), k['pvec'])


def test_map_pipeline_matches_oracle_and_flags():
    import oracle
    from f1tenth_gym_b200 import maps
    for name, fast in (('example_map', 1), ('berlin', 0)):
        path = maps.resolve_map_path(name)
        m = maps.load_map(path, '.png')
        o = oracle.OracleMap.from_yaml(path, '.png')
        assert np.array_equal(m.dt, o.dt)
        assert (m.orig_x, m.orig_y, m.orig_c, m.orig_s, m.resolution) == (o.orig_x, o.orig_y, o.orig_c, o.orig_s, o.resolution)
        assert m.fast_path == fast
        assert m.dt_oob == m.dt[-1, -1]
    m = maps.load_map(maps.resolve_map_path('example_map'), '.png')
    assert (m.height, m.width, m.resolution) == (1600, 1600, 0.0625)
    wp = maps.load_waypoints()
    assert wp.shape == (783, 3)
    assert maps.resolve_map_path('/tmp/custom') == '/tmp/custom.yaml'      # f110_env.py:117-118


def test_device_tables_construct_on_cpu():
    """DeviceMap / DeviceBeams only allocate and fill tensors: build them on the CPU device to check the
    struct wiring (field order, derived tables) without a GPU."""
    import torch
    from f1tenth_gym_b200 import maps
    from f1tenth_gym_b200.simulator import DeviceBeams, DeviceMap
    hm = maps.load_map(maps.resolve_map_path('example_map'), '.png')
    dm = DeviceMap(hm, torch.device('cpu'))
    assert dm.c.fast_path == 1 and dm.c.dt_codes and dm.c.dt_lut and dm.c.dt_cells and dm.c.sincos
    codes, lut = dm.dt_codes.numpy(), dm.dt_lut.numpy()
    cells = dm.dt_cells.numpy()
    ok = codes != 255
    assert ok.any() and np.array_equal(lut[codes[ok]], cells[ok])         # lossless coding
    assert np.array_equal(cells * hm.resolution, hm.dt)                  # exact power-of-two scaling
    assert (cells[~ok] > lut[254]).all()
    assert np.array_equal(dm.sincos.numpy()[:, 0], dm.sines.numpy())
    db = DeviceBeams(1080, 4.7, maps.DEFAULT_PARAMS, torch.device('cpu'))
    assert np.array_equal(db.cos_side.numpy()[:, 1], db.side_distances.numpy())
    assert db.c.num_beams == 1080 and db.c.cos_side
    hb = maps.load_map(maps.resolve_map_path('berlin'), '.png')
    dmb = DeviceMap(hb, torch.device('cpu'))
    assert dmb.c.fast_path == 0 and not dmb.c.dt_codes and not dmb.c.dt_cells


def declared_symbols():
    txt = open(HEADER).read()
    txt = re.sub(r'/\*.*?\*/', '', txt, flags=re.S)
    return sorted(set(re.findall(r'\b(f110_[a-z0-9_]+)\s*\(', txt)))


def test_library_exports_every_declared_symbol():
    from f1tenth_gym_b200 import _native as nat
    L = nat.lib()          # loads without a GPU; no compute call is made
    names = declared_symbols()
    assert len(names) >= 18
    for n in names:
        assert hasattr(L, n), n
    assert sorted(nat.SIGNATURES) == names
    assert L.f110_abi_version() == nat.ABI_VERSION
    assert L.f110_status_string(-2) == b'Map is not set for scan simulator.'
    # argument validation happens before any CUDA call
    assert L.f110_step(None, None, None, None, None) == -1
    assert L.f110_scan(ctypes.byref(nat.F110Map()), ctypes.byref(nat.F110Beams()), None, 1, None, None, None, None) == -2


def test_march_kernel_resource_budget():
    """The production ray-march kernels must keep the register and stack budget the measurements were taken with: 32 registers
    (64 warps per SM) and at most 24 bytes of stack per thread.  A same-results build whose caller-side spills grew to 56 bytes of
    stack was measurably slower (DESIGN.md 3.2, codegen caveat): this is the check to run after any edit to
    csrc/march_lean.cuh, before spending GPU time."""
    import shutil
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    lib_path = os.path.join(os.path.dirname(os.path.abspath(nat.__file__)), 'libf110_b200.so')
    out = subprocess.run([tool, '-res-usage', lib_path], capture_output=True, text=True).stdout
    usage = {}
    for fn, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', out):
        usage[fn] = (int(reg), int(stack))
    # k_march_lean<TABLE=0, NOISE=0, COUNT=0, CELLS=1, LAYERED=0, 512 threads, 4 blocks/SM, DYN=1, CL=1, IPT, RING=2>: the default
    # launches of the dynamic queue (4 / 2 entries per ticket, ticket size by run class)
    for ipt in (4, 2, 0):
        name = '_ZN4f11012k_march_leanILi0ELb0ELb0ELb1ELb0ELi512ELi4ELb1ELi1ELi%dELi2EEEvNS_5LeanKENS_10MarchQueueE' % ipt
        assert name in usage, name
        reg, stack = usage[name]
        assert reg <= 32, (name, reg)
        assert stack <= 24, (name, stack)


def test_sass_carries_the_sm90a_paths():
    """The built library is sm_90a code and contains what DESIGN.md says it does: the TMA tile load of the north_star march variant
    (UTMALDG with mbarrier SYNCS), the elect.sync queue pop (ELECT) and the programmatic-dependent-launch hooks (ACQBULK / PREEXIT)."""
    import shutil
    from f1tenth_gym_b200 import _native as nat
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    nat.lib()
    lib_path = os.path.join(os.path.dirname(os.path.abspath(nat.__file__)), 'libf110_b200.so')
    elf = subprocess.run([tool, '-lelf', lib_path], capture_output=True, text=True).stdout
    assert 'sm_90a' in elf and 'sm_100' not in elf, elf
    sass = subprocess.run([tool, '-sass', lib_path], capture_output=True, text=True).stdout
    for mnemonic in ('UTMALDG', 'SYNCS', 'ELECT', 'ACQBULK', 'PREEXIT', 'DADD.RM'):
        assert mnemonic in sass, mnemonic


def test_unpack_scans_u24_roundtrip():
    """Host decoder of the opt-in 24-bit scan block (f110_pack_scans_u24: round(range * 2^19), little-endian 3 bytes): 2^-19 m
    steps, 32 m of range, |error| <= 2^-20 m + fp32 rounding -- far inside the 1e-4 m parity tolerance."""
    from f1tenth_gym_b200.simulator import Simulator
    rng = np.random.default_rng(3)
    r = np.concatenate([rng.uniform(0.0, 30.0, 5000), [0.0, 30.0, 2.0 ** -19, 31.999998]])
    q = np.rint(r * 2.0 ** 19).astype(np.uint32)
    buf = np.stack([q & 255, (q >> 8) & 255, (q >> 16) & 255], axis=-1).astype(np.uint8)
    dec = Simulator.unpack_scans_u24(buf)
    assert dec.dtype == np.float32 and dec.shape == r.shape
    assert np.max(np.abs(dec.astype(np.float64) - r)) <= 2.0 ** -20 + 30.0 * 2.0 ** -24


def test_ctypes_structs_match_c_layout(tmp_path):
    from f1tenth_gym_b200 import _native as nat
    structs = {'f110_map': nat.F110Map, 'f110_beams': nat.F110Beams, 'f110_sim': nat.F110Sim,
               'f110_host_obs': nat.F110HostObs}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){']
    for cname, st in structs.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for f, _ in st._fields_:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
    lines.append('return 0;}')
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-o', str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines())
    for cname, st in structs.items():
        assert int(out[cname]) == ctypes.sizeof(st), cname
        for f, _ in st._fields_:
            assert int(out['%s.%s' % (cname, f)]) == getattr(st, f).offset, (cname, f)


def test_missing_library_fails_loudly(monkeypatch):
    from f1tenth_gym_b200 import _native as nat
    monkeypatch.setattr(nat, '_LIB', None)
    monkeypatch.setattr(nat, 'LIB_PATH', '/nonexistent/libf110_b200.so')
    with pytest.raises(nat.NativeLibraryError):
        nat.lib()
    import f1tenth_gym_b200 as f
    with pytest.raises(nat.NativeLibraryError):
        f.Simulator(f.maps.DEFAULT_PARAMS, 1, 0, device='cpu')


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under f1tenth_gym_b200/ may reference it."""
    pkg = os.path.join(ROOT, 'f1tenth_gym_b200')
    for dp, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith(('.py', '.cu', '.cuh', '.h')):
                txt = open(os.path.join(dp, fn)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', txt, flags=re.M), fn
                assert 'f110_oracle' not in txt, fn


def test_shard_ranges():
    from f1tenth_gym_b200.distributed import shard_range
    for n, w in ((131072, 8), (10, 3), (7, 8)):
        r = [shard_range(n, g, w) for g in range(w)]
        assert r[0][0] == 0 and r[-1][1] == n
        assert all(r[i][1] == r[i + 1][0] for i in range(w - 1))
        sizes = [b - a for a, b in r]
        assert max(sizes) - min(sizes) <= 1


WORKER = textwrap.dedent('''
    import os, sys
    sys.path.insert(0, %r)
    import torch, torch.distributed as dist
    from f1tenth_gym_b200.distributed import all_gather_obs, shard_range, reduce_max_scalar, reduce_sum_scalar
    rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
    dist.init_process_group('gloo', rank=rank, world_size=world)
    N = 7                                   # uneven split: 3 + 4 envs
    lo, hi = shard_range(N, rank, world)
    full = torch.arange(N * 2 * 5, dtype=torch.float32).reshape(N, 2, 5)
    got = all_gather_obs(full[lo:hi].clone())
    assert torch.equal(got, full), (rank, got.shape)
    assert reduce_max_scalar(float(rank + 1), 'cpu') == float(world)
    assert reduce_sum_scalar(float(hi - lo), 'cpu') == float(N)
    dist.barrier()
    dist.destroy_process_group()
    print('ok', rank)
''')


def test_all_gather_obs_gloo_world2(tmp_path):
    script = tmp_path / 'worker.py'
    script.write_text(WORKER % ROOT)
    procs = []
    port = 29000 + (os.getpid() % 2000)
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE='2', MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT))
    for p in procs:
        out, _ = p.communicate(timeout=240)
        assert p.returncode == 0, out.decode()
