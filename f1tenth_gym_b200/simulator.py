"""Batched Simulator: the host-side mirror of reference base_classes.py (Simulator / RaceCar) for
N independent environments x A agents stepped in lockstep by the CUDA path.

Mirrors the reference interface for this path — same constructor arguments, method names, argument
meaning and error behaviour:
    Simulator(params, num_agents, seed, time_step=0.01, ego_idx=0, integrator=Integrator.RK4,
              lidar_dist=0.0)                                   base_classes.py:465-497
    .set_map(map_path, map_ext)                                 :499-511
    .update_params(params, agent_idx=-1)   IndexError           :514-534
    .reset(poses)                           ValueError           :614-630
    .step(control_inputs) -> observations dict                  :553-612
plus the batch extensions `num_envs`, `num_beams`, `fov`, `device`, `noise_std`.

PyTorch is used only as the device-memory allocator and stream provider; all compute goes through
the C ABI in libf110_b200.so (include/f110_b200.h).  There is no CPU fallback.
"""
import ctypes as C
from enum import Enum

import numpy as np
import torch

from . import _native as nat
from . import maps as hostmaps
from . import param_draw as pdraw


RENDER_MAX_AGENTS = 64     # csrc/render.cuh F110_RENDER_MAX_AGENTS: car quads a block of k_render_views caches
RENDER_MAX_SIZE = 8192     # largest view height / width of f110_render_views
TRACK_MAX_WINDOW = 1024    # csrc/progress.cuh F110_TRACK_MAX_WINDOW: largest back + fwd + 1 of the progress tracker
# The cost weights of predict(cost=) and MPPIPlanner when none are given (include/f110_mppi.h f110_cost): metres, radians and
# commands per step, progress in metres over the horizon.  The closed-loop test of tests/test_gpu_mppi.py drives with them
# (DESIGN §3.15 has the sweep they were picked from).
COST_DEFAULTS = {'w_lat': 1.0, 'w_head': 1.0, 'w_clear': 20.0, 'clear_min': 0.5, 'w_dsteer': 1.0, 'w_dspeed': 0.01,
                 'w_prog': 10.0, 'w_wall': 1000.0}
PACKED_RANGE_LIMIT = 32.0  # f110_pack_scans_u24: 24 bits of 2^-19 m clamp every range at 32 m - 2^-19


class Integrator(Enum):     # base_classes.py:40-42
    RK4 = 1
    Euler = 2


def _stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class DeviceMap(object):
    """ScanSimulator2D state (laser_models.py:348-427) resident in HBM: fp64 DT grid + angle LUTs."""

    def __init__(self, host_map, device, theta_dis=2000, eps=0.0001, max_range=30.0, _device_dt=None):
        self.host = host_map
        self.device = device
        self.theta_dis = theta_dis
        sines, cosines = hostmaps.angle_lut(theta_dis)
        # cell-unit copy for the fast path (res = 2^-k: the division is an exact exponent shift)
        self.dt_cells = self.dt_codes = self.dt_lut = self.dt_cells_pad = self.dt_codes_pad = None
        if _device_dt is not None:
            self.dt = _device_dt
            if host_map.fast_path:
                self.dt_cells = self.dt / host_map.resolution     # IEEE fp64 division on the device, exact here
        else:
            self.dt = torch.from_numpy(host_map.dt).to(device)
            if host_map.fast_path:
                cells = host_map.dt / host_map.resolution
                codes, lut = hostmaps.code_table(cells)
                self.dt_cells = torch.from_numpy(cells).to(device)
                self.dt_codes = torch.from_numpy(codes).to(device)
                self.dt_lut = torch.from_numpy(lut).to(device)
                self.dt_codes_pad = self._pad(self.dt_codes, pitch_multiple=16)
        if self.dt_cells is not None:
            self.dt_cells_pad = self._pad(self.dt_cells)
        self.sines = torch.from_numpy(sines).to(device)
        self.cosines = torch.from_numpy(cosines).to(device)
        sc = np.ascontiguousarray(np.stack([sines, cosines], axis=1))
        self.sincos = torch.from_numpy(sc).to(device)
        self.sincos2 = torch.from_numpy(np.ascontiguousarray(np.concatenate([sc, sc], axis=0))).to(device)
        # smallest positive DT value (= resolution for an exact EDT): the lean march kernel tests `d != 0` for `d > eps`
        pos = self.dt[self.dt > 0]
        dt_min_positive = float(pos.min().item()) if pos.numel() else float('inf')
        self.c = nat.F110Map(host_map.height, host_map.width, host_map.resolution, host_map.orig_x,
                             host_map.orig_y, host_map.orig_c, host_map.orig_s, eps, max_range, theta_dis,
                             host_map.fast_path, host_map.dt_oob, nat.ptr(self.dt), nat.ptr(self.dt_cells),
                             nat.ptr(self.dt_codes), nat.ptr(self.dt_lut), nat.ptr(self.sines), nat.ptr(self.cosines),
                             nat.ptr(self.sincos), nat.ptr(self.dt_cells_pad), nat.ptr(self.dt_codes_pad),
                             0 if self.dt_codes_pad is None else self.dt_codes_pad.shape[1],
                             nat.ptr(self.sincos2), dt_min_positive, 1)
        # the padded cell-unit table again in 4 x 4-cell bricks (f110_map_brick): what the ray march of the tick reads
        self.dt_cells_brick = None
        n = nat.lib().f110_map_brick_elems(C.byref(self.c)) if self.dt_cells_pad is not None and self.dt_cells_pad.is_cuda else 0
        if n > 0:
            self.dt_cells_brick = torch.empty((n,), dtype=torch.float64, device=device)
            nat.check(nat.lib().f110_map_brick(C.byref(self.c), nat.ptr(self.dt_cells_brick), _stream_ptr(self.dt_cells_pad.device)))
        self.march_tables = nat.F110MarchTables(nat.ptr(self.dt_cells_brick))

    @staticmethod
    def _pad(t, pitch_multiple=1):
        """[H][W] -> [H+1][W+1 rounded up to pitch_multiple] with the extra row / columns holding t[-1,-1] (what an
        off-map lookup reads)."""
        H, W = t.shape
        Wp = -(-(W + 1) // pitch_multiple) * pitch_multiple
        out = torch.empty((H + 1, Wp), dtype=t.dtype, device=t.device)
        out[:] = t[-1, -1]
        out[:H, :W] = t
        return out.contiguous()

    @classmethod
    def stack(cls, maps, mixed_resolution=False, rotated_origins=False):
        """Multi-map batch (SURVEY 8f row 3): Simulator.set_device_map(stacked, env_map_ids) picks one layer per env.
        Maps that share size, resolution and origin are stacked into one [L][H][W] table.  Other unrotated maps of one
        resolution are stacked on a canvas (see _stack_canvas).  Mixed resolutions raise ValueError unless
        mixed_resolution=True: then the maps are stacked on a metre canvas with each layer's own resolution (see
        _stack_canvas), and every layer, a power-of-two one included, is marched in metres.  With one shared resolution
        the flag changes nothing.
        Maps whose origin has a yaw raise ValueError unless rotated_origins=True: then the maps are stacked on a metre canvas
        with each layer's own resolution and rotation (see _stack_canvas), marched by k_march_lean_rot; different
        resolutions still also need mixed_resolution=True.  Without a rotated map the flag changes nothing.
        Every layer must share theta_dis, eps and max_range (ValueError otherwise): the stack keeps one LUT and one set of
        march constants, the first map's."""
        m0 = maps[0]
        h0 = m0.host
        for m in maps[1:]:
            for k in ('theta_dis', 'eps', 'max_range'):
                if getattr(m.c, k) != getattr(m0.c, k):
                    raise ValueError('stacked maps must share %s: %r and %r' % (k, getattr(m0.c, k), getattr(m.c, k)))
        if len(maps) > 1 and any(m.host.orig_c != 1.0 or m.host.orig_s != 0.0 for m in maps):
            if not rotated_origins:
                raise ValueError('stacking maps with a rotated origin needs rotated_origins=True')
            return cls._stack_canvas(maps, mixed_resolution=mixed_resolution, rotated_origins=True)
        if mixed_resolution and any(m.host.resolution != h0.resolution for m in maps[1:]):
            return cls._stack_canvas(maps, mixed_resolution=True)
        key0 = (h0.height, h0.width, h0.resolution, h0.orig_x, h0.orig_y, h0.orig_c, h0.orig_s)
        if any((m.host.height, m.host.width, m.host.resolution, m.host.orig_x, m.host.orig_y, m.host.orig_c,
                m.host.orig_s) != key0 for m in maps[1:]):
            return cls._stack_canvas(maps)
        out = cls.__new__(cls)
        out.__dict__.update(m0.__dict__)
        out.layers = list(maps)
        out.dt = torch.stack([m.dt for m in maps]).contiguous()
        out.dt_cells = torch.stack([m.dt_cells for m in maps]).contiguous() if m0.dt_cells is not None else None
        out.dt_cells_pad = torch.stack([m.dt_cells_pad for m in maps]).contiguous() if m0.dt_cells_pad is not None else None
        out.dt_codes = out.dt_lut = out.dt_codes_pad = None
        out.dt_cells_brick = None           # the brick table is built for a single map only
        out.march_tables = nat.F110MarchTables()
        c = nat.F110Map.from_buffer_copy(m0.c)
        c.dt = nat.ptr(out.dt)
        c.dt_cells = nat.ptr(out.dt_cells)
        c.dt_cells_pad = nat.ptr(out.dt_cells_pad)
        c.dt_codes = None
        c.dt_lut = None
        c.dt_codes_pad = None
        c.num_layers = len(maps)
        c.dt_min_positive = min(m.c.dt_min_positive for m in maps)
        out.c = c
        return out

    @classmethod
    def _stack_canvas(cls, maps, mixed_resolution=False, rotated_origins=False):
        """Maps of different size and origin on one [L][Hc][Wc] canvas (Wc = max W_l, Hc = max H_l): layer l's table sits in
        the low corner of its slice and every other cell of the slice holds that layer's dt[-1,-1], which is what the
        reference reads off that map, so the march kernels clamp to the canvas and need no per-layer width or height.  The
        cell-unit padded table gets the same treatment with its extra row and column.  f110_map.layer_geom carries each
        layer's (orig_x, orig_y, x_max = W_l * res, y_max = H_l * res, W_l, H_l).
        mixed_resolution: the layers may differ in resolution.  Only the metre canvas is built (no cell-unit tables,
        fast_path 0), x_max / y_max are W_l * res_l and H_l * res_l, and f110_map.layer_res carries each layer's
        (res_l, 1 / res_l) with host copies of the finest and coarsest.  The struct's resolution stays the first map's.
        rotated_origins: the layers may have rotated origins.  The metre canvas as for mixed_resolution, with layer_res for
        every layer (also when they share one resolution), and f110_map.layer_rot carries each layer's (orig_c, orig_s)
        as HostMap computed them.  The struct's origin and rotation stay the first map's."""
        hs = [m.host for m in maps]
        h0 = hs[0]
        if not mixed_resolution and any(h.resolution != h0.resolution for h in hs):
            raise ValueError('stacked maps must share one resolution')
        if not rotated_origins and any(h.orig_c != 1.0 or h.orig_s != 0.0 for h in hs):
            raise ValueError('stacked maps of different size or origin need unrotated origins')
        metres = mixed_resolution or rotated_origins
        if not metres and any((m.dt_cells is None) != (maps[0].dt_cells is None) for m in maps):
            raise ValueError('stacked maps must all have, or all lack, the cell-unit table')
        cells = maps[0].dt_cells is not None and not metres
        L = len(maps)
        Hc, Wc = max(h.height for h in hs), max(h.width for h in hs)

        def canvas(tables, extra):
            out = torch.empty((L, Hc + extra, Wc + extra), dtype=tables[0].dtype, device=tables[0].device)
            for l, t in enumerate(tables):
                out[l] = t[-1, -1]
                out[l, :t.shape[0], :t.shape[1]] = t
            return out.contiguous()
        out = cls.__new__(cls)
        out.__dict__.update(maps[0].__dict__)
        out.layers = list(maps)
        out.dt = canvas([m.dt for m in maps], 0)
        out.dt_cells = canvas([m.dt_cells for m in maps], 0) if cells else None
        out.dt_cells_pad = canvas([m.dt_cells for m in maps], 1) if cells else None
        out.dt_codes = out.dt_lut = out.dt_codes_pad = None
        out.dt_cells_brick = None
        out.march_tables = nat.F110MarchTables()
        out.layer_geom_host = np.array([[h.orig_x, h.orig_y, h.width * h.resolution, h.height * h.resolution, h.width,
                                         h.height] for h in hs], dtype=np.float64)
        out.layer_geom = torch.from_numpy(out.layer_geom_host).to(maps[0].device)
        c = nat.F110Map.from_buffer_copy(maps[0].c)
        c.height, c.width = Hc, Wc
        c.dt = nat.ptr(out.dt)
        c.dt_cells = nat.ptr(out.dt_cells)
        c.dt_cells_pad = nat.ptr(out.dt_cells_pad)
        c.dt_codes = None
        c.dt_lut = None
        c.dt_codes_pad = None
        c.codes_pitch = 0
        c.num_layers = L
        c.dt_min_positive = min(m.c.dt_min_positive for m in maps)
        c.layer_geom = nat.ptr(out.layer_geom)
        c.layer_orig_max = float(np.abs(out.layer_geom_host[:, :2]).max())
        if metres:
            c.fast_path = 0
            out.layer_res_host = np.array([[h.resolution, 1.0 / h.resolution] for h in hs], dtype=np.float64)
            out.layer_res = torch.from_numpy(out.layer_res_host).to(maps[0].device)
            c.layer_res = nat.ptr(out.layer_res)
            c.layer_res_min = float(out.layer_res_host[:, 0].min())
            c.layer_res_max = float(out.layer_res_host[:, 0].max())
        if rotated_origins:
            out.layer_rot_host = np.array([[h.orig_c, h.orig_s] for h in hs], dtype=np.float64)
            out.layer_rot = torch.from_numpy(out.layer_rot_host).to(maps[0].device)
            c.layer_rot = nat.ptr(out.layer_rot)
        out.c = c
        return out

    @classmethod
    def from_device_dt(cls, dt, resolution, origin, **kw):
        """A map whose fp64 distance table [H][W] (metres) already lives on the device (e.g. rasterised track +
        f110_edt): nothing but the out-of-bounds scalar dt[-1,-1] crosses PCIe."""
        dt = dt.contiguous()
        meta = hostmaps.HostMap.meta(dt.shape[0], dt.shape[1], resolution, origin, float(dt[-1, -1].item()))
        return cls(meta, dt.device, _device_dt=dt, **kw)

    @classmethod
    def from_yaml(cls, map_path, map_ext, device, edt='scipy', **kw):
        """edt='scipy': the reference's host pipeline; edt='device': C ABI f110_edt (bit-identical table)."""
        if edt == 'device':
            return cls(hostmaps.load_map_device_edt(map_path, map_ext, device), device, **kw)
        return cls(hostmaps.load_map(map_path, map_ext), device, **kw)


class DeviceBeams(object):
    """Per-beam tables of RaceCar.__init__ (base_classes.py:122-158) in HBM."""

    def __init__(self, num_beams, fov, params, device, theta_dis=2000):
        self.num_beams, self.fov = num_beams, fov
        sa, co, sd = hostmaps.beam_tables(num_beams, fov, params)
        self.scan_angles = torch.from_numpy(sa).to(device)
        self.cosines = torch.from_numpy(co).to(device)
        self.side_distances = torch.from_numpy(sd).to(device)
        self.cos_side = torch.from_numpy(np.ascontiguousarray(np.stack([co, sd], axis=1))).to(device)
        self.angle_increment = fov / (num_beams - 1)
        self.c = nat.F110Beams(num_beams, fov, self.angle_increment,
                               hostmaps.theta_index_increment(num_beams, fov, theta_dis),
                               nat.ptr(self.scan_angles), nat.ptr(self.cosines), nat.ptr(self.side_distances),
                               nat.ptr(self.cos_side), float(sd.max()))


def centerline_segments(table):
    """One closed centerline (n, 2) (x, y) in metres, progress in row order -> ((n, 8) fp64 segment records, length L).
    A last row equal to the first is dropped; the table is then closed with segment n-1 -> 0.  Record i = (x_i, y_i, dx, dy,
    l2 = dx**2 + dy**2, s_i, len_i = sqrt(l2), h_i = arctan2(dy, dx)); s = np.cumsum of the lengths, shifted to start at 0, and
    L its last entry.  ValueError for fewer than 3 points, non-finite values or a zero-length segment."""
    T = np.asarray(table.cpu() if torch.is_tensor(table) else table, dtype=np.float64)
    if T.ndim != 2 or T.shape[1] != 2:
        raise ValueError('a centerline must be an (n, 2) table of (x, y), got shape %s' % (T.shape,))
    if not np.all(np.isfinite(T)):
        raise ValueError('a centerline must hold finite values')
    if T.shape[0] > 1 and T[-1, 0] == T[0, 0] and T[-1, 1] == T[0, 1]:
        T = T[:-1]
    if T.shape[0] < 3:
        raise ValueError('a centerline needs at least 3 distinct points, got %d' % T.shape[0])
    d = np.roll(T, -1, axis=0) - T
    l2 = d[:, 0] ** 2 + d[:, 1] ** 2
    if np.any(l2 == 0):
        raise ValueError('a centerline must not repeat a point (zero-length segment %d)' % int(np.argmax(l2 == 0)))
    length = np.sqrt(l2)
    cum = np.cumsum(length)
    s = np.concatenate([[0.0], cum[:-1]])
    h = np.arctan2(d[:, 1], d[:, 0])
    return np.ascontiguousarray(np.stack([T[:, 0], T[:, 1], d[:, 0], d[:, 1], l2, s, length, h], axis=1)), float(cum[-1])


class CenterlineTables(object):
    """Closed centerlines on the device (C ABI f110_track): one (n, 2) table, or a list of them (one per map layer)."""

    def __init__(self, tables, device):
        if isinstance(tables, (list, tuple)) and len(tables) and np.ndim(tables[0]) == 2:
            tables = list(tables)
        else:
            tables = [tables]
        recs, lengths = zip(*[centerline_segments(t) for t in tables])
        self.num_tables = len(recs)
        self.num_segments = [r.shape[0] for r in recs]
        self.lengths = np.array(lengths, dtype=np.float64)
        self.records = list(recs)
        starts = np.concatenate([[0], np.cumsum(self.num_segments)]).astype(np.int32)
        self.segments = torch.from_numpy(np.concatenate(recs)).to(device)
        self.table_start = torch.from_numpy(starts).to(device)
        self.c = nat.F110Track(self.num_tables, min(self.num_segments), nat.ptr(self.table_start), nat.ptr(self.segments))


def check_theta_dis(device_map, theta_dis, who):
    """ValueError unless device_map's sin / cos LUT has theta_dis entries: beam tables built for one theta_dis step through
    another's LUT with the wrong increment, so every beam after the first would point the wrong way."""
    got = int(device_map.c.theta_dis)
    if got != int(theta_dis):
        raise ValueError('the map was built with theta_dis=%d but this %s has theta_dis=%d; build both with the same value'
                         % (got, who, int(theta_dis)))


def empty_map_struct():
    """A map struct with no DT bound: stepping with it raises ValueError like the reference
    (laser_models.py:445-446 'Map is not set for scan simulator.')."""
    return nat.F110Map()


class Simulator(object):
    """N x A batched simulator.  All state lives in persistent device buffers (SoA over the flat agent
    index a = env*A + agent); the observation tensors returned by step() are VIEWS of those buffers
    and are overwritten by the next step (the reference likewise returns aliases of internal arrays,
    base_classes.py:594-602)."""

    def __init__(self, params, num_agents, seed, time_step=0.01, ego_idx=0, integrator=Integrator.RK4,
                 lidar_dist=0.0, num_envs=1, num_beams=1080, fov=4.7, device=None, noise_std=0.0,
                 count_lookups=False, march_queue=True, march_item_beams=32, theta_dis=2000):
        """theta_dis: entries of the map's sin / cos LUT (ScanSimulator2D's theta_dis) that the beam tables step through;
        set_device_map refuses a map built for another value."""
        nat.lib()   # fail loudly right away if the CUDA library is missing
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        self.num_agents = int(num_agents)
        self.num_envs = int(num_envs)
        self.seed = seed
        self.time_step = time_step
        self.ego_idx = ego_idx
        self.params = params
        self.integrator = integrator
        self.lidar_dist = lidar_dist
        self.num_beams, self.fov = num_beams, fov
        self.theta_dis = int(theta_dis)
        if isinstance(integrator, Integrator):
            integ = integrator.value
        elif integrator in (1, 2):
            integ = int(integrator)
        else:
            name = getattr(integrator, 'name', integrator)
            raise SyntaxError("Invalid Integrator Specified. Provided %s. Please choose RK4 or Euler" % name)
        N, A, B = self.num_envs, self.num_agents, num_beams
        NA = N * A
        dev = self.device
        f64 = dict(dtype=torch.float64, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        self.params_dev = torch.from_numpy(np.tile(hostmaps.params_vector(params), (A, 1))).to(dev)
        self.state = torch.zeros((7, NA), **f64)
        self.steer_buf = torch.zeros((2, NA), **f64)
        self.steer_cnt = torch.zeros((NA,), **i32)
        self.scan_pose = torch.zeros((NA, 4), **f64)
        self.agent_poses = torch.zeros((NA, 5), **f64)
        self.scans = torch.zeros((NA, B), dtype=torch.float32, device=dev)
        self.wall_flag = torch.zeros((NA,), **i32)
        self.collisions = torch.zeros((NA,), **f64)
        self.collision_idx = torch.full((NA,), -1, **i32)
        # F110Env-level arrays (f110_env.py:165-189), batched
        self.current_time = torch.zeros((N,), **f64)
        self.lap_times = torch.zeros((NA,), **f64)
        self.lap_counts = torch.zeros((NA,), **f64)
        self.toggle_list = torch.zeros((NA,), **f64)
        self.near_starts = torch.ones((NA,), **i32)
        self.start_xs = torch.zeros((NA,), **f64)
        self.start_ys = torch.zeros((NA,), **f64)
        self.start_thetas = torch.zeros((NA,), **f64)
        self.start_rot = torch.eye(2, **f64).reshape(1, 4).repeat(N, 1).contiguous()
        self.done = torch.zeros((N,), dtype=torch.uint8, device=dev)
        self.checkpoint_done = torch.zeros((NA,), dtype=torch.uint8, device=dev)
        self.env_arrivals = torch.zeros((N,), **i32)
        self.lookup_counter = torch.zeros((1,), dtype=torch.int64, device=dev) if count_lookups else None
        self.tick_counter = torch.zeros((1,), dtype=torch.int64, device=dev)
        # work queue of the persistent ray-march kernel (csrc/march.cuh): last tick's heavy items go first
        ib = int(march_item_beams)
        assert ib in (32, 64)
        self.march_ipa = (B + ib - 1) // ib if (march_queue and (B + ib - 1) // ib <= 256) else 0
        items = NA * self.march_ipa
        self.march_cost = torch.full((NA * 256,), -1, **i32) if self.march_ipa else None
        self.march_order = torch.zeros((3, items), **i32) if self.march_ipa else None
        self.march_count = torch.zeros((4,), **i32) if self.march_ipa else None
        self.march_rec = torch.zeros((NA, 8), **f64) if self.march_ipa else None
        self.beams = DeviceBeams(num_beams, fov, params, dev, self.theta_dis)
        self.map = None
        self.env_layer = None
        self._map_struct = empty_map_struct()
        self._march_tables = nat.F110MarchTables()
        self._actions_dev = torch.zeros((NA, 2), **f64)
        self.c = nat.F110Sim(
            N, A, integ, ego_idx, 0, time_step, lidar_dist, 0.005, float(params['length']), float(params['width']),
            nat.ptr(self.params_dev), nat.ptr(self.state), nat.ptr(self.steer_buf), nat.ptr(self.steer_cnt),
            nat.ptr(self.scan_pose), nat.ptr(self.agent_poses), nat.ptr(self.scans), nat.ptr(self.wall_flag),
            nat.ptr(self.collisions), nat.ptr(self.collision_idx), nat.ptr(self.current_time),
            nat.ptr(self.lap_times), nat.ptr(self.lap_counts), nat.ptr(self.toggle_list),
            nat.ptr(self.near_starts), nat.ptr(self.start_xs), nat.ptr(self.start_ys),
            nat.ptr(self.start_thetas), nat.ptr(self.start_rot), nat.ptr(self.done),
            nat.ptr(self.checkpoint_done), nat.ptr(self.env_arrivals), None, nat.ptr(self.lookup_counter), nat.ptr(self.tick_counter),
            nat.ptr(self.march_cost), nat.ptr(self.march_order), nat.ptr(self.march_count), self.march_ipa,
            nat.ptr(self.march_rec), float(noise_std), int(seed) & 0xFFFFFFFFFFFFFFFF)
        self._graph = None
        self._zeros_NA = torch.zeros((N, A), dtype=torch.float64, device=dev)     # obs['linear_vels_y'] (always 0, :606)
        self.centerlines = None
        self.track_seg = self.track_s = self.track_d = self.track_heading_error = None
        self.track_progress = self.track_delta = None
        # outputs and scratch of tick_repeat (C ABI f110_repeat), allocated on first use
        self.done_any = self.done_tick = self.repeat_list = self.repeat_list_count = self.marched_agents = None
        self.track_delta_sum = None
        self._repeat_c = None
        self._repeat_ticks = 0      # intermediate agent-ticks issued since the counter was last read (marched_fraction)
        self._repeat_plain = False
        # static box obstacles (C ABI f110_obstacles), set by set_obstacles
        self._obst = None
        self.obstacle_boxes = self.obstacle_active = self.obstacle_hit = None
        self._obst_keep = ()
        # agents without a lidar (C ABI f110_lidar), set by set_lidar; None: every slot has one
        self._lidar = None
        self._lidar_slots = (True,) * A
        self.lidar_list = self.lidar_list_count = self.lidar_listed = None
        # episode mode (C ABI f110_episodes), set by set_episodes; None: off
        self._episodes = None
        self.ep_ticks = self.ep_terminated = self.ep_truncated = self.ep_length = None
        self.final_state = self.final_scans = self.final_collisions = self.final_collision_idx = None
        self.final_lap_times = self.final_lap_counts = self.ep_list = self.ep_list_count = None
        # ... and its part under a held action (C ABI f110_episode_repeat)
        self._episode_repeat = None
        self.ep_end_tick = self.ep_snap_rec = self.ep_snap_poses = self.ep_snap_wall_flag = None
        self.ep_scan_list = self.ep_scan_count = None
        # per-episode parameter draws (C ABI f110_param_draw), set by set_param_draw; None: off
        self._param_draw = self.param_draw = None
        self.param_lo = self.param_hi = self.final_params = None

    # ------------------------------------------------------------------ configuration
    def set_map(self, map_path, map_ext, edt='scipy'):
        """base_classes.py:499-511 / laser_models.py:383-427 (load-time: PIL + yaml + EDT; edt='device' runs the
        exact distance transform on the GPU instead of scipy on the host)."""
        self.set_device_map(DeviceMap.from_yaml(map_path, map_ext, self.device, edt=edt, theta_dis=self.theta_dis))

    def set_device_map(self, device_map, env_map_ids=None):
        """env_map_ids (N,) ints: which layer of a DeviceMap.stack() each env uses (multi-map batches).  ValueError for a map
        whose theta_dis differs from the simulator's: the beams would step through its LUT with the wrong increment."""
        check_theta_dis(device_map, self.theta_dis, 'Simulator')
        self.map = device_map
        self._map_struct = device_map.c
        self._march_tables = getattr(device_map, 'march_tables', None) or nat.F110MarchTables()
        self._graph = None
        self.set_centerlines(None)      # the centerlines belong to the old map
        layers = getattr(device_map.c, 'num_layers', 1)
        if layers > 1:
            ids = torch.zeros((self.num_envs,), dtype=torch.int32) if env_map_ids is None else \
                torch.as_tensor(env_map_ids, dtype=torch.int32)
            if ids.numel() != self.num_envs or int(ids.min()) < 0 or int(ids.max()) >= layers:
                raise ValueError('env_map_ids must hold num_envs layer indices in [0, %d)' % layers)
            self.env_layer = ids.to(self.device).contiguous()
            self.c.env_layer = nat.ptr(self.env_layer)
        else:
            self.env_layer = None
            self.c.env_layer = None

    def update_params(self, params, agent_idx=-1, env_mask=None):
        """base_classes.py:514-534.  agent_idx < 0: every agent slot; else that slot (in every env).
        Batch extension: env_mask (N,) bool restricts the update to those envs — the parameter table then
        becomes per env ([N*A][18], dynamics randomisation); `params` may also be a (N, 18) / (N, A, 18) tensor
        of per-env parameter vectors (key order maps.PARAM_KEYS)."""
        if not (agent_idx < 0 or 0 <= agent_idx < self.num_agents):
            raise IndexError('Index given is out of bounds for list of agents.')
        N, A = self.num_envs, self.num_agents
        per_env_values = not isinstance(params, dict)
        if env_mask is None and not per_env_values and not self.c.params_per_env:
            pv = torch.from_numpy(hostmaps.params_vector(params)).to(self.device)
            if agent_idx < 0:
                self.params_dev[:] = pv
            else:
                self.params_dev[agent_idx] = pv
            return
        self._params_per_env()
        if per_env_values:
            pv = torch.as_tensor(params, dtype=torch.float64).to(self.device)
            pv = pv.reshape(N, -1, 18)                        # (N,1,18) broadcasts over agents, or (N,A,18)
        else:
            pv = torch.from_numpy(hostmaps.params_vector(params)).to(self.device).reshape(1, 1, 18)
        m = torch.ones((N,), dtype=torch.bool, device=self.device) if env_mask is None else \
            torch.as_tensor(env_mask).to(device=self.device, dtype=torch.bool)
        tgt = self.params_dev if agent_idx < 0 else self.params_dev[:, agent_idx:agent_idx + 1]
        src = pv if (agent_idx < 0 or pv.shape[1] == 1) else pv[:, agent_idx:agent_idx + 1]
        tgt[m] = src.expand(N, tgt.shape[1], 18)[m]

    def _params_per_env(self):
        """Expand the shared parameter table to one row per env and slot ([N*A][18]), once."""
        if not self.c.params_per_env:
            self.params_dev = self.params_dev.unsqueeze(0).repeat(self.num_envs, 1, 1).contiguous()
            self.c.params = nat.ptr(self.params_dev)
            self.c.params_per_env = 1
            self._graph = None

    @property
    def param_table(self):
        """(N, A, 18) fp64 device view of the parameter table (maps.PARAM_KEYS order), the values the next tick runs with.  A
        view of the live buffer: write through update_params, not into it."""
        N, A = self.num_envs, self.num_agents
        if self.c.params_per_env:
            return self.params_dev.view(N, A, 18)
        return self.params_dev.unsqueeze(0).expand(N, A, 18)

    def set_param_draw(self, ranges, groups=None, per_env=False, seed=0):
        """Per-episode dynamics randomisation (C ABI f110_param_draw, include/f110_param_draw.h): every env that starts a new
        episode gets a fresh car, drawn on the device -- after the auto-reset of tick / autoreset / tick_repeat (after each tick
        of the call), after the restart of episode mode, in every captured graph of those, and on redraw_params.  ranges: a
        {key: (lo, hi)} dict for every slot, or a list of A such dicts ({} = the slot is never drawn); groups: lists of keys
        that share one uniform number (e.g. [['m', 'I']]); per_env: every slot of an env shares its draws; seed: the draw's
        seed.  The draw is f1tenth_gym_b200.param_draw.draw_rows.  Expands the table to per env as update_params does (one
        host read checks its undrawn values) and drops a captured graph.  ValueError for what param_draw.parse refuses and for
        undrawn values of a drawn slot that break the sign conditions (DESIGN §3.13).  None turns the draws off and keeps the
        table."""
        self._graph = None
        if ranges is None:
            self._param_draw = self.param_draw = None
            self.param_lo = self.param_hi = self.final_params = None
            return
        d = pdraw.parse(ranges, groups, per_env, seed, self.num_agents)
        pdraw.check_table(self.param_table.cpu().numpy(), d)
        self._params_per_env()
        dev = self.device
        self.param_lo = torch.from_numpy(d['lo']).to(dev)
        self.param_hi = torch.from_numpy(d['hi']).to(dev)
        self.final_params = self.params_dev.clone()
        keys = (C.c_uint32 * 32)(*[int(v) for v in d['keys']])
        group = (C.c_int32 * 18)(*[int(v) for v in d['group']])
        self._param_draw = nat.F110ParamDraw(nat.ptr(self.param_lo), nat.ptr(self.param_hi), keys, group,
                                             1 if d['per_env'] else 0, d['seed'], nat.ptr(self.final_params))
        self.param_draw = d         # the validated draw on the host (param_draw.parse), for draw_rows

    def redraw_params(self, env_mask=None):
        """Draw the masked envs' parameters now (None: every env), at the current tick counter (C ABI f110_params_draw), as
        F110Env.reset does after placing the agents.  The draw is a function of (seed, tick counter, env, slot, group), so a
        redraw at the counter of an env's previous draw repeats it.  ValueError without set_param_draw."""
        if self._param_draw is None:
            raise ValueError('redraw_params needs set_param_draw first')
        m, mp = self._mask_ptr(env_mask)
        nat.check(nat.lib().f110_params_draw(C.byref(self.c), C.byref(self._param_draw), mp, _stream_ptr(self.device)))

    def _draw_autoreset(self, L):
        if self._param_draw is not None:
            nat.check(L.f110_params_draw_autoreset(C.byref(self.c), C.byref(self._param_draw), _stream_ptr(self.device)))

    def _draw_episodes(self, L):
        if self._param_draw is not None:
            nat.check(L.f110_params_draw_episodes(C.byref(self.c), C.byref(self._param_draw), C.byref(self._episodes),
                                                  _stream_ptr(self.device)))

    def set_noise(self, std_dev, seed=None):
        """Scan noise N(0, std_dev^2) (laser_models.py:429,450-452); 0 disables (parity runs)."""
        self.c.noise_std = float(std_dev)
        if seed is not None:
            self.c.noise_seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self._graph = None

    # ------------------------------------------------------------------ helpers
    def _poses_tensor(self, poses):
        N, A = self.num_envs, self.num_agents
        p = torch.as_tensor(poses, dtype=torch.float64)
        if p.dim() == 2:
            if p.shape[0] != A:
                raise ValueError('Number of poses for reset does not match number of agents.')
            p = p.unsqueeze(0).expand(N, A, 3)
        elif p.dim() != 3 or p.shape[0] != N or p.shape[1] != A:
            raise ValueError('Number of poses for reset does not match number of agents.')
        return p.to(self.device).contiguous()

    def _actions_tensor(self, control_inputs):
        N, A = self.num_envs, self.num_agents
        a = control_inputs
        if not (torch.is_tensor(a) and a.is_cuda and a.dtype == torch.float64 and a.is_contiguous()
                and a.numel() == N * A * 2):
            a = torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a, dtype=torch.float64)
            if a.dim() == 2 and N > 1:
                a = a.unsqueeze(0).expand(N, A, 2)
            if a.numel() != N * A * 2:
                raise ValueError('control_inputs must have shape (num_envs, num_agents, 2)')
            self._actions_dev.copy_(a.reshape(N * A, 2), non_blocking=True)
            a = self._actions_dev
        return a

    def _mask_ptr(self, env_mask):
        if env_mask is None:
            return None, None
        m = torch.as_tensor(env_mask).to(device=self.device, dtype=torch.uint8).contiguous()
        if m.numel() != self.num_envs:
            raise ValueError('env_mask must have num_envs entries')
        return m, nat.ptr(m)

    # ------------------------------------------------------------------ reference-surface methods
    def reset(self, poses, env_mask=None):
        """Simulator.reset (base_classes.py:614-630): zero state, place agents, empty steer FIFO.
        poses: (A,3) broadcast to every env, or (N,A,3).  env_mask (N,) bool: partial reset."""
        p = self._poses_tensor(poses)
        m, mp = self._mask_ptr(env_mask)
        nat.check(nat.lib().f110_reset(C.byref(self.c), nat.ptr(p), mp, _stream_ptr(self.device)))
        self._unacquire(m)

    def env_reset(self, poses, env_mask=None):
        """Counters and start frame of F110Env.reset (f110_env.py:319-331) + Simulator.reset."""
        p = self._poses_tensor(poses)
        m, mp = self._mask_ptr(env_mask)
        L = nat.lib()
        nat.check(L.f110_env_reset(C.byref(self.c), nat.ptr(p), mp, _stream_ptr(self.device)))
        nat.check(L.f110_reset(C.byref(self.c), nat.ptr(p), mp, _stream_ptr(self.device)))
        self._unacquire(m)
        if self.ep_ticks is not None:       # a device-side masked fill: no host synchronisation
            if m is None:
                self.ep_ticks.zero_()
            else:
                self.ep_ticks.masked_fill_(m.bool(), 0)

    def _unacquire(self, mask):
        """seg = -1 (not acquired) for the agents of the masked envs (mask: (N,) uint8 device tensor, or None = all)."""
        if self.track_seg is None:
            return
        if mask is None:
            self.track_seg.fill_(-1)
        else:
            self.track_seg.view(self.num_envs, self.num_agents).masked_fill_(mask.bool()[:, None], -1)

    def step(self, control_inputs):
        """Simulator.step (base_classes.py:553-612). control_inputs (N,A,2) = (steer, speed)."""
        a = self._actions_tensor(control_inputs)
        nat.check(nat.lib().f110_step_lidar(C.byref(self.c), C.byref(self._map_struct), C.byref(self._march_tables),
                                            C.byref(self.beams.c), nat.ptr(a), self._obst_ref(), self._lidar_ref(),
                                            _stream_ptr(self.device)))
        return self.observations()

    def env_post_step(self):
        """Tail of F110Env.step: time + lap logic + done (f110_env.py:294-302, 204-246)."""
        nat.check(nat.lib().f110_env_post_step(C.byref(self.c), _stream_ptr(self.device)))

    def _start_table(self, poses):
        """Auto-reset start poses -> (device (K,3) table, K).  `poses` is one (K,3) device tensor shared by every env, or, for
        a stacked DeviceMap, a list of one (K_l,3) table per layer: they are concatenated on the device and
        f110_sim.start_offsets is set so that an env restarts from its own map's table."""
        self.c.start_offsets = None
        self.c.num_start_tables = 0
        if poses is None:
            return None, 0
        if not isinstance(poses, (list, tuple)):
            return poses, poses.shape[0]
        layers = getattr(self._map_struct, 'num_layers', 1)
        if layers <= 1 or self.env_layer is None or len(poses) != layers:
            raise ValueError('autoreset_poses as a list needs one start table per layer of the stacked map (%d)'
                             % max(layers, 1))
        tabs = [torch.as_tensor(p, dtype=torch.float64).to(self.device).reshape(-1, 3) for p in poses]
        offs = np.concatenate([[0], np.cumsum([t.shape[0] for t in tabs])]).astype(np.int32)
        self._start_offsets = (C.c_int32 * offs.size)(*offs.tolist())
        self.c.start_offsets = C.addressof(self._start_offsets)
        self.c.num_start_tables = layers
        return torch.cat(tabs).contiguous(), int(offs[-1])

    def autoreset(self, start_poses, pose_gap=23, seed=12345):
        """Reset every env whose ego collided to a hashed draw from start_poses (device (K,3) fp64, or a list of one
        (K_l,3) table per layer of a stacked map)."""
        table, n = self._start_table(start_poses)
        L = nat.lib()
        nat.check(L.f110_autoreset_obst(C.byref(self.c), nat.ptr(table), n, pose_gap, int(seed), 0, self._obst_ref(),
                                        _stream_ptr(self.device)))
        self._draw_autoreset(L)

    def tick(self, control_inputs, env_level=True, autoreset_poses=None, pose_gap=23, seed=12345):
        """One whole tick in three launches (C ABI f110_tick): step + lap logic + optional auto-reset, same
        results as step(); env_post_step(); autoreset()."""
        a = self._actions_tensor(control_inputs)
        table, n = self._start_table(autoreset_poses)
        L = nat.lib()
        episodes = self._episode_path(table, env_level)
        self._enqueue_tick(L, a, env_level, table, n, pose_gap, seed, episodes, progress=False)
        obs = self.observations()
        if episodes:
            obs['terminated'], obs['truncated'] = self.ep_terminated, self.ep_truncated
        return obs

    def _enqueue_tick(self, L, actions, env_level, table, num_start, pose_gap, seed, episodes, progress):
        """Enqueue one tick: the episode tick (f110_tick_episodes) or f110_tick_lidar, the parameter draw of the envs it
        restarted, then update_progress() with progress."""
        if episodes:
            self._episodes.track_seg = nat.ptr(self.track_seg)
            nat.check(L.f110_tick_episodes(C.byref(self.c), C.byref(self._map_struct), C.byref(self._march_tables),
                                           C.byref(self.beams.c), nat.ptr(actions), nat.ptr(table), num_start, pose_gap,
                                           int(seed), self._obst_ref(), self._lidar_ref(), C.byref(self._episodes),
                                           _stream_ptr(self.device)))
            self._draw_episodes(L)
        else:
            nat.check(L.f110_tick_lidar(C.byref(self.c), C.byref(self._map_struct), C.byref(self._march_tables),
                                        C.byref(self.beams.c), nat.ptr(actions), 1 if env_level else 0, nat.ptr(table),
                                        num_start, pose_gap, int(seed), self._obst_ref(), self._lidar_ref(),
                                        _stream_ptr(self.device)))
            if table is not None:
                self._draw_autoreset(L)
        if progress:
            self._launch_progress(L)

    # ------------------------------------------------------------------ episodes
    def set_episodes(self, max_ticks=None):
        """Episode mode (C ABI f110_tick_episodes, include/f110_episodes.h): tick() and capture_graph() with autoreset_poses then
        end an env's episode when it is done (terminated: ego collision or every agent checkpoint-done) or has run max_ticks
        ticks (truncated; None or 0: no time limit), keep its final observation in final_observation, and restart it as
        F110Env.reset does: the auto-reset's start-pose draw, then one zero-action tick of that env alone, whose observation
        the env then holds.  The tick that ends an episode still reports done = 1.  False turns the mode off.  Drops a
        captured graph.  ValueError for a negative max_ticks or more than 32 agents per env."""
        self._graph = None
        if max_ticks is False:
            self._episodes = None
            self.ep_ticks = self.ep_terminated = self.ep_truncated = self.ep_length = None
            self.final_state = self.final_scans = self.final_collisions = self.final_collision_idx = None
            self.final_lap_times = self.final_lap_counts = self.ep_list = self.ep_list_count = None
            self.ep_end_tick = self.ep_snap_rec = self.ep_snap_poses = self.ep_snap_wall_flag = None
            self.ep_scan_list = self.ep_scan_count = None
            self._episode_repeat = None
            return
        T = 0 if max_ticks is None else max_ticks
        if isinstance(T, bool) or int(T) != T or int(T) < 0 or int(T) > 0x7FFFFFFF:
            raise ValueError('max_ticks must be None or an int >= 0, got %r' % (max_ticks,))
        if self.num_agents > 32:
            raise ValueError('episode mode restarts envs of at most 32 agents, this simulator has %d' % self.num_agents)
        N, NA, dev = self.num_envs, self.num_envs * self.num_agents, self.device
        if self._episodes is None:
            f64 = dict(dtype=torch.float64, device=dev)
            self.ep_ticks = torch.zeros((N,), dtype=torch.int32, device=dev)
            self.ep_terminated = torch.zeros((N,), dtype=torch.uint8, device=dev)
            self.ep_truncated = torch.zeros((N,), dtype=torch.uint8, device=dev)
            self.ep_length = torch.zeros((N,), dtype=torch.int32, device=dev)
            self.final_state = torch.zeros((7, NA), **f64)
            self.final_scans = torch.zeros((NA, self.num_beams), dtype=torch.float32, device=dev)
            self.final_collisions = torch.zeros((NA,), **f64)
            self.final_collision_idx = torch.full((NA,), -1, dtype=torch.int32, device=dev)
            self.final_lap_times = torch.zeros((NA,), **f64)
            self.final_lap_counts = torch.zeros((NA,), **f64)
            self.ep_list = torch.zeros((N,), dtype=torch.int32, device=dev)
            self.ep_list_count = torch.zeros((1,), dtype=torch.int32, device=dev)
            # episodes under a held action (tick_repeat / capture_graph with repeat > 1)
            self.ep_end_tick = torch.full((N,), -1, dtype=torch.int32, device=dev)
            self.ep_snap_rec = torch.zeros((NA, 8), **f64)
            self.ep_snap_poses = torch.zeros((NA, 5), **f64)
            self.ep_snap_wall_flag = torch.zeros((NA,), dtype=torch.int32, device=dev)
            self.ep_scan_list = torch.zeros((N,), dtype=torch.int32, device=dev)
            self.ep_scan_count = torch.zeros((1,), dtype=torch.int32, device=dev)
            self._episode_repeat = nat.F110EpisodeRepeat(nat.ptr(self.ep_end_tick), nat.ptr(self.ep_snap_rec),
                                                         nat.ptr(self.ep_snap_poses), nat.ptr(self.ep_snap_wall_flag),
                                                         nat.ptr(self.ep_scan_list), nat.ptr(self.ep_scan_count), None)
        self._episodes = nat.F110Episodes(int(T), nat.ptr(self.ep_ticks), nat.ptr(self.ep_terminated), nat.ptr(self.ep_truncated),
                                          nat.ptr(self.ep_length), nat.ptr(self.final_state), nat.ptr(self.final_scans),
                                          nat.ptr(self.final_collisions), nat.ptr(self.final_collision_idx),
                                          nat.ptr(self.final_lap_times), nat.ptr(self.final_lap_counts), nat.ptr(self.ep_list),
                                          nat.ptr(self.ep_list_count), None)

    @property
    def episode_ticks(self):
        """(N,) int32: ticks of each env's running episode (the restart's zero-action tick does not count)."""
        return self.ep_ticks

    @property
    def terminated(self):
        """(N,) uint8: the env's episode ended on the last episode tick because it was done."""
        return self.ep_terminated

    @property
    def truncated(self):
        """(N,) uint8: the env's episode ended on the last episode tick at the time limit without being done."""
        return self.ep_truncated

    @property
    def end_tick(self):
        """(N,) int32: the tick 0..K-1 of the last tick_repeat call in episode mode at which the env's episode ended, -1 = none."""
        return self.ep_end_tick

    @property
    def episode_length(self):
        """(N,) int32: ticks of each env's last ended episode."""
        return self.ep_length

    @property
    def final_observation(self):
        """The last ended episode's final observation of each env, shaped like observations(): views of the final_* buffers,
        bit for bit what the tick that ended it left, rewritten only when the env ends another episode.  'params' (N, A, 18) is the
        parameter table the episode ran with: with set_param_draw the rows the restart's draw replaced, else the table."""
        if self._episodes is None:
            return None
        N, A, B = self.num_envs, self.num_agents, self.num_beams
        st = self.final_state
        return {'ego_idx': self.ego_idx, 'scans': self.final_scans.view(N, A, B),
                'poses_x': st[0].view(N, A), 'poses_y': st[1].view(N, A), 'poses_theta': st[4].view(N, A),
                'linear_vels_x': st[3].view(N, A), 'linear_vels_y': self._zeros_NA, 'ang_vels_z': st[5].view(N, A),
                'collisions': self.final_collisions.view(N, A), 'collision_idx': self.final_collision_idx.view(N, A),
                'lap_times': self.final_lap_times.view(N, A), 'lap_counts': self.final_lap_counts.view(N, A),
                'params': self.param_table if self._param_draw is None else self.final_params.view(N, A, 18)}

    def _episode_path(self, table, env_level):
        if self._episodes is None or table is None:
            return False
        if not env_level:
            raise ValueError('episode mode needs env_level=True: the end of an episode is decided by done')
        return True

    def _no_episodes(self, who):
        if self._episodes is not None:
            raise ValueError('%s does not run episode mode; call set_episodes(False) first or use tick / capture_graph' % who)

    # ------------------------------------------------------------------ agents without a lidar
    def set_lidar(self, slots):
        """Which agent slots have a lidar (C ABI f110_lidar): a length-A sequence of bools, the same for every env, or None for
        all.  A sensorless agent is simulated exactly as before -- dynamics, the iTTC wall check on its wall-only scan, collisions,
        lap logic, done, auto-reset, obstacle contact -- and the other agents still see its body; only its own scan is not
        computed.  Its row of `scans` is filled with NaN here, once, and no tick writes it while the short path runs (no scan
        noise, a lean ray march, beams.side_max below max_range, at most 32 agents per env); on any other configuration the mask
        is ignored and every scan is computed as without it.  step, tick, tick_repeat (its last tick) and capture_graph use the
        mask; the host-buffer paths and step_profile raise ValueError while a slot is sensorless.  A slot that gets its lidar
        back has its scan from the next tick on.  Drops a captured graph.  ValueError for a wrong length, or for more than 32
        agents with a False entry."""
        A, N = self.num_agents, self.num_envs
        new = (True,) * A if slots is None else tuple(bool(v) for v in slots)
        if len(new) != A:
            raise ValueError('lidar needs one bool per agent slot (%d), got %d' % (A, len(new)))
        if not all(new) and A > 32:
            raise ValueError('a lidar mask covers at most 32 agent slots, this simulator has %d' % A)
        old = self._lidar_slots
        self._lidar_slots = new
        self._graph = None
        if all(new):
            self._lidar = None
        else:
            if self.lidar_list is None:
                dev = self.device
                self.lidar_list = torch.zeros((N * A,), dtype=torch.int32, device=dev)
                self.lidar_list_count = torch.zeros((1,), dtype=torch.int32, device=dev)
                self.lidar_listed = torch.zeros((1,), dtype=torch.int64, device=dev)
            mask = sum(1 << i for i, v in enumerate(new) if v)
            self._lidar = nat.F110Lidar(mask, nat.ptr(self.lidar_list), nat.ptr(self.lidar_list_count),
                                        nat.ptr(self.lidar_listed))
            off = [i for i, v in enumerate(new) if not v and old[i]]
            if off:     # so that a stale row cannot pass for a scan
                self.scans.view(N, A, self.num_beams)[:, off] = float('nan')
        back = [i for i, v in enumerate(new) if v and not old[i]]
        if back and self.march_cost is not None:
            # no lookup history while the slot was sensorless: its items are queued as very heavy, as after a reset
            self.march_cost.view(N, A, 256)[:, back] = -1

    @property
    def lidar(self):
        """Which agent slots have a lidar (set_lidar): a tuple of A bools."""
        return self._lidar_slots

    def _lidar_ref(self):
        return None if self._lidar is None else C.byref(self._lidar)

    def _no_lidar_mask(self, who):
        if self._lidar is not None:
            raise ValueError('%s computes every scan; call set_lidar(None) first or use step / tick' % who)

    # ------------------------------------------------------------------ static box obstacles
    def _obst_ref(self):
        return None if self._obst is None else C.byref(self._obst)

    def _no_obstacles(self, who):
        if self._obst is not None:
            raise ValueError('%s does not simulate obstacles; call clear_obstacles() first or use step / tick' % who)

    def set_obstacles(self, boxes, active=None):
        """Static box obstacles (C ABI f110_obstacles, csrc/obstacles.cuh): parked cars of an env without a sensor that never
        move.  Every agent's scan is clipped against the boxes of its env, contact sets collisions (collision_idx = A + slot)
        without zeroing state, and the iTTC check does not see them.  boxes: (K, 5) rows (x, y, yaw, length, width) for every
        env, or (N, K, 5); 1 <= K <= 16.  active: (K,) or (N, K) bools, default all.  A slot that is inactive, not finite or of
        size <= 0 is absent.  The data land in obstacle_boxes (N, K, 5) / obstacle_active (N, K), which every tick reads afresh
        (write into them to move boxes, also under a captured graph); obstacle_hit (N*A,) int32 gets the highest slot each
        agent touched on the last tick, -1 = none.  Keeps the respawn draw of set_obstacle_draw when K is unchanged."""
        N = self.num_envs
        b = torch.as_tensor(boxes, dtype=torch.float64)
        if b.dim() == 2:
            b = b.unsqueeze(0).expand(N, -1, -1)
        if b.dim() != 3 or b.shape[0] != N or b.shape[2] != 5 or not 1 <= b.shape[1] <= nat.MAX_OBSTACLES:
            raise ValueError('boxes must be (K, 5) or (num_envs, K, 5) with 1 <= K <= %d, got %s'
                             % (nat.MAX_OBSTACLES, tuple(b.shape)))
        K = b.shape[1]
        act = torch.ones((N, K), dtype=torch.bool) if active is None else torch.as_tensor(active).to(torch.bool)
        if act.dim() == 1:
            act = act.unsqueeze(0).expand(N, -1)
        if tuple(act.shape) != (N, K):
            raise ValueError('active must be (K,) or (num_envs, K) with K = %d, got %s' % (K, tuple(act.shape)))
        if self._obst is None or self._obst.per_env != K:
            dev = self.device
            self.obstacle_boxes = torch.zeros((N, K, 5), dtype=torch.float64, device=dev)
            self.obstacle_active = torch.zeros((N, K), dtype=torch.uint8, device=dev)
            self.obstacle_hit = torch.full((N * self.num_agents,), -1, dtype=torch.int32, device=dev)
            self._obst = nat.F110Obstacles(K, nat.ptr(self.obstacle_boxes), nat.ptr(self.obstacle_active),
                                           nat.ptr(self.obstacle_hit), None, None, 0, 0, 0, 0, 0.0, 0)
            self._obst_keep = ()
            self._graph = None
        self.obstacle_boxes.copy_(b)
        self.obstacle_active.copy_(act.to(torch.uint8))

    def set_obstacle_draw(self, candidates, count=(1, 1), clearance=1.0, seed=0):
        """Redraw an env's boxes whenever the auto-reset restarts it (and on respawn_obstacles): candidates is one (C, 5) table of
        boxes for every env, or for a stacked map a list of one table per layer; slot k takes a hashed row of its env's table,
        count = (lo, hi) slots are active (uniform, lo <= hi <= K), and a box whose centre lies closer than `clearance` metres to
        an agent's new position stays inactive.  The draw is f1tenth_gym_b200.obstacles.respawn_draw.  Needs set_obstacles."""
        if self._obst is None:
            raise ValueError('set_obstacle_draw needs set_obstacles first')
        K = self._obst.per_env
        try:
            lo, hi = (int(v) for v in count)
        except (TypeError, ValueError):
            raise ValueError('count must be (lo, hi), got %r' % (count,))
        if not 0 <= lo <= hi <= K:
            raise ValueError('count must satisfy 0 <= lo <= hi <= K = %d, got %r' % (K, count))
        clearance = float(clearance)
        if not (np.isfinite(clearance) and clearance >= 0.0):
            raise ValueError('clearance must be finite and >= 0, got %r' % clearance)
        per_layer = isinstance(candidates, (list, tuple))
        tabs = list(candidates) if per_layer else [candidates]
        tabs = [torch.as_tensor(np.asarray(t) if not torch.is_tensor(t) else t, dtype=torch.float64).reshape(-1, 5) for t in tabs]
        if any(t.shape[0] < 1 or not bool(torch.isfinite(t).all()) for t in tabs):
            raise ValueError('every candidate table needs at least one finite (x, y, yaw, length, width) row')
        layers = getattr(self._map_struct, 'num_layers', 1)
        offs = None
        if per_layer:
            if layers <= 1 or self.env_layer is None or len(tabs) != layers:
                raise ValueError('candidates as a list needs one table per layer of the stacked map (%d)' % max(layers, 1))
            offs = np.concatenate([[0], np.cumsum([t.shape[0] for t in tabs])]).astype(np.int32)
        cand = torch.cat(tabs).to(self.device).contiguous()
        self._obst_offsets = None if offs is None else (C.c_int32 * offs.size)(*offs.tolist())
        self._obst_keep = (cand,)
        o = self._obst
        o.candidates, o.num_candidates = nat.ptr(cand), cand.shape[0]
        o.cand_offsets = None if offs is None else C.addressof(self._obst_offsets)
        o.num_cand_tables = 0 if offs is None else layers
        o.count_min, o.count_max, o.clearance = lo, hi, clearance
        o.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self._graph = None

    def respawn_obstacles(self, env_mask=None):
        """The respawn draw for the masked envs (None: all) around the agents' current positions, at the current tick counter
        (reads it: one host synchronisation).  Call it after placing the agents."""
        if self._obst is None or not self._obst.candidates:
            raise ValueError('respawn_obstacles needs set_obstacles and set_obstacle_draw first')
        m, mp = self._mask_ptr(env_mask)
        nat.check(nat.lib().f110_obstacles_respawn(C.byref(self.c), C.byref(self._obst), mp, int(self.tick_counter.item()),
                                                   _stream_ptr(self.device)))

    def clear_obstacles(self):
        """Remove every obstacle: the simulator runs exactly as without them."""
        self._obst = None
        self.obstacle_boxes = self.obstacle_active = self.obstacle_hit = None
        self._obst_keep = ()
        self._graph = None

    def _repeat_struct(self):
        """The f110_repeat outputs and scratch, allocated once."""
        if self._repeat_c is None:
            N, NA, dev = self.num_envs, self.num_envs * self.num_agents, self.device
            self.done_any = torch.zeros((N,), dtype=torch.uint8, device=dev)
            self.done_tick = torch.full((N,), -1, dtype=torch.int32, device=dev)
            self.repeat_list = torch.zeros((NA,), dtype=torch.int32, device=dev)
            self.repeat_list_count = torch.zeros((nat.MAX_REPEAT,), dtype=torch.int32, device=dev)
            self.marched_agents = torch.zeros((1,), dtype=torch.int64, device=dev)
            self._repeat_c = nat.F110Repeat(nat.ptr(self.done_any), nat.ptr(self.done_tick), nat.ptr(self.repeat_list),
                                            nat.ptr(self.repeat_list_count), nat.ptr(self.marched_agents))
        return self._repeat_c

    def _check_repeat(self, repeat):
        if int(repeat) != repeat or not 1 <= int(repeat) <= nat.MAX_REPEAT:
            raise ValueError('repeat must be an int in [1, %d], got %r' % (nat.MAX_REPEAT, repeat))
        return int(repeat)

    def _issue_repeat(self, L, actions, K, call, env_level, table, num_start, pose_gap, seed, progress, episodes=False):
        """Enqueue one f110_tick_repeat call (f110_tick_repeat_episodes with episodes=True); progress: the tracker is updated
        after every tick of the call (the same ticks, issued one by one) and track_delta_sum gets the sum of the call's deltas."""
        def ticks(first, count):
            if episodes:
                nat.check(L.f110_tick_repeat_episodes_ticks(
                    C.byref(self.c), C.byref(self._map_struct), C.byref(self._march_tables), C.byref(self.beams.c),
                    nat.ptr(actions), K, first, count, C.byref(call), nat.ptr(table), num_start, pose_gap, int(seed),
                    self._obst_ref(), self._lidar_ref(), C.byref(self._episodes), C.byref(self._episode_repeat),
                    _stream_ptr(self.device)))
                return
            nat.check(L.f110_tick_repeat_ticks_lidar(C.byref(self.c), C.byref(self._map_struct), C.byref(self._march_tables),
                                                     C.byref(self.beams.c), nat.ptr(actions), K, first, count, C.byref(call),
                                                     1 if env_level else 0, nat.ptr(table), num_start, pose_gap, int(seed),
                                                     self._obst_ref(), self._lidar_ref(), _stream_ptr(self.device)))
        if episodes:
            self._episodes.track_seg = nat.ptr(self.track_seg)
            self._episode_repeat.track_delta_sum = nat.ptr(self.track_delta_sum) if progress else None
        # the in-call auto-reset restarts envs on every tick: with a draw, each tick is issued alone and followed by the draw
        per_tick_draw = self._param_draw is not None and not episodes and table is not None
        if not progress and not per_tick_draw:
            ticks(0, K)
        else:
            for t in range(K):
                ticks(t, 1)
                if per_tick_draw:
                    self._draw_autoreset(L)
                if progress:
                    nat.check(L.f110_track_progress_sum(C.byref(self.c), C.byref(self.centerlines.c), C.byref(self._progress_c),
                                                        nat.ptr(self.track_delta_sum), 1 if t == 0 else 0,
                                                        _stream_ptr(self.device)))
        if episodes:
            self._draw_episodes(L)

    def _repeat_call(self, env_level, progress):
        """The f110_repeat struct of a call (without the done outputs when the env level is off) after allocating what the
        call writes."""
        rep = self._repeat_struct()
        if progress:
            if self.centerlines is None:
                raise ValueError('no centerlines: call set_centerlines first')
            if self.track_delta_sum is None:
                self.track_delta_sum = torch.zeros_like(self.track_delta)
        return rep if env_level else nat.F110Repeat(None, None, rep.list, rep.list_count, rep.marched_agents)

    def tick_repeat(self, control_inputs, repeat, env_level=True, autoreset_poses=None, pose_gap=23, seed=12345, progress=False):
        """`repeat` ticks under one action in one call (C ABI f110_tick_repeat): everything except the scans is what `repeat`
        calls of tick() leave, and the scans are the last tick's.  Returns observations() plus 'done_any' (N,) uint8, whether
        an env was done on any tick of the call, and 'done_tick' (N,) int32, the first such tick or -1 (device views, overwritten
        by the next call; both need env_level).  On the ticks before the last only the agents a wall could stop are marched.
        progress=True (needs set_centerlines): update_progress() after every tick of the call; track_delta_sum (N*A,) then
        holds each agent's progress over the whole call.
        In episode mode (set_episodes) with autoreset_poses and env_level (C ABI f110_tick_repeat_episodes): an env's episode
        stops at the first tick of the call that ends it; its final_observation, episode_length and flags are that tick's, done
        is that tick's and done_any / done_tick count the ticks up to it; after the call it is restarted as tick() restarts it.
        The other envs are what tick_repeat leaves.  Adds 'terminated', 'truncated' and 'end_tick' (the tick 0..K-1 at which
        the episode ended, -1 = none); with progress=True a restarted env's track_delta_sum is 0.  Episode mode without
        autoreset_poses raises ValueError.  With set_param_draw, an env restarted by the in-call auto-reset is drawn right after
        its tick (the call is then issued tick by tick) and drives the rest of the call on its new car; in episode mode the
        restarted envs are drawn after the call."""
        K = self._check_repeat(repeat)
        a = self._actions_tensor(control_inputs)
        table, n = self._start_table(autoreset_poses)
        episodes = self._episode_path(table, env_level)
        if not episodes:
            self._no_episodes('tick_repeat without autoreset_poses')
        call = self._repeat_call(env_level, progress)
        self._issue_repeat(nat.lib(), a, K, call, env_level, table, n, pose_gap, seed, progress, episodes)
        self._repeat_ticks += (K - 1) * self.num_envs * self.num_agents
        self._repeat_plain = b'sub=full' in nat.lib().f110_debug_last_launch()      # the call ran plain ticks throughout
        obs = self.observations()
        if env_level:
            obs['done_any'], obs['done_tick'] = self.done_any, self.done_tick
        if episodes:
            obs['terminated'], obs['truncated'], obs['end_tick'] = self.ep_terminated, self.ep_truncated, self.ep_end_tick
        return obs

    def marched_fraction(self):
        """Share of the agent-ticks on the intermediate ticks of the tick_repeat calls since the last reading that had to be
        ray-marched (1.0 when the calls ran plain ticks; None before any intermediate tick).  Synchronises the host: a
        measurement, not for the hot loop.  Calls replayed from a captured graph are not counted."""
        if self._repeat_ticks == 0:
            return None
        frac = 1.0 if self._repeat_plain else float(self.marched_agents.item()) / self._repeat_ticks
        self.marched_agents.zero_()
        self._repeat_ticks = 0
        return frac

    def observations(self):
        N, A, B = self.num_envs, self.num_agents, self.num_beams
        st = self.state
        return {'ego_idx': self.ego_idx,
                'scans': self.scans.view(N, A, B),
                'poses_x': st[0].view(N, A), 'poses_y': st[1].view(N, A), 'poses_theta': st[4].view(N, A),
                'linear_vels_x': st[3].view(N, A),
                'linear_vels_y': self._zeros_NA,
                'ang_vels_z': st[5].view(N, A),
                'collisions': self.collisions.view(N, A)}

    # ------------------------------------------------------------------ centerline progress
    def set_centerlines(self, tables, window=(8, 56), reacquire_dist=5.0):
        """Closed centerlines for update_progress / project_centerline (C ABI f110_track, csrc/progress.cuh): one (n, 2) table
        of (x, y) in metres for a single map, or a list of one table per layer of a stacked map; progress runs in row order.
        A last row equal to the first is dropped.  window = (back, fwd): a tracked agent searches segments seg - back ..
        seg + fwd; reacquire_dist: a window whose best distance exceeds it falls back to the global projection.  ValueError for
        a table of fewer than 3 points, non-finite values, a zero-length segment, a table count other than the map's layer
        count, back + fwd + 1 outside [1, 1024] or reacquire_dist not finite and > 0.  Every agent starts unacquired.
        None turns tracking off."""
        self._graph = None
        self.track_delta_sum = None
        if tables is None:
            self.centerlines = None
            self.track_seg = self.track_s = self.track_d = self.track_heading_error = None
            self.track_progress = self.track_delta = None
            return
        try:
            back, fwd = (int(v) for v in window)
        except (TypeError, ValueError):
            raise ValueError('window must be (back, fwd), got %r' % (window,))
        if back < 0 or fwd < 0 or back + fwd + 1 > TRACK_MAX_WINDOW:
            raise ValueError('window (back, fwd) needs back, fwd >= 0 and back + fwd + 1 <= %d, got %r'
                             % (TRACK_MAX_WINDOW, window))
        r = float(reacquire_dist)
        if not (np.isfinite(r) and r > 0.0):
            raise ValueError('reacquire_dist must be finite and > 0, got %r' % (reacquire_dist,))
        ct = CenterlineTables(tables, self.device)
        layers = max(1, int(getattr(self._map_struct, 'num_layers', 1)))
        if ct.num_tables != layers:
            raise ValueError('%d centerline tables for a map of %d layers' % (ct.num_tables, layers))
        N, A = self.num_envs, self.num_agents
        f64 = dict(dtype=torch.float64, device=self.device)
        self.centerlines = ct
        self.track_seg = torch.full((N * A,), -1, dtype=torch.int32, device=self.device)
        self.track_s, self.track_d, self.track_heading_error, self.track_progress, self.track_delta = (
            torch.zeros((N * A,), **f64) for _ in range(5))
        self._progress_c = nat.F110Progress(nat.ptr(self.track_seg), nat.ptr(self.track_s), nat.ptr(self.track_d),
                                            nat.ptr(self.track_heading_error), nat.ptr(self.track_progress),
                                            nat.ptr(self.track_delta), back, fwd, r)
        self._progress_views = {'s': self.track_s.view(N, A), 'd': self.track_d.view(N, A),
                                'heading_error': self.track_heading_error.view(N, A),
                                'progress': self.track_progress.view(N, A), 'delta': self.track_delta.view(N, A)}

    def _launch_progress(self, L):
        nat.check(L.f110_track_progress(C.byref(self.c), C.byref(self.centerlines.c), C.byref(self._progress_c),
                                        _stream_ptr(self.device)))

    def update_progress(self):
        """One launch (C ABI f110_track_progress): every agent's progress along its map's centerline from the current pose.
        Returns views (N, A) 's', 'd', 'heading_error', 'progress', 'delta', overwritten by the next update.
        An agent reset since its last step (reset, env_reset, or the auto-reset of tick) is acquired afresh with progress 0
        and delta 0.  On the tick that auto-resets an env the update sees the new episode: that tick's delta is 0 and the
        crash tick's last partial delta is lost."""
        if self.centerlines is None:
            raise ValueError('no centerlines: call set_centerlines first')
        self._launch_progress(nat.lib())
        return self._progress_views

    def project_centerline(self, poses, table_ids=None):
        """Stateless projection (C ABI f110_track_project) of poses (M, 3) (x, y, yaw) -> fp64 (M, 5) device tensor of
        (seg, t, d, s, heading_error); table_ids (M,) ints pick each pose's table (needed with more than one table).  A
        non-finite pose or a table id outside [0, num_tables) gives a NaN row."""
        if self.centerlines is None:
            raise ValueError('no centerlines: call set_centerlines first')
        p = torch.as_tensor(poses, dtype=torch.float64).to(self.device).reshape(-1, 3).contiguous()
        M = p.shape[0]
        if M < 1:
            raise ValueError('project_centerline needs at least one pose')
        ids = None
        if table_ids is not None:
            ids = torch.as_tensor(table_ids).to(device=self.device, dtype=torch.int32).reshape(-1).contiguous()
            if ids.numel() != M:
                raise ValueError('table_ids must hold one table index per pose')
        elif self.centerlines.num_tables > 1:
            raise ValueError('%d centerline tables: pass table_ids' % self.centerlines.num_tables)
        out = torch.empty((M, 5), dtype=torch.float64, device=self.device)
        nat.check(nat.lib().f110_track_project(C.byref(self.centerlines.c), nat.ptr(p), nat.ptr(ids), M, nat.ptr(out),
                                               _stream_ptr(self.device)))
        return out

    # ------------------------------------------------------------------ predicted futures
    def predict(self, actions, agent_ids=None, record_states=False, record_clearance=False, cost=None, prev_action=None):
        """K candidate futures of M agents, H ticks each, in one launch (C ABI f110_predict, include/f110_predict.h), for
        sampling-based control (MPPI, CEM, random shooting).  actions: (M, K, H, 2) fp64 (steer, speed) per step; agent_ids:
        the M flat source agents e*A + slot (repeats allowed), None = every agent (M = N*A).  Sample (m, k) starts from agent
        agent_ids[m]'s current state, steer FIFO, parameter row and map layer and runs, per step, that agent's tick alone: FIFO,
        pid, RK4 / Euler, yaw wrap, scan pose, the iTTC wall check on the wall-only scan (a hit zeroes state[3:]) -- no scan
        noise, opponents, boxes, laps, done or auto-reset.  With the scan noise off, step h equals the agent's state after h + 1
        ticks of step / tick under the same actions, bit for bit.  Returns {'final_state': (M, K, 7), 'wall_step': (M, K) int32
        (first step whose wall check fired, -1 for none)} plus 'states' (M, K, H, 7) with record_states and 'clearance'
        (M, K, H) fp32 (the distance transform at each step's scan pose, metres) with record_clearance; state order x, y,
        steer, v, yaw, yaw_rate, slip.  The tensors are views of buffers kept while (M, K, H, flags) stay the same and
        overwritten by the next call, so a call after a first one of the same shape can be captured in a CUDA graph.
        Ids given on the host are range-checked (ValueError); a CUDA int32 tensor goes to the kernel unchecked, and an id
        outside [0, N*A) there gives NaN states, wall_step -1 and NaN clearance.  ValueError before any device work for a
        bad shape, dtype, device or size, and for a map on which the held-action short path cannot run (no lean ray march,
        side distances unknown or not below max_range).

        cost: a dict of cost weights (C ABI f110_predict_scored, include/f110_mppi.h) -- any of w_lat, w_head, w_clear, w_dsteer,
        w_dspeed, w_prog, w_wall (finite, >= 0) and clear_min (metres, finite); missing keys take COST_DEFAULTS -- adds
        'cost' (M, K) fp64: per step h, w_lat * d^2 + w_head * e^2 + w_clear * max(0, clear_min - clearance)^2 + w_dsteer *
        (change of steer command)^2 + w_dspeed * (change of speed command)^2, minus w_prog times the progress along the
        centerline after the last step, plus w_wall when the wall check fired.  d, e and the progress are those of the
        set_centerlines tracker (its window and reacquire_dist) started at the source agent's pose; the other outputs are
        unchanged.  prev_action (M, 2): the command before step 0, for the rate terms of step 0 (None: no rate terms there).
        NaN for a sample whose tracker loses the centerline or whose source is invalid.  ValueError before any device work
        without centerlines, for an unknown key, a bad weight or a bad prev_action."""
        NA = self.num_envs * self.num_agents
        cost_c = None if cost is None else self._cost_struct(cost)
        if self.map is None:
            raise ValueError('predict needs a map: call set_map or set_device_map first')
        mc, bc = self._map_struct, self.beams.c
        if not (self.march_rec is not None and mc.sincos2 and mc.dt_min_positive > mc.eps and 0.0 < bc.side_max < mc.max_range):
            raise ValueError('predict needs the lean ray march (march queue, doubled LUT, dt_min_positive > eps) and side '
                             'distances below max_range')
        on_dev = torch.is_tensor(actions) and actions.is_cuda
        if on_dev:
            if actions.dtype != torch.float64 or actions.device != self.state.device:
                raise ValueError('actions on the device must be float64 on %s, got %s on %s'
                                 % (self.state.device, actions.dtype, actions.device))
            act = actions.contiguous()
        else:
            act = torch.as_tensor(np.asarray(actions) if not torch.is_tensor(actions) else actions, dtype=torch.float64)
        if act.dim() != 4 or act.shape[3] != 2:
            raise ValueError('actions must have shape (M, K, H, 2), got %s' % (tuple(act.shape),))
        M, K, H = (int(v) for v in act.shape[:3])
        if agent_ids is None:
            ids = self._view_ids(None)
        elif torch.is_tensor(agent_ids) and agent_ids.is_cuda:
            if agent_ids.dtype != torch.int32 or agent_ids.device != self.state.device:
                raise ValueError('agent_ids on the device must be int32 on %s' % self.state.device)
            ids = agent_ids.reshape(-1).contiguous()
        else:
            ids = None
            a = agent_ids.numpy() if torch.is_tensor(agent_ids) else np.asarray(agent_ids)
            if a.dtype.kind not in 'iu':
                raise ValueError('agent_ids must be integers')
            a = a.reshape(-1)
            if a.size and (int(a.min()) < 0 or int(a.max()) >= NA):
                raise ValueError('agent_ids must lie in [0, %d), got [%d, %d]' % (NA, int(a.min()), int(a.max())))
        n_ids = ids.numel() if ids is not None else a.size
        if n_ids != M:
            raise ValueError('actions hold %d agents, agent_ids %d' % (M, n_ids))
        if M < 1 or K < 1 or not 1 <= H <= nat.PREDICT_MAX_H or M * K > 0x7fffffff:
            raise ValueError('predict needs M >= 1, K >= 1, 1 <= H <= %d and M * K < 2^31, got M=%d K=%d H=%d'
                             % (nat.PREDICT_MAX_H, M, K, H))
        prev = None
        if prev_action is not None:
            if cost is None:
                raise ValueError('prev_action is an input of the cost: pass cost as well')
            prev = torch.as_tensor(prev_action, dtype=torch.float64).to(self.device).contiguous()
            if tuple(prev.shape) != (M, 2):
                raise ValueError('prev_action must have shape (M, 2) = (%d, 2), got %s' % (M, tuple(prev.shape)))
        key = (M, K, H, bool(record_states), bool(record_clearance), cost is not None)
        buf = getattr(self, '_predict_buf', None)
        if buf is None or buf['key'] != key:
            dev = self.device
            buf = {'key': key,
                   'final_state': torch.empty((M, K, 7), dtype=torch.float64, device=dev),
                   'wall_step': torch.empty((M, K), dtype=torch.int32, device=dev),
                   'states': torch.empty((M, K, H, 7), dtype=torch.float64, device=dev) if record_states else None,
                   'clearance': torch.empty((M, K, H), dtype=torch.float32, device=dev) if record_clearance else None,
                   'ids': torch.empty((M,), dtype=torch.int32, device=dev), 'actions': None}
            if cost is not None:
                buf['cost'] = torch.empty((M, K), dtype=torch.float64, device=dev)
                buf['seg0'] = torch.empty((M,), dtype=torch.int32, device=dev)
                buf['s0'] = torch.empty((M,), dtype=torch.float64, device=dev)
            self._predict_buf = buf
        if ids is None:
            buf['ids'].copy_(torch.from_numpy(a.astype(np.int32)), non_blocking=True)
            ids = buf['ids']
        if not on_dev:
            if buf['actions'] is None:
                buf['actions'] = torch.empty((M, K, H, 2), dtype=torch.float64, device=self.device)
            buf['actions'].copy_(act, non_blocking=True)
            act = buf['actions']
        args = nat.F110PredictArgs(nat.ptr(ids), nat.ptr(act), M, K, H, nat.ptr(buf['final_state']), nat.ptr(buf['wall_step']),
                                   nat.ptr(buf['states']), nat.ptr(buf['clearance']))
        if cost_c is None:
            rc = nat.lib().f110_predict(C.byref(self.c), C.byref(mc), C.byref(self._march_tables), C.byref(bc), C.byref(args),
                                        _stream_ptr(self.device))
        else:
            cost_c.prev_action, cost_c.cost, cost_c.seg0, cost_c.s0 = (nat.ptr(prev), nat.ptr(buf['cost']), nat.ptr(buf['seg0']),
                                                                       nat.ptr(buf['s0']))
            rc = nat.lib().f110_predict_scored(C.byref(self.c), C.byref(mc), C.byref(self._march_tables), C.byref(bc),
                                               C.byref(self.centerlines.c), C.byref(args), C.byref(cost_c),
                                               _stream_ptr(self.device))
        if rc == -1:        # F110_ERR_INVALID: nothing was enqueued
            raise ValueError('f110_predict refused this simulator, map or beam setup (see include/f110_predict.h)')
        nat.check(rc)
        out = {'final_state': buf['final_state'], 'wall_step': buf['wall_step']}
        if cost is not None:
            out['cost'] = buf['cost']
        if record_states:
            out['states'] = buf['states']
        if record_clearance:
            out['clearance'] = buf['clearance']
        return out

    def _cost_struct(self, cost):
        """f110_cost from a dict of weights (missing keys: COST_DEFAULTS) and the tracker settings of set_centerlines; the
        pointers are left for the caller.  ValueError without centerlines, for an unknown key or a bad value."""
        if self.centerlines is None:
            raise ValueError('a cost needs centerlines: call set_centerlines first')
        if not isinstance(cost, dict):
            raise ValueError('cost must be a dict of weights, got %r' % (type(cost).__name__,))
        unknown = set(cost) - set(COST_DEFAULTS)
        if unknown:
            raise ValueError('unknown cost keys %s (known: %s)' % (sorted(unknown), sorted(COST_DEFAULTS)))
        w = dict(COST_DEFAULTS)
        for k, v in cost.items():
            try:
                w[k] = float(v)
            except (TypeError, ValueError):
                raise ValueError('cost %s must be a number, got %r' % (k, v))
            if not np.isfinite(w[k]) or (k != 'clear_min' and w[k] < 0.0):
                raise ValueError('cost %s must be finite%s, got %r' % (k, '' if k == 'clear_min' else ' and >= 0', v))
        pc = self._progress_c
        c = nat.F110Cost()
        for k in nat.COST_WEIGHTS + ('clear_min',):
            setattr(c, k, w[k])
        c.back, c.fwd, c.reacquire_dist = pc.back, pc.fwd, pc.reacquire_dist
        return c

    # ------------------------------------------------------------------ views
    def render_views(self, agent_ids=None, size=(64, 64), metres_per_pixel=0.1, forward_offset=0.0, heading_up=True,
                     out=None):
        """Top-down class views (C ABI f110_render_views, csrc/render.cuh) -> uint8 (V, H, W) on the device: 0 off-map,
        1 free, 2 wall (dt == 0), 3 another agent of the env, 4 the followed agent, 5 a static obstacle (set_obstacles), 255 an
        invalid view.  View k follows flat
        agent agent_ids[k] (None: every agent, (N*A, H, W), which reshapes to (N, A, H, W)), centred forward_offset metres
        ahead of it, with its heading up or world-aligned; size = (H, W) pixels of metres_per_pixel each.
        Ids given on the host (int, sequence, numpy, CPU tensor) are range-checked (ValueError); a CUDA tensor must be int32
        (ValueError otherwise) and goes to the kernel unchecked: an id outside [0, N*A) there gives an all-255 view.  With None or a contiguous int32 CUDA
        tensor of ids and `out` (uint8 CUDA (V, H, W), contiguous) the call is exactly one kernel launch."""
        H, W = self._view_size(size)
        s, f = float(metres_per_pixel), float(forward_offset)
        if not (np.isfinite(s) and s > 0.0):
            raise ValueError('metres_per_pixel must be finite and > 0, got %r' % (metres_per_pixel,))
        if not np.isfinite(f):
            raise ValueError('forward_offset must be finite, got %r' % (forward_offset,))
        if self.num_agents > RENDER_MAX_AGENTS:
            raise ValueError('render_views draws at most %d agents per env' % RENDER_MAX_AGENTS)
        ids = self._view_ids(agent_ids)
        V = ids.shape[0]
        if out is None:
            out = torch.empty((V, H, W), dtype=torch.uint8, device=self.device)
        elif not (torch.is_tensor(out) and out.dtype == torch.uint8 and out.device == self.state.device and out.is_contiguous()
                  and tuple(out.shape) == (V, H, W)):
            # (self.state.device, not self.device: device='cuda' has no index, the tensors allocated on it have one)
            raise ValueError('out must be a contiguous uint8 tensor of shape %s on %s' % ((V, H, W), self.state.device))
        nat.check(nat.lib().f110_render_views_obst(C.byref(self.c), C.byref(self._map_struct), self._obst_ref(), nat.ptr(ids), V,
                                                   H, W, s, f, 1 if heading_up else 0, nat.ptr(out), _stream_ptr(self.device)))
        return out

    @staticmethod
    def _view_size(size):
        try:
            H, W = (int(v) for v in size)
        except (TypeError, ValueError):
            raise ValueError('size must be (height, width), got %r' % (size,))
        if tuple(size) != (H, W) or not (1 <= H <= RENDER_MAX_SIZE and 1 <= W <= RENDER_MAX_SIZE):
            raise ValueError('size must be two ints in [1, %d], got %r' % (RENDER_MAX_SIZE, size))
        return H, W

    def _view_ids(self, agent_ids):
        """agent_ids -> contiguous int32 device tensor [V]."""
        NA = self.num_envs * self.num_agents
        if agent_ids is None:
            if getattr(self, '_all_agent_ids', None) is None:
                self._all_agent_ids = torch.arange(NA, dtype=torch.int32, device=self.device)
            return self._all_agent_ids
        if torch.is_tensor(agent_ids) and agent_ids.is_cuda:
            # passed on as they are, without a host synchronisation: only int32 keeps every id the caller wrote (a narrowing
            # cast would wrap 2**32 + 3 to agent 3), and the kernel gives an all-255 view for one outside [0, N*A)
            if agent_ids.dtype != torch.int32:
                raise ValueError('agent_ids on the device must be int32, got %s' % agent_ids.dtype)
            ids = agent_ids.reshape(-1)
        else:
            a = agent_ids.numpy() if torch.is_tensor(agent_ids) else np.asarray(agent_ids)
            if a.dtype.kind not in 'iu':
                raise ValueError('agent_ids must be integers')
            a = a.reshape(-1)
            if a.size and (int(a.min()) < 0 or int(a.max()) >= NA):
                raise ValueError('agent_ids must lie in [0, %d), got [%d, %d]' % (NA, int(a.min()), int(a.max())))
            ids = torch.from_numpy(a.astype(np.int32))
        if ids.numel() < 1:
            raise ValueError('agent_ids must name at least one agent')
        return ids.to(device=self.device, dtype=torch.int32).contiguous()

    # ------------------------------------------------------------------ throughput paths
    def capture_graph(self, actions, autoreset_poses=None, pose_gap=23, autoreset_seed=12345, env_level=False,
                      progress=False, repeat=1):
        """Capture one tick (f110_step [+ env_post_step] [+ autoreset]) reading `actions` (a persistent
        device tensor the caller overwrites between replays) into a CUDA graph.  The warm-up tick that precedes the
        capture runs on a snapshot: every simulation buffer (state, FIFO, scans, lap counters, tick counter / noise
        stream, march queue history, progress tracker) is restored afterwards, so capturing has no side effect on the
        simulation.  progress=True appends update_progress() to the captured tick (needs set_centerlines).
        repeat > 1 captures tick_repeat(actions, repeat) instead (done_any / done_tick with env_level); with progress=True the
        tracker is updated after every tick of the call and track_delta_sum (N*A,) holds the sum of the call's deltas.
        With episode mode set (set_episodes), autoreset_poses and env_level=True capture the episode tick instead, and with
        repeat > 1 the episode call of tick_repeat.  With set_param_draw the draws of those calls are captured with them."""
        assert actions.is_cuda and actions.dtype == torch.float64 and actions.is_contiguous()
        if progress and self.centerlines is None:
            raise ValueError('capture_graph(progress=True) needs set_centerlines first')
        L = nat.lib()
        K = self._check_repeat(repeat)
        if K > 1 and (autoreset_poses is None or not env_level):
            self._no_episodes('capture_graph(repeat > 1) without autoreset_poses and env_level')
        call = self._repeat_call(env_level, progress) if K > 1 else None
        names = ('state', 'steer_buf', 'steer_cnt', 'scan_pose', 'agent_poses', 'scans', 'wall_flag', 'collisions',
                 'collision_idx', 'current_time', 'lap_times', 'lap_counts', 'toggle_list', 'near_starts', 'start_xs',
                 'start_ys', 'start_thetas', 'start_rot', 'done', 'checkpoint_done', 'tick_counter', 'march_cost',
                 'march_order', 'march_count', 'march_rec', 'track_seg', 'track_s', 'track_d', 'track_heading_error',
                 'track_progress', 'track_delta', 'done_any', 'done_tick', 'repeat_list', 'repeat_list_count',
                 'marched_agents', 'track_delta_sum', 'obstacle_boxes', 'obstacle_active', 'obstacle_hit', 'lidar_list',
                 'lidar_list_count', 'lidar_listed', 'ep_ticks', 'ep_terminated', 'ep_truncated', 'ep_length', 'final_state',
                 'final_scans', 'final_collisions', 'final_collision_idx', 'final_lap_times', 'final_lap_counts', 'ep_list',
                 'ep_list_count', 'ep_end_tick', 'ep_snap_rec', 'ep_snap_poses', 'ep_snap_wall_flag', 'ep_scan_list',
                 'ep_scan_count', 'params_dev', 'final_params')
        snapshot = {n: getattr(self, n).clone() for n in names if getattr(self, n, None) is not None}
        table, num_start = self._start_table(autoreset_poses)     # a list of per-layer tables is concatenated once, here
        episodes = self._episode_path(table, env_level)

        def tick():
            if K > 1:
                self._issue_repeat(L, actions, K, call, env_level, table, num_start, pose_gap, autoreset_seed, progress, episodes)
            else:
                self._enqueue_tick(L, actions, env_level, table, num_start, pose_gap, autoreset_seed, episodes, progress)
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            tick()      # warm-up outside capture (module load, first-launch work)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        for n, t in snapshot.items():
            getattr(self, n).copy_(t)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            tick()
        self._graph = g
        self._graph_keep = (actions, table) + ((self.centerlines, self._progress_views) if progress else ()) + \
            ((call,) if K > 1 else ()) + ((self._obst, self.obstacle_boxes, self.obstacle_active, self.obstacle_hit) +
                                          self._obst_keep if self._obst is not None else ()) + \
            ((self._lidar, self.lidar_list, self.lidar_list_count, self.lidar_listed) if self._lidar is not None else ()) + \
            ((self._episodes,) if episodes else ()) + ((self._episode_repeat,) if episodes and K > 1 else ()) + \
            ((self.param_lo, self.param_hi, self.final_params) if self._param_draw is not None else ())
        return g

    def replay(self):
        self._graph.replay()

    def make_host_io(self, with_scans=True, packed_scans=False):
        """Pinned host buffers for step_host() / step_host_async().  packed_scans=True (async path only): the scan block
        crosses PCIe as 24-bit fixed point (io['scans_u24'] uint8 [NA, B, 3]; decode with unpack_scans_u24) instead of fp32."""
        self._no_lidar_mask('make_host_io')
        self._no_episodes('make_host_io')
        N, A, B = self.num_envs, self.num_agents, self.num_beams
        NA = N * A
        if packed_scans:
            with_scans = False
        io = {'actions': torch.zeros((NA, 2), dtype=torch.float64).pin_memory(),
              'scans': torch.zeros((NA, B), dtype=torch.float32).pin_memory() if with_scans else None,
              'scans_u24': torch.zeros((NA, B, 3), dtype=torch.uint8).pin_memory() if packed_scans else None,
              'state': torch.zeros((7, NA), dtype=torch.float64).pin_memory(),
              'collisions': torch.zeros((NA,), dtype=torch.float64).pin_memory(),
              'done': torch.zeros((N,), dtype=torch.uint8).pin_memory(),
              'lap_times': torch.zeros((NA,), dtype=torch.float64).pin_memory(),
              'lap_counts': torch.zeros((NA,), dtype=torch.float64).pin_memory()}
        io['_struct'] = nat.F110HostObs(nat.ptr(io['scans']), nat.ptr(io['state']), nat.ptr(io['collisions']),
                                        nat.ptr(io['done']), nat.ptr(io['lap_times']), nat.ptr(io['lap_counts']),
                                        nat.ptr(io['scans_u24']))
        return io

    @staticmethod
    def unpack_scans_u24(buf):
        """uint8 [..., 3] (io['scans_u24']) -> float32 ranges: (b0 | b1 << 8 | b2 << 16) * 2^-19 m."""
        b = (buf.numpy() if torch.is_tensor(buf) else np.asarray(buf)).astype(np.uint32)
        return ((b[..., 0] | (b[..., 1] << 8) | (b[..., 2] << 16)).astype(np.float32) * np.float32(2.0 ** -19))

    def step_host(self, io):
        """One tick through HOST buffers (C ABI f110_step_host): H2D actions, step, env_post_step,
        D2H observation, stream sync.  io from make_host_io(); fill io['actions'] first.  ValueError with obstacles set."""
        self._no_obstacles('step_host')
        self._no_lidar_mask('step_host')
        self._no_episodes('step_host')
        nat.check(nat.lib().f110_step_host(C.byref(self.c), C.byref(self._map_struct), C.byref(self.beams.c),
                                           nat.ptr(io['actions']), nat.ptr(self._actions_dev),
                                           C.byref(io['_struct']), _stream_ptr(self.device)))
        return io

    def make_host_pipeline(self, depth=2, with_scans=True, packed_scans=False):
        """`depth` independent sets of (pinned host obs, device staging, events, actions scratch) for
        step_host_async(); one shared copy stream.  packed_scans=True: ValueError for a map whose max_range plus 8 sigma of
        the scan noise reaches 32 m, where the 24-bit block clamps (step_host_async checks again once the map or the noise
        changed)."""
        self._no_lidar_mask('make_host_pipeline')
        self._no_episodes('make_host_pipeline')
        N, A, B = self.num_envs, self.num_agents, self.num_beams
        NA = N * A
        dev = self.device
        sets = []
        if packed_scans:
            with_scans = False
            self._check_packed_range()
        copy_stream = torch.cuda.Stream(dev)
        for _ in range(depth):
            io = self.make_host_io(with_scans, packed_scans)
            st = {'scans': torch.zeros((NA, B), dtype=torch.float32, device=dev) if with_scans else None,
                  'scans_u24': torch.zeros((NA, B, 3), dtype=torch.uint8, device=dev) if packed_scans else None,
                  'state': torch.zeros((7, NA), dtype=torch.float64, device=dev),
                  'collisions': torch.zeros((NA,), dtype=torch.float64, device=dev),
                  'done': torch.zeros((N,), dtype=torch.uint8, device=dev),
                  'lap_times': torch.zeros((NA,), dtype=torch.float64, device=dev),
                  'lap_counts': torch.zeros((NA,), dtype=torch.float64, device=dev)}
            io['_stage'] = st
            io['_stage_struct'] = nat.F110HostObs(nat.ptr(st['scans']), nat.ptr(st['state']), nat.ptr(st['collisions']),
                                                  nat.ptr(st['done']), nat.ptr(st['lap_times']), nat.ptr(st['lap_counts']),
                                                  nat.ptr(st['scans_u24']))
            io['_actions_dev'] = torch.zeros((NA, 2), dtype=torch.float64, device=dev)
            io['_ev_tick'] = torch.cuda.Event()
            io['_ev_copy'] = torch.cuda.Event()
            io['_ev_tick'].record()
            io['_ev_copy'].record()
            io['_copy_stream'] = copy_stream
            io['_packed_checked'] = (self._map_struct, self.c.noise_std) if packed_scans else None
            sets.append(io)
        torch.cuda.synchronize(dev)
        return sets

    def _check_packed_range(self):
        """ValueError unless every range of the current map (max_range plus 8 sigma of the scan noise) stays below the 32 m
        where the 24-bit scan block clamps."""
        if self.map is None:
            return
        top = float(self._map_struct.max_range) + 8.0 * max(float(self.c.noise_std), 0.0)
        if not top < PACKED_RANGE_LIMIT:
            raise ValueError('packed_scans holds ranges below %g m only, but this map reaches max_range + 8 * noise_std = %g m'
                             % (PACKED_RANGE_LIMIT, top))

    def step_host_async(self, io):
        """Enqueue one tick whose observation lands in io's pinned host buffers (C ABI f110_step_host_async);
        returns immediately.  Call wait_host(io) before reading them or before reusing io.  With a packed io, ValueError
        (before anything is enqueued) when the map or the noise changed since the last check and now reaches 32 m.  ValueError
        with obstacles set."""
        self._no_obstacles('step_host_async')
        self._no_lidar_mask('step_host_async')
        self._no_episodes('step_host_async')
        if io['scans_u24'] is not None:
            checked = io.get('_packed_checked')
            if checked is None or checked[0] is not self._map_struct or checked[1] != self.c.noise_std:
                self._check_packed_range()
                io['_packed_checked'] = (self._map_struct, self.c.noise_std)
        nat.check(nat.lib().f110_step_host_async_ex(
            C.byref(self.c), C.byref(self._map_struct), C.byref(self._march_tables), C.byref(self.beams.c), nat.ptr(io['actions']),
            nat.ptr(io['_actions_dev']), C.byref(io['_stage_struct']), C.byref(io['_struct']),
            _stream_ptr(self.device), C.c_void_p(io['_copy_stream'].cuda_stream),
            C.c_void_p(io['_ev_tick'].cuda_event), C.c_void_p(io['_ev_copy'].cuda_event)))
        return io

    @staticmethod
    def wait_host(io):
        io['_ev_copy'].synchronize()

    def step_profile(self, control_inputs):
        """One tick with CUDA events around each kernel -> (dynamics_ms, raymarch_ms, finalize_ms).  ValueError with obstacles
        set."""
        self._no_obstacles('step_profile')
        self._no_lidar_mask('step_profile')
        self._no_episodes('step_profile')
        a = self._actions_tensor(control_inputs)
        ms = (C.c_float * 3)()
        nat.check(nat.lib().f110_step_profile_ex(C.byref(self.c), C.byref(self._map_struct), C.byref(self._march_tables),
                                                 C.byref(self.beams.c), nat.ptr(a), ms, _stream_ptr(self.device)))
        return float(ms[0]), float(ms[1]), float(ms[2])

    def lookups(self):
        return int(self.lookup_counter.item()) if self.lookup_counter is not None else None
