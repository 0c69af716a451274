"""Batched CUDA versions of the reference's @njit kernels, same names and argument meaning, operating on
torch CUDA tensors with a leading batch dimension M.  Thin wrappers over the C ABI standalone entry
points (include/f110_b200.h); used by the unit-parity tests and usable on their own.

    reference function                       file:line                         here
    vehicle_dynamics_st(x, u, *16 params)    dynamic_models.py:123-176         vehicle_dynamics_st(x[M,7], u[M,2], params)
    pid(speed, steer, cur_speed, cur_steer..) dynamic_models.py:178-221        pid(inputs[M,4], params) -> (accl[M], sv[M])
    get_vertices(pose, length, width)        collision_models.py:237-260       get_vertices(poses[M,3], length, width)
    collision(v1, v2)                        collision_models.py:113-182       collision(va[M,4,2], vb[M,4,2])
    collision_multiple(vertices)             collision_models.py:184-212       collision_multiple(verts[M,n,4,2])
    check_ttc_jit(scan, vel, ...)            laser_models.py:188-217           check_ttc(scans[M,B], vel[M], beams)
    ray_cast(pose, scan, scan_angles, verts) laser_models.py:318-346           ray_cast(poses[M,3], scans[M,B], opp[M,4,2], beams)
    ScanSimulator2D(num_beams, fov).scan     laser_models.py:348-457           ScanSimulator2D(...).scan(poses[M,3])
"""
import ctypes as C

import numpy as np
import torch

from . import _native as nat
from . import maps as hostmaps
from .simulator import DeviceBeams, DeviceMap, _stream_ptr, check_theta_dis


def _dev(t, dtype=torch.float64, device=None):
    if not torch.is_tensor(t):
        t = torch.as_tensor(np.asarray(t))
    if device is None:
        device = t.device if t.is_cuda else torch.device('cuda', torch.cuda.current_device())
    return t.to(device=device, dtype=dtype).contiguous()


def _params_dev(params, device):
    if isinstance(params, dict):
        params = hostmaps.params_vector(params)
    return _dev(params, device=device)


def vehicle_dynamics_st(x, u, params):
    x = _dev(x).reshape(-1, 7)
    u = _dev(u, device=x.device).reshape(-1, 2)
    p = _params_dev(params, x.device)
    f = torch.empty_like(x)
    nat.check(nat.lib().f110_vehicle_dynamics_st(nat.ptr(x), nat.ptr(u), nat.ptr(p), x.shape[0], nat.ptr(f),
                                                 _stream_ptr(x.device)))
    return f


def vehicle_dynamics_ks(x, u, params):
    """dynamic_models.py:90-121: x[M,5] = (x, y, steer, v, yaw), u[M,2] -> f[M,5]."""
    x = _dev(x).reshape(-1, 5)
    u = _dev(u, device=x.device).reshape(-1, 2)
    p = _params_dev(params, x.device)
    f = torch.empty_like(x)
    nat.check(nat.lib().f110_vehicle_dynamics_ks(nat.ptr(x), nat.ptr(u), nat.ptr(p), x.shape[0], nat.ptr(f),
                                                 _stream_ptr(x.device)))
    return f


def pid(inputs, params):
    """inputs[M,4] = (speed, steer, current_speed, current_steer) -> (accl[M], sv[M])."""
    x = _dev(inputs).reshape(-1, 4)
    p = _params_dev(params, x.device)
    out = torch.empty((x.shape[0], 2), dtype=torch.float64, device=x.device)
    nat.check(nat.lib().f110_pid(nat.ptr(x), nat.ptr(p), x.shape[0], nat.ptr(out), _stream_ptr(x.device)))
    return out[:, 0], out[:, 1]


def get_vertices(poses, length, width):
    p = _dev(poses).reshape(-1, 3)
    out = torch.empty((p.shape[0], 4, 2), dtype=torch.float64, device=p.device)
    nat.check(nat.lib().f110_get_vertices(nat.ptr(p), float(length), float(width), p.shape[0], nat.ptr(out),
                                          _stream_ptr(p.device)))
    return out


def collision(va, vb):
    va = _dev(va).reshape(-1, 4, 2)
    vb = _dev(vb, device=va.device).reshape(-1, 4, 2)
    out = torch.empty((va.shape[0],), dtype=torch.int32, device=va.device)
    nat.check(nat.lib().f110_collision(nat.ptr(va), nat.ptr(vb), va.shape[0], nat.ptr(out), _stream_ptr(va.device)))
    return out.bool()


def collision_multiple(vertices):
    v = _dev(vertices)
    if v.dim() == 3:
        v = v.unsqueeze(0)
    M, n = v.shape[0], v.shape[1]
    col = torch.empty((M, n), dtype=torch.float64, device=v.device)
    idx = torch.empty((M, n), dtype=torch.float64, device=v.device)
    nat.check(nat.lib().f110_collision_multiple(nat.ptr(v), M, n, nat.ptr(col), nat.ptr(idx), _stream_ptr(v.device)))
    return col, idx


def check_ttc(scans, vel, beams, ttc_thresh=0.005):
    s = _dev(scans).reshape(-1, beams.num_beams)
    v = _dev(vel, device=s.device).reshape(-1)
    out = torch.empty((s.shape[0],), dtype=torch.int32, device=s.device)
    nat.check(nat.lib().f110_check_ttc(C.byref(beams.c), nat.ptr(s), nat.ptr(v), float(ttc_thresh), s.shape[0],
                                       nat.ptr(out), _stream_ptr(s.device)))
    return out.bool()


def ray_cast(poses, scans, opp_vertices, beams, return_window=False):
    """Returns the modified fp32 scans (a copy), optionally with the (min_ind, max_ind) windows."""
    p = _dev(poses).reshape(-1, 3)
    s = _dev(scans, dtype=torch.float32, device=p.device).reshape(-1, beams.num_beams).clone()
    v = _dev(opp_vertices, device=p.device).reshape(-1, 4, 2)
    win = torch.empty((p.shape[0], 2), dtype=torch.int32, device=p.device)
    nat.check(nat.lib().f110_ray_cast(C.byref(beams.c), nat.ptr(p), nat.ptr(v), p.shape[0], nat.ptr(s), nat.ptr(win),
                                      _stream_ptr(p.device)))
    return (s, win) if return_window else s


# most beams one f110_scan_layers call writes (M * num_beams < 2^32: the kernel's 32-bit indices); scan(layer_ids=...) splits
# a larger batch into calls of at most this many beams
SCAN_LAYERS_MAX_ELEMENTS = (1 << 32) - 1


class ScanSimulator2D(object):
    """laser_models.py:348-457.  scan() takes one pose (3,) or a batch (M,3) and returns fp32 ranges
    (M,B) on the device; `rng`/`std_dev` follow the reference: rng=None disables the noise, otherwise
    rng is an integer seed for the device Philox stream (statistical parity with numpy's Generator)."""

    def __init__(self, num_beams, fov, eps=0.0001, theta_dis=2000, max_range=30.0, device=None):
        nat.lib()
        self.num_beams, self.fov, self.eps, self.theta_dis, self.max_range = num_beams, fov, eps, theta_dis, max_range
        self.angle_increment = fov / (num_beams - 1)
        self.theta_index_increment = theta_dis * self.angle_increment / (2. * np.pi)
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        self.beams = DeviceBeams(num_beams, fov, hostmaps.DEFAULT_PARAMS, self.device, theta_dis)
        self.map = None
        self.map_height = None
        self._noise_offset = 0      # running element offset into the Philox stream: ranges never overlap across calls

    def set_map(self, map_path, map_ext):
        self.map = DeviceMap.from_yaml(map_path, map_ext, self.device, theta_dis=self.theta_dis, eps=self.eps,
                                       max_range=self.max_range)
        self.map_height, self.map_width = self.map.host.height, self.map.host.width
        self.map_resolution = self.map.host.resolution
        return True

    def set_device_map(self, device_map):
        """A DeviceMap built elsewhere (device EDT, generated track) instead of a yaml + image on disk.  ValueError for a map
        built with another theta_dis than this scan simulator's (its beam tables would step through the wrong LUT)."""
        check_theta_dis(device_map, self.theta_dis, 'ScanSimulator2D')
        self.map = device_map
        self.map_height, self.map_width = device_map.host.height, device_map.host.width
        self.map_resolution = device_map.host.resolution
        return True

    def scan(self, pose, rng=None, std_dev=0.01, out_f64=False, count_lookups=False, layer_ids=None):
        """layer_ids=None: f110_scan on the map (one map; layer 0 of a same-size stack; a canvas stack raises F110Error).
        layer_ids an int or (M,) ints: f110_scan_layers, pose k on layer layer_ids[k] of the map (any map the Simulator
        accepts, e.g. set_device_map(sim.map) and layer_ids=sim.env_layer[env_ids]); ValueError for a wrong length or an id
        outside [0, num_layers)."""
        if self.map_height is None:
            raise ValueError('Map is not set for scan simulator.')
        p = _dev(pose, device=self.device).reshape(-1, 3)
        M = p.shape[0]
        o32 = torch.empty((M, self.num_beams), dtype=torch.float32, device=self.device) if not out_f64 else None
        o64 = torch.empty((M, self.num_beams), dtype=torch.float64, device=self.device) if out_f64 else None
        cnt = torch.zeros((1,), dtype=torch.int64, device=self.device) if count_lookups else None
        L = nat.lib()
        if layer_ids is None:
            nat.check(L.f110_scan(C.byref(self.map.c), C.byref(self.beams.c), nat.ptr(p), M, nat.ptr(o32), nat.ptr(o64),
                                  nat.ptr(cnt), _stream_ptr(self.device)))
        else:
            ids = self._layer_ids(layer_ids, M)
            step = max(1, min(SCAN_LAYERS_MAX_ELEMENTS // self.num_beams, 0x7fffffff))
            for k in range(0, M, step):
                m = min(step, M - k)
                nat.check(L.f110_scan_layers(C.byref(self.map.c), C.byref(self.beams.c), nat.ptr(p[k:k + m]),
                                             nat.ptr(ids[k:k + m]), m, nat.ptr(None if o32 is None else o32[k:k + m]),
                                             nat.ptr(None if o64 is None else o64[k:k + m]), nat.ptr(cnt),
                                             _stream_ptr(self.device)))
        out = o64 if out_f64 else o32
        if rng is not None:
            if out_f64:
                raise ValueError('noise is only applied to the fp32 output')
            nat.check(L.f110_scan_noise(nat.ptr(out), out.numel(), float(std_dev), int(rng) & 0xFFFFFFFFFFFFFFFF,
                                        self._noise_offset, _stream_ptr(self.device)))
            self._noise_offset += out.numel()
        return (out, int(cnt.item())) if count_lookups else out

    def _layer_ids(self, layer_ids, M):
        """layer_ids (int, or M ints) -> contiguous int32 device tensor [M], checked against the map's layer count."""
        layers = max(1, int(self.map.c.num_layers))
        ids = torch.as_tensor(layer_ids) if torch.is_tensor(layer_ids) else torch.as_tensor(np.asarray(layer_ids))
        if ids.dim() == 0:
            ids = ids.reshape(1).expand(M)
        if ids.dim() != 1 or ids.shape[0] != M:
            raise ValueError('layer_ids must be one int or one per pose (%d), got shape %s' % (M, tuple(ids.shape)))
        if ids.dtype.is_floating_point or ids.dtype == torch.bool or ids.is_complex():
            raise ValueError('layer_ids must be integers')
        lo, hi = int(ids.min()), int(ids.max())
        if lo < 0 or hi >= layers:
            raise ValueError('layer_ids must lie in [0, %d), got [%d, %d]' % (layers, lo, hi))
        return ids.to(device=self.device, dtype=torch.int32).contiguous()

    def get_increment(self):
        return self.angle_increment
