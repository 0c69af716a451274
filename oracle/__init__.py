"""ctypes front-end of the CPU parity oracle (oracle/f110_oracle.c).

TEST INFRASTRUCTURE ONLY — see the header of f110_oracle.c.  Imported by tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs; never by the
product package f1tenth_gym_b200.

Host-side table construction below restates the reference's load-time code with numpy
(same third-party calls the reference makes: PIL, yaml, scipy.ndimage.distance_transform_edt):
  load_map      <- laser_models.py:383-427 (ScanSimulator2D.set_map) + :40-53 (get_dt)
  angle_lut     <- laser_models.py:379-381
  beam_tables   <- base_classes.py:122-158 (RaceCar.__init__)
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

PARAM_KEYS = ['mu', 'C_Sf', 'C_Sr', 'lf', 'lr', 'h', 'm', 'I', 's_min', 's_max', 'sv_min', 'sv_max',
              'v_switch', 'a_max', 'v_min', 'v_max', 'width', 'length']
DEFAULT_PARAMS = {'mu': 1.0489, 'C_Sf': 4.718, 'C_Sr': 5.4562, 'lf': 0.15875, 'lr': 0.17145, 'h': 0.074,
                  'm': 3.74, 'I': 0.04712, 's_min': -0.4189, 's_max': 0.4189, 'sv_min': -3.2,
                  'sv_max': 3.2, 'v_switch': 7.319, 'a_max': 9.51, 'v_min': -5.0, 'v_max': 20.0,
                  'width': 0.31, 'length': 0.58}   # f110_env.py:130

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)


class _Map(C.Structure):
    _fields_ = [('height', C.c_int32), ('width', C.c_int32), ('resolution', C.c_double),
                ('orig_x', C.c_double), ('orig_y', C.c_double), ('orig_c', C.c_double),
                ('orig_s', C.c_double), ('dt', _dp), ('theta_dis', C.c_int32), ('sines', _dp),
                ('cosines', _dp), ('eps', C.c_double), ('max_range', C.c_double)]


def build(force=False):
    so = os.path.join(_HERE, 'libf110_oracle.so')
    src = os.path.join(_HERE, 'f110_oracle.c')
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(['make', '-C', _HERE, '-s', '-B'])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.orc_vehicle_dynamics_ks.argtypes = [_dp, _dp, _dp, _dp]
        L.orc_vehicle_dynamics_st.argtypes = [_dp, _dp, _dp, _dp]
        L.orc_pid.argtypes = [C.c_double] * 8 + [_dp]
        L.orc_get_scan.argtypes = [C.POINTER(_Map), _dp, C.c_int, C.c_double, C.c_double, _dp,
                                   C.POINTER(C.c_int64)]
        L.orc_check_ttc.argtypes = [_dp, C.c_int, C.c_double, _dp, _dp, C.c_double]
        L.orc_check_ttc.restype = C.c_int
        L.orc_blocked_view_indices.argtypes = [_dp, _dp, _dp, C.c_int, _ip, _ip]
        L.orc_ray_cast.argtypes = [_dp, _dp, _dp, C.c_int, _dp]
        L.orc_get_vertices.argtypes = [_dp, C.c_double, C.c_double, _dp]
        L.orc_collision.argtypes = [_dp, _dp]
        L.orc_collision.restype = C.c_int
        L.orc_collision_multiple.argtypes = [_dp, C.c_int, _dp, _dp]
        L.orc_sim_create.restype = C.c_void_p
        L.orc_sim_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double,
                                     C.c_double, C.POINTER(_Map), _dp, _dp, _dp, _dp]
        L.orc_sim_destroy.argtypes = [C.c_void_p]
        L.orc_sim_set_ego.argtypes = [C.c_void_p, C.c_int]
        L.orc_sim_set_ego.restype = C.c_int
        for name in ('state', 'scans', 'collisions', 'collision_idx', 'lap_times', 'lap_counts',
                     'toggle_list', 'params', 'steer_buf'):
            f = getattr(L, 'orc_sim_' + name)
            f.restype = _dp
            f.argtypes = [C.c_void_p]
        for name in ('in_collision', 'steer_cnt'):
            f = getattr(L, 'orc_sim_' + name)
            f.restype = _ip
            f.argtypes = [C.c_void_p]
        L.orc_sim_nlook.restype = C.c_int64
        L.orc_sim_nlook.argtypes = [C.c_void_p]
        L.orc_sim_current_time.restype = C.c_double
        L.orc_sim_current_time.argtypes = [C.c_void_p]
        L.orc_sim_reset.argtypes = [C.c_void_p, _dp]
        L.orc_sim_step.argtypes = [C.c_void_p, _dp]
        L.orc_env_post_step.argtypes = [C.c_void_p]
        L.orc_env_post_step.restype = C.c_int
        L.orc_env_reset.argtypes = [C.c_void_p, _dp]
        L.orc_env_reset.restype = C.c_int
        L.orc_rollout.restype = C.c_int64
        L.orc_rollout.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, _dp, C.c_int, C.c_int,
                                  C.c_uint64, C.c_int, C.POINTER(C.c_int64)]
        L.orc_sim_scans_pre.restype = _dp
        L.orc_sim_scans_pre.argtypes = [C.c_void_p]
        L.orc_env_restart.argtypes = [C.c_void_p, _dp]
        L.orc_step_batch.argtypes = [C.POINTER(C.c_void_p), C.c_int, _dp, _dp, C.c_int, C.c_int]
        L.orc_gather.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, _dp]
        L.orc_pure_pursuit.argtypes = [_dp, _dp, _dp, C.c_int] + [C.c_double] * 7 + [_dp]
        L.orc_num_cores.restype = C.c_int
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(_dp)


def _f64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64))


# ----------------------------------------------------------------------------- host tables

def angle_lut(theta_dis=2000):
    theta_arr = np.linspace(0.0, 2 * np.pi, num=theta_dis)
    return np.sin(theta_arr), np.cos(theta_arr)


def params_vector(params):
    return np.array([float(params[k]) for k in PARAM_KEYS], dtype=np.float64)


def beam_tables(num_beams, fov, params):
    """scan_angles, cosines, side_distances exactly as RaceCar.__init__ builds them."""
    inc = fov / (num_beams - 1)
    dist_sides = params['width'] / 2.
    dist_fr = (params['lf'] + params['lr']) / 2.
    scan_angles = np.zeros((num_beams,))
    cosines = np.zeros((num_beams,))
    side = np.zeros((num_beams,))
    for i in range(num_beams):
        angle = -fov / 2. + i * inc
        scan_angles[i] = angle
        cosines[i] = np.cos(angle)
        if angle > 0:
            if angle < np.pi / 2:
                side[i] = min(dist_sides / np.sin(angle), dist_fr / np.cos(angle))
            else:
                side[i] = min(dist_sides / np.cos(angle - np.pi / 2.), dist_fr / np.sin(angle - np.pi / 2.))
        else:
            if angle > -np.pi / 2:
                side[i] = min(dist_sides / np.sin(-angle), dist_fr / np.cos(-angle))
            else:
                side[i] = min(dist_sides / np.cos(-angle - np.pi / 2), dist_fr / np.sin(-angle - np.pi / 2))
    return scan_angles, cosines, side


class OracleMap(object):
    """Distance-transform map + LUTs, the state ScanSimulator2D holds (laser_models.py:348-427)."""

    def __init__(self, dt, resolution, origin, theta_dis=2000, eps=0.0001, max_range=30.0):
        self.dt = _f64(dt)
        self.height, self.width = self.dt.shape
        self.resolution = float(resolution)
        self.orig_x, self.orig_y = float(origin[0]), float(origin[1])
        self.orig_s, self.orig_c = float(np.sin(origin[2])), float(np.cos(origin[2]))
        self.theta_dis = theta_dis
        self.sines, self.cosines = angle_lut(theta_dis)
        self.eps, self.max_range = eps, max_range
        self.c = _Map(self.height, self.width, self.resolution, self.orig_x, self.orig_y, self.orig_c,
                      self.orig_s, _p(self.dt), theta_dis, _p(self.sines), _p(self.cosines), eps,
                      max_range)

    @classmethod
    def from_yaml(cls, map_path, map_ext, **kw):
        import yaml
        from PIL import Image
        from scipy.ndimage import distance_transform_edt as edt
        img_path = os.path.splitext(map_path)[0] + map_ext
        img = np.array(Image.open(img_path).transpose(Image.FLIP_TOP_BOTTOM)).astype(np.float64)
        img[img <= 128.] = 0.
        img[img > 128.] = 255.
        with open(map_path, 'r') as f:
            meta = yaml.safe_load(f)
        res = meta['resolution']
        return cls(res * edt(img), res, meta['origin'], **kw)


def theta_index_increment(num_beams, fov, theta_dis=2000):
    angle_increment = fov / (num_beams - 1)
    return theta_dis * angle_increment / (2. * np.pi)


# ----------------------------------------------------------------------------- functional ops

def vehicle_dynamics_st(x, u, pvec):
    x, u, pvec = _f64(x), _f64(u), _f64(pvec)
    f = np.empty(7)
    lib().orc_vehicle_dynamics_st(_p(x), _p(u), _p(pvec), _p(f))
    return f


def vehicle_dynamics_ks(x, u, pvec):
    x, u, pvec = _f64(x), _f64(u), _f64(pvec)
    f = np.empty(5)
    lib().orc_vehicle_dynamics_ks(_p(x), _p(u), _p(pvec), _p(f))
    return f


def pid(speed, steer, current_speed, current_steer, max_sv, max_a, max_v, min_v):
    out = np.empty(2)
    lib().orc_pid(speed, steer, current_speed, current_steer, max_sv, max_a, max_v, min_v, _p(out))
    return out[0], out[1]


def get_scan(omap, pose, num_beams=1080, fov=4.7, count=False):
    pose = _f64(pose)
    scan = np.empty(num_beams)
    n = C.c_int64(0)
    lib().orc_get_scan(C.byref(omap.c), _p(pose), num_beams, fov,
                       theta_index_increment(num_beams, fov, omap.theta_dis), _p(scan), C.byref(n))
    return (scan, n.value) if count else scan


def check_ttc(scan, vel, cosines, side_distances, ttc_thresh=0.005):
    scan, cosines, side_distances = _f64(scan), _f64(cosines), _f64(side_distances)
    return bool(lib().orc_check_ttc(_p(scan), scan.shape[0], vel, _p(cosines), _p(side_distances),
                                    ttc_thresh))


def ray_cast(pose, scan, scan_angles, vertices):
    pose, scan_angles, vertices = _f64(pose), _f64(scan_angles), _f64(vertices)
    scan = _f64(scan).copy()
    lib().orc_ray_cast(_p(pose), _p(scan), _p(scan_angles), scan.shape[0], _p(vertices))
    return scan


def blocked_view_indices(pose, vertices, scan_angles):
    pose, scan_angles, vertices = _f64(pose), _f64(scan_angles), _f64(vertices)
    lo, hi = C.c_int32(0), C.c_int32(0)
    lib().orc_blocked_view_indices(_p(pose), _p(vertices), _p(scan_angles), scan_angles.shape[0],
                                   C.byref(lo), C.byref(hi))
    return lo.value, hi.value


def get_vertices(pose, length, width):
    pose = _f64(pose)
    v = np.empty((4, 2))
    lib().orc_get_vertices(_p(pose), length, width, _p(v))
    return v


def collision(v1, v2):
    v1, v2 = _f64(v1), _f64(v2)
    return bool(lib().orc_collision(_p(v1), _p(v2)))


def collision_multiple(vertices):
    vertices = _f64(vertices)
    n = vertices.shape[0]
    col, idx = np.empty(n), np.empty(n)
    lib().orc_collision_multiple(_p(vertices), n, _p(col), _p(idx))
    return col, idx


# ----------------------------------------------------------------------------- Simulator

class OracleSim(object):
    """One environment: base_classes.Simulator semantics (+ F110Env lap logic)."""

    def __init__(self, omap, params=None, num_agents=2, num_beams=1080, fov=4.7, timestep=0.01,
                 integrator=1, lidar_dist=0.0, ego_idx=0):
        """ego_idx: F110Env's ego (f110_env.py:145): its collision sets `done`, its start yaw the lap frame."""
        params = dict(DEFAULT_PARAMS) if params is None else params
        if not 0 <= ego_idx < num_agents:
            raise ValueError('ego_idx %r outside [0, %d)' % (ego_idx, num_agents))
        self.omap = omap
        self.num_agents, self.num_beams = num_agents, num_beams
        self.ego_idx = ego_idx
        self._tabs = beam_tables(num_beams, fov, params)
        pv = np.tile(params_vector(params), (num_agents, 1))
        self._h = lib().orc_sim_create(num_agents, num_beams, integrator, timestep, fov,
                                       theta_index_increment(num_beams, fov, omap.theta_dis),
                                       lidar_dist, C.byref(omap.c), _p(self._tabs[0]),
                                       _p(self._tabs[1]), _p(self._tabs[2]), _p(pv))
        if lib().orc_sim_set_ego(self._h, ego_idx) != 0:
            raise ValueError('orc_sim_set_ego refused ego_idx %r' % ego_idx)
        A, B = num_agents, num_beams
        L = lib()
        h = self._h
        self.state = np.ctypeslib.as_array(L.orc_sim_state(h), (A, 7))
        self.scans = np.ctypeslib.as_array(L.orc_sim_scans(h), (A, B))
        self.collisions = np.ctypeslib.as_array(L.orc_sim_collisions(h), (A,))
        self.collision_idx = np.ctypeslib.as_array(L.orc_sim_collision_idx(h), (A,))
        self.lap_times = np.ctypeslib.as_array(L.orc_sim_lap_times(h), (A,))
        self.lap_counts = np.ctypeslib.as_array(L.orc_sim_lap_counts(h), (A,))
        self.toggle_list = np.ctypeslib.as_array(L.orc_sim_toggle_list(h), (A,))
        self.params = np.ctypeslib.as_array(L.orc_sim_params(h), (A, 18))
        self.in_collision = np.ctypeslib.as_array(L.orc_sim_in_collision(h), (A,))
        self.steer_cnt = np.ctypeslib.as_array(L.orc_sim_steer_cnt(h), (A,))
        self.steer_buf = np.ctypeslib.as_array(L.orc_sim_steer_buf(h), (A, 2))
        self.scans_pre = np.ctypeslib.as_array(L.orc_sim_scans_pre(h), (A, B))

    def __del__(self):
        try:
            lib().orc_sim_destroy(self._h)
        except Exception:
            pass

    @property
    def nlook(self):
        return lib().orc_sim_nlook(self._h)

    @property
    def current_time(self):
        return lib().orc_sim_current_time(self._h)

    def reset(self, poses):
        poses = _f64(poses)
        if poses.shape[0] != self.num_agents:
            raise ValueError('Number of poses for reset does not match number of agents.')
        lib().orc_sim_reset(self._h, _p(poses))

    def step(self, control_inputs):
        a = _f64(control_inputs)
        assert a.shape == (self.num_agents, 2)
        lib().orc_sim_step(self._h, _p(a))

    def env_reset(self, poses):
        poses = _f64(poses)
        return bool(lib().orc_env_reset(self._h, _p(poses)))

    def env_post_step(self):
        return bool(lib().orc_env_post_step(self._h))

    def env_restart(self, poses):
        """The device auto-reset of this env (f110_autoreset): Simulator.reset + env counters and start frame, no
        zero-action step; `done` and the collision observation of the ending tick are kept."""
        poses = _f64(poses)
        assert poses.shape == (self.num_agents, 3)
        lib().orc_env_restart(self._h, _p(poses))


_FIELDS = {'state': 0, 'scans': 1, 'scans_pre': 2, 'collisions': 3, 'collision_idx': 4, 'in_collision': 5,
           'lap_times': 6, 'lap_counts': 7, 'toggle_list': 8, 'done': 9, 'current_time': 10, 'nlook': 11}


def _handles(sims):
    return (C.c_void_p * len(sims))(*[s._h for s in sims])


def step_batch(sims, actions, noise=None, env_level=False, num_threads=0):
    """One step of every OracleSim in `sims` (same num_agents / num_beams), spread over the host cores.
    actions (n, A, 2); noise (n, A, B) additive scan noise or None; env_level: also the F110Env lap logic and done
    (read back with gather(sims, 'done'))."""
    n = len(sims)
    A, B = sims[0].num_agents, sims[0].num_beams
    a = _f64(actions)
    assert a.shape == (n, A, 2)
    nz = None
    if noise is not None:
        nz = _f64(noise)
        assert nz.shape == (n, A, B)
    lib().orc_step_batch(_handles(sims), n, _p(a), None if nz is None else _p(nz), 1 if env_level else 0, num_threads)


def gather(sims, field):
    """One field of every sim as an array: (n, A, 7) state, (n, A, B) scans / scans_pre, (n,) done / current_time /
    nlook, (n, A) otherwise."""
    n = len(sims)
    A, B = sims[0].num_agents, sims[0].num_beams
    shape = {'state': (n, A, 7), 'scans': (n, A, B), 'scans_pre': (n, A, B), 'done': (n,), 'current_time': (n,),
             'nlook': (n,)}.get(field, (n, A))
    out = np.empty(shape)
    lib().orc_gather(_handles(sims), n, _FIELDS[field], _p(out))
    return out


def rollout(sims, ticks, start_poses, pose_gap=23, seed=12345, num_threads=0):
    """Benchmark-policy rollout over independent OracleSims (SURVEY.md 8d). Returns
    (agent_steps, dt_lookups)."""
    start_poses = _f64(start_poses)
    arr = (C.c_void_p * len(sims))(*[s._h for s in sims])
    n = C.c_int64(0)
    tot = lib().orc_rollout(arr, len(sims), ticks, _p(start_poses), start_poses.shape[0], pose_gap,
                            seed, num_threads, C.byref(n))
    return tot, n.value


def pure_pursuit(wx, wy, wv, pose, lookahead_distance, vgain, wheelbase, max_reacquire=20.0):
    """examples/waypoint_follow.py PurePursuitPlanner.plan -> (speed, steering_angle)."""
    wx, wy, wv = _f64(wx), _f64(wy), _f64(wv)
    out = np.empty(2)
    lib().orc_pure_pursuit(_p(wx), _p(wy), _p(wv), wx.shape[0], float(pose[0]), float(pose[1]), float(pose[2]),
                           lookahead_distance, vgain, wheelbase, max_reacquire, _p(out))
    return out[0], out[1]


def num_cores():
    return lib().orc_num_cores()
