"""Goldens off the default configuration, from the UNMODIFIED reference (numba path, scan noise off).

Run in the build container only (needs the reference tree):   python tests/golden/make_golden_configs.py

kat_configs.npz   laser_models.ScanSimulator2D(B, fov, eps=, theta_dis=, max_range=).scan(pose, None) on example_map
                  (0.0625 m, cell units on the device) and berlin (0.05 m, metre units), one configuration per row of
                  CONFIGS: theta_dis 1000 / 4000 / 32767, max_range 5 / 40, eps 0.01, fov 0.1 / pi / 6.28 / 7.0, B 2 / 3 / 33
                  / 100 / 8224, and one row that changes several knobs at once.  160 poses per map (free space, anywhere on the
                  map, hugging the border, far outside, two absurd coordinates); the 8224-beam row scans the first 16.
                  Arrays: configs (K, 5) = (B, fov, eps, theta_dis, max_range); names (K,); poses_<map> (160, 3);
                  scan_<k>_<map> (M, B) fp64; meta (what the script ran on).
env_ego1.npz      the real F110Env(ego_idx=1) with two cars, each driven by the example's PurePursuitPlanner, recorded every
                  tick as env_race2.npz is (prefix ego_crash_ / opp_crash_).  ego_crash: from tick 150 the ego (agent 1)
                  drives straight on at the planner's speed until it hits a wall, which ends the episode.  opp_crash: the same
                  for agent 0, whose collision does not end the episode; 700 ticks are recorded.  Both check `done` and the lap
                  frame of a non-zero ego.

The committed fixtures were made with the versions `meta` lists.  The scans are plain fp64 arithmetic and libm sin / cos
through numba; re-running on the same stack gives the same arrays.
"""
import os
import platform
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
from oracle import ref_import  # noqa: E402

ns = ref_import.load()
lm = ns.laser_models

#          B     fov        eps     theta_dis  max_range
CONFIGS = [(100, 4.7, 0.0001, 1000, 30.0),
           (100, 4.7, 0.0001, 4000, 30.0),
           (100, 4.7, 0.0001, 32767, 30.0),
           (100, 4.7, 0.0001, 2000, 5.0),
           (100, 4.7, 0.0001, 2000, 40.0),
           (100, 4.7, 0.01, 2000, 30.0),
           (33, 0.1, 0.0001, 2000, 30.0),
           (33, np.pi, 0.0001, 2000, 30.0),
           (33, 6.28, 0.0001, 2000, 30.0),
           (33, 7.0, 0.0001, 2000, 30.0),
           (2, 4.7, 0.0001, 2000, 30.0),
           (3, 4.7, 0.0001, 2000, 30.0),
           (33, 4.7, 0.0001, 2000, 30.0),
           (8224, 4.7, 0.0001, 2000, 30.0),
           (33, np.pi, 0.01, 4000, 40.0)]
NAMES = ['td1000', 'td4000', 'td32767', 'mr5', 'mr40', 'eps0.01', 'fov0.1', 'fovpi', 'fov6.28', 'fov7', 'b2', 'b3', 'b33',
         'b8224', 'mixed']
MAPS = (('example_map', ns.example_map), ('berlin', os.path.join(ns.maps_dir, 'berlin.yaml')))
WP = np.loadtxt(ns.example_waypoints, delimiter=';', skiprows=3)


def meta():
    import numba
    import scipy
    return 'python %s, numpy %s, numba %s, scipy %s, %s %s' % (platform.python_version(), np.__version__, numba.__version__,
                                                              scipy.__version__, platform.machine(), platform.processor())


def poses_for(s, rng):
    H, W = s.dt.shape
    res, ox, oy = s.map_resolution, s.orig_x, s.orig_y
    out = []
    free = np.argwhere(s.dt > 0.3)
    for r, c in free[rng.choice(free.shape[0], 96, replace=False)]:      # free space
        out.append([c * res + ox + rng.uniform(0, res), r * res + oy + rng.uniform(0, res), rng.uniform(-7, 7)])
    for _ in range(32):                                                  # anywhere, also inside walls
        out.append([ox + rng.uniform(0, W * res), oy + rng.uniform(0, H * res), rng.uniform(0, 2 * np.pi)])
    for k in range(16):                                                  # hugging the border, inside and outside
        t, d, side = rng.uniform(0, 1), rng.uniform(-3, 3) * res, k % 4
        x = ox + (t * W * res if side < 2 else (d if side == 2 else W * res + d))
        y = oy + ((d if side == 0 else H * res + d) if side < 2 else t * H * res)
        out.append([x, y, rng.uniform(0, 2 * np.pi)])
    for _ in range(14):                                                  # far outside
        out.append([ox + rng.uniform(-200, 200 + W * res), oy + rng.uniform(-200, 200 + H * res), rng.uniform(0, 2 * np.pi)])
    out.append([3.0e8, -1.0, 0.5])                                       # absurd coordinates
    out.append([-2.0, -4.0e9, 2.5])
    return np.array(out)


def kat_configs():
    rng = np.random.default_rng(20261016)
    out = {'configs': np.array(CONFIGS, dtype=np.float64), 'names': np.array(NAMES), 'meta': np.array(meta())}
    for name, yaml in MAPS:
        s0 = lm.ScanSimulator2D(2, 4.7)
        s0.set_map(yaml, '.png')
        poses = poses_for(s0, rng)
        out['poses_' + name] = poses
        for k, (B, fov, eps, td, mr) in enumerate(CONFIGS):
            s = lm.ScanSimulator2D(B, fov, eps=eps, theta_dis=td, max_range=mr)
            s.set_map(yaml, '.png')
            ps = poses[:16] if B > 1080 else poses
            out['scan_%d_%s' % (k, name)] = np.stack([s.scan(p, None) for p in ps])
    path = os.path.join(HERE, 'kat_configs.npz')
    np.savez_compressed(path, **out)
    print('%-28s %8.1f KB  (%s)' % ('kat_configs.npz', os.path.getsize(path) / 1024, out['meta']))


# ----------------------------------------------------------------------------- F110Env with ego_idx = 1
def wp_pose(k):
    k = k % WP.shape[0]
    return np.array([WP[k, 1], WP[k, 2], WP[k, 3] + np.pi / 2])


def _f110_env_module():
    """f110_env with gym / pyglet stubbed (as make_golden._run_real_env)."""
    gym = types.ModuleType('gym')
    gym.Env = object
    for sub in ('error', 'spaces', 'utils'):
        setattr(gym, sub, types.ModuleType('gym.' + sub)); sys.modules['gym.' + sub] = getattr(gym, sub)
    seeding = types.ModuleType('gym.utils.seeding'); gym.utils.seeding = seeding
    sys.modules['gym.utils.seeding'] = seeding
    envs = types.ModuleType('gym.envs'); reg = types.ModuleType('gym.envs.registration')
    reg.register = lambda **k: None; envs.registration = reg; gym.envs = envs
    sys.modules.update({'gym': gym, 'gym.envs': envs, 'gym.envs.registration': reg})
    pyglet = types.ModuleType('pyglet'); pyglet.options = {}
    gl = types.ModuleType('pyglet.gl'); gl.GL_POINTS = 0; pyglet.gl = gl
    sys.modules.update({'pyglet': pyglet, 'pyglet.gl': gl})
    from f110_gym.envs import f110_env
    return f110_env


def _run_ego1(crasher, max_ticks):
    """Two pure-pursuit cars in F110Env(ego_idx=1); from tick 150 agent `crasher` keeps steering 0 (straight on into a wall)."""
    f110_env = _f110_env_module()
    ex = os.path.join(ref_import.REF_ROOT, 'examples')
    if ex not in sys.path:
        sys.path.insert(0, ex)
    import waypoint_follow as wf
    from argparse import Namespace
    import yaml
    cwd = os.getcwd()
    os.chdir(ex)
    try:
        with open('config_example_map.yaml') as f:
            conf = Namespace(**yaml.safe_load(f))
        ns.RaceCar.scan_simulator = None
        A = 2
        env = f110_env.F110Env(map=conf.map_path, map_ext=conf.map_ext, num_agents=A, timestep=0.01,
                               integrator=ns.Integrator.RK4, ego_idx=1)
        planner = wf.PurePursuitPlanner(conf, 0.17145 + 0.15875)
        gains = [(0.82461887897713965, 1.1), (0.82461887897713965, 1.375)]
        pose0 = np.stack([wp_pose(0), wp_pose(60)])
        orig_reset = env.sim.reset

        def reset_noise_off(p):
            orig_reset(p)
            for a in env.sim.agents:
                a.scan_rng = None
        env.sim.reset = reset_noise_off
        obs, rew, done, info = env.reset(pose0)
        rec = dict(actions=[], states=[], lap_times=[], lap_counts=[], done=[], toggles=[], collisions=[])

        def record(act, done):
            rec['actions'].append(act)
            rec['states'].append(np.array([a.state.copy() for a in env.sim.agents]))
            rec['lap_times'].append(env.lap_times.copy()); rec['lap_counts'].append(env.lap_counts.copy())
            rec['done'].append(done); rec['toggles'].append(env.toggle_list.copy())
            rec['collisions'].append(obs['collisions'].copy())
        record(np.zeros((A, 2)), done)
        while not done and len(rec['done']) < max_ticks:
            t = len(rec['done'])
            act = np.zeros((A, 2))
            for i in range(A):
                speed, steer = planner.plan(obs['poses_x'][i], obs['poses_y'][i], obs['poses_theta'][i], gains[i][0], gains[i][1])
                act[i] = [0.0 if (i == crasher and t >= 150) else steer, speed]
            obs, rew, done, info = env.step(act)
            record(act, done)
    finally:
        os.chdir(cwd)
    out = {k: np.array(v) for k, v in rec.items()}
    out['pose0'] = pose0
    print('ego_idx 1, agent %d crashes: ticks %d done %s collisions %s toggles %s' % (
        crasher, len(rec['done']), rec['done'][-1], rec['collisions'][-1], rec['toggles'][-1]))
    return out


def env_ego1():
    out = {}
    for prefix, crasher, max_ticks in (('ego_crash_', 1, 3000), ('opp_crash_', 0, 700)):
        out.update({prefix + k: v for k, v in _run_ego1(crasher, max_ticks).items()})
    out['meta'] = np.array(meta())
    path = os.path.join(HERE, 'env_ego1.npz')
    np.savez_compressed(path, **out)
    print('%-28s %8.1f KB' % ('env_ego1.npz', os.path.getsize(path) / 1024))


if __name__ == '__main__':
    groups = {'kat_configs': kat_configs, 'env_ego1': env_ego1}
    for name in (sys.argv[1:] or list(groups)):          # python make_golden_configs.py [group ...]
        groups[name]()
