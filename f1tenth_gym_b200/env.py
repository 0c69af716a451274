"""F110Env façade — the gym.Env-shaped surface of reference f110_env.py:53-418, batched.

    env = F110Env(map=..., map_ext='.png', num_agents=2, timestep=0.01, integrator=Integrator.RK4,
                  num_envs=4096)                       # num_envs is the batch extension
    obs, reward, done, info = env.reset(poses)         # poses (A,3) or (N,A,3); runs ONE zero-action tick
    obs, reward, done, info = env.step(action)         # action (N,A,2) = (steer, speed)

kwargs and defaults are the reference's (f110_env.py:104-159): seed=12345, map='vegas', map_ext='.png',
params=<18-key dict>, num_agents=2, timestep=0.01, ego_idx=0, integrator=RK4, lidar_dist=0.0.
Extensions: num_envs (None = single env, reference-shaped numpy/list outputs; int = batched torch
tensors (N,A,...) that are views of device buffers valid until the next step), num_beams, fov, device,
scan_noise_std (reference default 0.01; 0 disables the noise for bit-reproducible parity runs),
local_map={'size': (H, W), 'metres_per_pixel': s, 'forward_offset': f} (adds obs['local_map']: each agent's heading-up class
view of Simulator.render_views, (N, A, H, W) uint8 on the device in batched mode, numpy (A, H, W) for a single env).
render(mode='rgb_array') draws each env's ego on the device (world-aligned, the reference window's colours).
centerline=<(n, 2) table, or one per map of a list> (Simulator.set_centerlines) adds obs['track_s'], obs['track_d'],
obs['track_heading_error'] and obs['progress'] ((N, A) device tensors in batched mode, numpy (A,) for a single env), updated
after every step on the device; reward='progress' (needs centerline) returns the ego's progress along its centerline in that
step, (N,) on the device (a copy, still valid after the next step) or a float, instead of the reference's constant timestep.
An env reset since its last step restarts its progress at 0, so the step that resets an env earns 0.
action_repeat=K (default 1): step() holds the action for K ticks (Simulator.tick_repeat, one call).  done is then "done on any
of the K ticks" and info['done_tick'] the first such tick (-1: none); the reward is K * timestep, or with reward='progress' the
sum of the ego's K deltas; lap_times, lap_counts, the progress keys and the scans are the last tick's.  The only difference to
calling step() K times is which scans exist.  reset() still runs exactly one zero-action tick.
Batched mode also takes a list of maps, map=['berlin', 'vegas', ...] with map_ext one extension or a list, stacked into
one simulator (DeviceMap.stack: one resolution, unrotated origins); env e drives on map env_map_ids[e] (default e % L).
mixed_resolution=True also stacks maps of different resolutions (e.g. generated tracks with the bundled maps); every map
of such a batch is then marched in metres, the power-of-two ones included.  rotated_origins=True also stacks maps whose
yaml origin has a yaw (marched in metres in each map's rotated frame by k_march_lean_rot).
obstacles={'candidates': (C, 5) table or one per map, 'count': (lo, hi), 'clearance': m, 'seed': s} (batched mode only;
Simulator.set_obstacles / set_obstacle_draw with hi slots per env): static box obstacles, redrawn on the device for every env by
reset() after it places the agents and for the masked envs by reset_envs(); obs['obstacles'] (N, K, 5) and
obs['obstacle_active'] (N, K) are views of the device buffers, and local_map / rgb_array draw the boxes (class 5).
lidar=[True, False, ...] (batched mode only; Simulator.set_lidar): which agent slots have a lidar.  A sensorless agent (a
scripted opponent, a policy on state or local_map observations) is simulated as before, and its row of obs['scans'] is NaN.
Its scan is skipped only without scan noise (scan_noise_std=0.0): with the default 0.01 every scan is still computed.
autoreset={'poses': (K, 3) start table or one per map, 'max_episode_steps': T, 'seed': s, 'pose_gap': g} (batched mode only,
action_repeat 1; Simulator.set_episodes): step() ends the episode of every env that is done or has run T steps (None or 0: no
limit) and restarts it on the device as reset() would: a start pose drawn from the table, then one zero-action tick, whose
observation obs holds for that env.  done = terminated | truncated; info adds 'terminated', 'truncated', 'episode_length' and
'final_observation' (the ended episode's last observation: state keys, scans, collisions, lap_times, lap_counts).  All are
views of device buffers, overwritten by the next step.  local_map and the progress keys are those after the restart; with
reward='progress' a restarted env earns 0 on that step.  reset() and reset_envs() zero the episode counters.
autoreset={..., 'action_repeat': K} (Simulator.tick_repeat in episode mode) holds each action for K ticks, and an env's episode
stops at the first of them that ends it, as a frame-skip wrapper that stops at done would: its final_observation, flags and
done are that tick's, and it restarts after the call.  T counts step() calls (a time limit of T * K ticks); info also gets
'end_tick' (the tick 0..K-1 at which the episode ended, -1 = none) and episode_length is in step() calls (ceil(ticks / K)).
The reward is (end_tick + 1) * timestep for an env that ended and K * timestep otherwise, (N,) on the device; with
reward='progress' a restarted env earns 0 and the others the sum of the ego's K deltas.  The top-level action_repeat, which
runs straight through an env's end, cannot be combined with autoreset.
param_draw={'ranges': {key: (lo, hi)} or one dict per agent, 'groups': [['m', 'I']], 'per_env': bool, 'seed': s} (batched mode
only; Simulator.set_param_draw): per-episode dynamics randomisation.  reset() draws every env's car after placing the agents,
reset_envs() the masked envs', and the autoreset modes draw every env they restart on the device; info['params'] is the (N, A, 18)
parameter table after the step (maps.PARAM_KEYS order), i.e. a restarted env's new car.
The gym 0.19 API with the non-standard reset(poses) is kept on purpose (SURVEY.md 8b).
"""
import numpy as np
import torch

from . import maps as hostmaps
from . import param_draw as pdraw
from .simulator import RENDER_MAX_AGENTS, Integrator, Simulator

# observation key -> Simulator.update_progress view (added with the centerline kwarg)
PROGRESS_KEYS = (('track_s', 's'), ('track_d', 'd'), ('track_heading_error', 'heading_error'), ('progress', 'progress'))


class F110Env(object):
    metadata = {'render.modes': ['human', 'human_fast', 'rgb_array']}
    render_callbacks = []

    def __init__(self, **kwargs):
        self.seed = kwargs.get('seed', 12345)
        if 'map' in kwargs:
            self.map_name = kwargs['map']
            if isinstance(self.map_name, (list, tuple)):
                self.map_path = [hostmaps.resolve_map_path(m) for m in self.map_name]
            else:
                self.map_path = hostmaps.resolve_map_path(self.map_name)
        else:
            self.map_name = 'vegas'
            self.map_path = hostmaps.resolve_map_path('vegas')
        self.map_ext = kwargs.get('map_ext', '.png')
        self.params = kwargs.get('params', dict(hostmaps.DEFAULT_PARAMS))
        self.num_agents = kwargs.get('num_agents', 2)
        self._local_map = self._local_map_settings(kwargs.get('local_map', None))
        if self._local_map is not None and self.num_agents > RENDER_MAX_AGENTS:
            raise ValueError('local_map draws at most %d agents per env' % RENDER_MAX_AGENTS)
        self.timestep = kwargs.get('timestep', 0.01)
        self.ego_idx = kwargs.get('ego_idx', 0)
        self.integrator = kwargs.get('integrator', Integrator.RK4)
        self.lidar_dist = kwargs.get('lidar_dist', 0.0)
        num_envs = kwargs.get('num_envs', None)
        self.batched = num_envs is not None
        self.num_envs = int(num_envs) if self.batched else 1
        if isinstance(self.map_path, (list, tuple)) and not self.batched:
            raise ValueError('a list of maps needs the batched mode (num_envs)')
        self._obstacles = self._obstacle_settings(kwargs.get('obstacles', None), self.batched)
        lidar = kwargs.get('lidar', None)
        if lidar is not None:
            if not self.batched:
                raise ValueError('lidar= needs the batched mode (num_envs): single-env mode runs on Simulator.step_host')
            lidar = [bool(v) for v in lidar]
            if len(lidar) != self.num_agents:
                raise ValueError('lidar needs one bool per agent (%d), got %d' % (self.num_agents, len(lidar)))
        self._autoreset = self._autoreset_settings(kwargs.get('autoreset', None), self.batched,
                                                   kwargs.get('action_repeat', 1))
        self._param_draw = self._param_draw_settings(kwargs.get('param_draw', None), self.batched, self.params,
                                                     self.num_agents)
        self.start_thresh = 0.5
        self.sim = Simulator(self.params, self.num_agents, self.seed, time_step=self.timestep,
                             ego_idx=self.ego_idx, integrator=self.integrator, lidar_dist=self.lidar_dist,
                             num_envs=self.num_envs, num_beams=kwargs.get('num_beams', 1080),
                             fov=kwargs.get('fov', 4.7), device=kwargs.get('device', None),
                             noise_std=kwargs.get('scan_noise_std', 0.01))
        self.env_map_ids = kwargs.get('env_map_ids', None)
        self.mixed_resolution = bool(kwargs.get('mixed_resolution', False))
        self.rotated_origins = bool(kwargs.get('rotated_origins', False))
        self.reward_kind = kwargs.get('reward', 'timestep')
        if self.reward_kind not in ('timestep', 'progress'):
            raise ValueError("reward must be 'timestep' or 'progress', got %r" % (self.reward_kind,))
        self.centerline = kwargs.get('centerline', None)
        if self.reward_kind == 'progress' and self.centerline is None:
            raise ValueError("reward='progress' needs centerline=")
        self.action_repeat = kwargs.get('action_repeat', 1)
        if int(self.action_repeat) != self.action_repeat or not 1 <= self.action_repeat <= 64:
            raise ValueError('action_repeat must be an int in [1, 64], got %r' % (self.action_repeat,))
        self.action_repeat = int(self.action_repeat)
        self._set_map(self.map_path, self.map_ext)
        if lidar is not None:
            self.sim.set_lidar(lidar)
        if self._autoreset is not None:
            self.sim.set_episodes(self._autoreset['max_episode_steps'] * self._autoreset['action_repeat'])
            p = self._autoreset['poses']
            self._autoreset['poses'] = [t.to(self.sim.device) for t in p] if isinstance(p, list) else p.to(self.sim.device).contiguous()
        if self._param_draw is not None:
            cfg = self._param_draw
            self.sim.set_param_draw(cfg['ranges'], cfg.get('groups'), cfg.get('per_env', False), cfg.get('seed', 0))
        if self._obstacles is not None:
            cand, count, clearance, seed = self._obstacles
            self.sim.set_obstacles(np.zeros((count[1], 5)), np.zeros(count[1], bool))
            self.sim.set_obstacle_draw(cand, count=count, clearance=clearance, seed=seed)
        self.render_obs = None
        self._local_map_buf = None
        self._palette = None
        # single-env mode: the whole observation comes back in ONE batch of async copies + one stream sync
        # (C ABI f110_step_host) instead of a blocking .cpu() per field
        self._io = None if self.batched else self.sim.make_host_io()

    # env-level state lives on the device (f110_env.py:165-189); expose the reference's attribute names
    @property
    def lap_times(self):
        return self._out(self.sim.lap_times)

    @property
    def lap_counts(self):
        return self._out(self.sim.lap_counts)

    @property
    def toggle_list(self):
        return self._out(self.sim.toggle_list)

    @property
    def current_time(self):
        return self.sim.current_time if self.batched else float(self.sim.current_time[0].item())

    @property
    def collisions(self):
        return self._out(self.sim.collisions)

    def _out(self, t):
        t = t.view(self.num_envs, self.num_agents)
        return t if self.batched else t[0].cpu().numpy()

    def _finish(self, obs, episode=False):
        sim = self.sim
        if not episode:
            sim.env_post_step()
        N, A = self.num_envs, self.num_agents
        reward = self.timestep
        if self.batched:
            if self._local_map is not None:
                obs['local_map'] = self._render_local_map()
            obs['lap_times'] = sim.lap_times.view(N, A)
            obs['lap_counts'] = sim.lap_counts.view(N, A)
            self._obstacle_obs(obs)
            if self.centerline is not None:
                p = sim.update_progress()
                for k, v in PROGRESS_KEYS:
                    obs[k] = p[v]
                if self.reward_kind == 'progress':
                    # a copy: rewards are often kept across steps (rollout buffers), and the delta buffer is overwritten
                    reward = p['delta'][:, self.ego_idx].clone()
            done = sim.done.bool()
            info = {'checkpoint_done': sim.checkpoint_done.view(N, A).bool()}
            if episode:
                term, trunc = obs.pop('terminated').bool(), obs.pop('truncated').bool()
                done = term | trunc
                info.update(terminated=term, truncated=trunc, episode_length=sim.episode_length,
                            final_observation=sim.final_observation)
            self._param_info(info)
            return obs, reward, done, info
        # single-env, reference-shaped (base_classes.py:594-612): lists of per-agent values
        o = {'ego_idx': obs['ego_idx'],
             'scans': [s for s in obs['scans'][0].double().cpu().numpy()],
             'collisions': obs['collisions'][0].cpu().numpy(),
             'lap_times': sim.lap_times.cpu().numpy(), 'lap_counts': sim.lap_counts.cpu().numpy()}
        for k in ('poses_x', 'poses_y', 'poses_theta', 'linear_vels_x', 'linear_vels_y', 'ang_vels_z'):
            o[k] = [float(v) for v in obs[k][0].cpu().numpy()]
        if self._local_map is not None:
            o['local_map'] = self._render_local_map()[0].cpu().numpy()
        reward = self._progress_single(o)
        done = bool(sim.done[0].item())
        info = {'checkpoint_done': sim.checkpoint_done.bool().cpu().numpy()}
        return o, reward, done, info

    def _progress_single(self, o):
        """Single env: the progress keys as numpy (A,) arrays; returns the reward (the ego's delta, or the timestep)."""
        if self.centerline is None:
            return self.timestep
        p = self.sim.update_progress()
        for k, v in PROGRESS_KEYS:
            o[k] = p[v][0].cpu().numpy()
        return float(p['delta'][0, self.ego_idx].item()) if self.reward_kind == 'progress' else self.timestep

    def _step_single(self, action):
        """Reference-shaped step of ONE env (base_classes.py:594-612 obs dict of per-agent lists): actions go through a
        pinned buffer, f110_step_host runs step + lap logic and copies scans / state / collisions / done / laps back."""
        sim, io, A = self.sim, self._io, self.num_agents
        a = np.asarray(action.cpu() if torch.is_tensor(action) else action, dtype=np.float64).reshape(A, 2)
        io['actions'].numpy()[:] = a
        sim.step_host(io)
        st = io['state'].numpy()                      # [7][A]
        lap_counts = io['lap_counts'].numpy().copy()
        o = {'ego_idx': self.ego_idx,
             'scans': [s for s in io['scans'].numpy().astype(np.float64)],
             'poses_x': [float(v) for v in st[0]], 'poses_y': [float(v) for v in st[1]],
             'poses_theta': [float(v) for v in st[4]], 'linear_vels_x': [float(v) for v in st[3]],
             'linear_vels_y': [0.0] * A, 'ang_vels_z': [float(v) for v in st[5]],
             'collisions': io['collisions'].numpy().copy(),
             'lap_times': io['lap_times'].numpy().copy(), 'lap_counts': lap_counts}
        if self._local_map is not None:
            o['local_map'] = self._render_local_map()[0].cpu().numpy()
        reward = self._progress_single(o)
        # toggle_list >= 4 (f110_env.py:243) <=> lap_counts = floor(toggle / 2) >= 2
        return o, reward, bool(io['done'].numpy()[0]), {'checkpoint_done': lap_counts >= 2}

    def step(self, action):
        """f110_env.py:263-304; with action_repeat=K, K ticks under `action` (see the module text)."""
        if self.action_repeat > 1:
            return self._step_repeat(action)
        if not self.batched:
            return self._step_single(action)
        if self._autoreset is not None and self._autoreset['action_repeat'] > 1:
            return self._step_episode_repeat(action)
        if self._autoreset is not None:
            ar = self._autoreset
            obs = self.sim.tick(action, env_level=True, autoreset_poses=ar['poses'], pose_gap=ar['pose_gap'], seed=ar['seed'])
            return self._finish(obs, episode=True)
        obs = self.sim.step(action)
        return self._finish(obs)

    def _step_repeat(self, action):
        sim, K, N, A = self.sim, self.action_repeat, self.num_envs, self.num_agents
        tracked = self.centerline is not None
        a = action if torch.is_tensor(action) else np.asarray(action, dtype=np.float64).reshape(N, A, 2)
        obs = sim.tick_repeat(a, K, env_level=True, progress=tracked)
        obs['lap_times'], obs['lap_counts'] = sim.lap_times.view(N, A), sim.lap_counts.view(N, A)
        self._obstacle_obs(obs)
        if self._local_map is not None:
            obs['local_map'] = self._render_local_map()
        reward = K * self.timestep
        if tracked:
            for k, v in PROGRESS_KEYS:
                obs[k] = sim._progress_views[v]
            if self.reward_kind == 'progress':
                reward = sim.track_delta_sum.view(N, A)[:, self.ego_idx].clone()
        done, done_tick = obs.pop('done_any').bool(), obs.pop('done_tick')
        info = {'checkpoint_done': sim.checkpoint_done.view(N, A).bool(), 'done_tick': done_tick}
        if self.batched:
            self._param_info(info)
            return obs, reward, done, info
        # single env, reference-shaped: lists of per-agent values
        o = {k: (v if k == 'ego_idx' else v[0].cpu().numpy()) for k, v in obs.items()}
        o['scans'] = [s for s in o['scans'].astype(np.float64)]
        for k in ('poses_x', 'poses_y', 'poses_theta', 'linear_vels_x', 'linear_vels_y', 'ang_vels_z'):
            o[k] = [float(v) for v in o[k]]
        reward = float(reward[0].item()) if torch.is_tensor(reward) else reward
        return o, reward, bool(done[0].item()), {'checkpoint_done': info['checkpoint_done'][0].cpu().numpy(),
                                                'done_tick': int(done_tick[0].item())}

    def _step_episode_repeat(self, action):
        """Batched episode mode with autoreset['action_repeat'] = K: one Simulator.tick_repeat call in episode mode."""
        sim, ar, N, A = self.sim, self._autoreset, self.num_envs, self.num_agents
        K = ar['action_repeat']
        tracked = self.centerline is not None
        a = action if torch.is_tensor(action) else np.asarray(action, dtype=np.float64).reshape(N, A, 2)
        obs = sim.tick_repeat(a, K, env_level=True, autoreset_poses=ar['poses'], pose_gap=ar['pose_gap'], seed=ar['seed'],
                              progress=tracked)
        obs['lap_times'], obs['lap_counts'] = sim.lap_times.view(N, A), sim.lap_counts.view(N, A)
        self._obstacle_obs(obs)
        if self._local_map is not None:
            obs['local_map'] = self._render_local_map()
        for k in ('done_any', 'done_tick'):
            obs.pop(k)
        term, trunc, end_tick = obs.pop('terminated').bool(), obs.pop('truncated').bool(), obs.pop('end_tick')
        # the ticks the env spent in its episode during the step
        reward = torch.where(end_tick >= 0, end_tick + 1, K).to(torch.float64) * self.timestep
        if tracked:
            for k, v in PROGRESS_KEYS:
                obs[k] = sim._progress_views[v]
            if self.reward_kind == 'progress':
                reward = sim.track_delta_sum.view(N, A)[:, self.ego_idx].clone()
        info = {'checkpoint_done': sim.checkpoint_done.view(N, A).bool(), 'terminated': term, 'truncated': trunc,
                'end_tick': end_tick, 'episode_length': (sim.episode_length + (K - 1)) // K,
                'final_observation': sim.final_observation}
        self._param_info(info)
        return obs, reward, term | trunc, info

    def reset(self, poses):
        """f110_env.py:306-349: zero counters, start frame, Simulator.reset, then ONE zero-action tick
        whose (obs, reward, done, info) is returned."""
        self.sim.env_reset(poses)
        if self._obstacles is not None:
            self.sim.respawn_obstacles()
        if self._param_draw is not None:
            self.sim.redraw_params()
        action = torch.zeros((self.num_envs, self.num_agents, 2), dtype=torch.float64, device=self.sim.device)
        if not self.batched:
            return self._step_single(action)
        return self._finish(self.sim.step(action))

    def reset_envs(self, env_mask, poses):
        """Batch extension: re-initialise only the masked envs (counters + Simulator.reset, then their obstacles and, with
        param_draw, their cars are redrawn); no tick is run."""
        self.sim.env_reset(poses, env_mask)
        if self._obstacles is not None:
            self.sim.respawn_obstacles(env_mask)
        if self._param_draw is not None:
            self.sim.redraw_params(env_mask)

    def _param_info(self, info):
        if self._param_draw is not None:
            info['params'] = self.sim.param_table

    @staticmethod
    def _param_draw_settings(cfg, batched, params, num_agents):
        """param_draw kwarg -> the dict, validated (param_draw.parse, and the sign conditions on the undrawn values of
        `params`), or None; ValueError before any device work."""
        if cfg is None:
            return None
        if not batched:
            raise ValueError('param_draw needs the batched mode (num_envs)')
        if not isinstance(cfg, dict) or 'ranges' not in cfg or set(cfg) - {'ranges', 'groups', 'per_env', 'seed'}:
            raise ValueError("param_draw must be a dict with 'ranges' and optionally 'groups', 'per_env', 'seed', got %r" % (cfg,))
        if cfg['ranges'] is None:
            raise ValueError('param_draw ranges must be a {key: (lo, hi)} dict or a list of one per agent slot')
        try:
            seed = int(cfg.get('seed', 0))
        except (TypeError, ValueError):
            raise ValueError('param_draw seed must be an int, got %r' % (cfg.get('seed'),))
        d = pdraw.parse(cfg['ranges'], cfg.get('groups'), cfg.get('per_env', False), seed, num_agents)
        pdraw.check_table(np.tile(hostmaps.params_vector(params), (1, num_agents, 1)), d)
        return dict(cfg, seed=seed)

    def _autoreset_settings(self, cfg, batched, action_repeat):
        """autoreset kwarg -> {'poses': device table or list, 'max_episode_steps', 'seed', 'pose_gap', 'action_repeat'}, or
        None; ValueError before any device work."""
        if cfg is None:
            return None
        if not batched:
            raise ValueError('autoreset needs the batched mode (num_envs)')
        if action_repeat != 1:
            raise ValueError("autoreset takes the held action as autoreset={..., 'action_repeat': K}, which ends each episode at "
                             'its own tick; the top-level action_repeat runs through an env\'s end and must stay 1')
        keys = {'poses', 'max_episode_steps', 'seed', 'pose_gap', 'action_repeat'}
        if not isinstance(cfg, dict) or 'poses' not in cfg or set(cfg) - keys:
            raise ValueError("autoreset must be a dict with 'poses' and optionally 'max_episode_steps', 'seed', 'pose_gap', "
                             "'action_repeat', got %r" % (cfg,))
        T = cfg.get('max_episode_steps', None)
        T = 0 if T is None else T
        if isinstance(T, bool) or int(T) != T or int(T) < 0:
            raise ValueError('autoreset max_episode_steps must be None or an int >= 0, got %r' % (T,))
        K = cfg.get('action_repeat', 1)
        if isinstance(K, bool) or not isinstance(K, (int, float, np.integer)) or int(K) != K or not 1 <= int(K) <= 64:
            raise ValueError('autoreset action_repeat must be an int in [1, 64], got %r' % (K,))
        if int(T) * int(K) > 0x7FFFFFFF:
            raise ValueError('autoreset max_episode_steps * action_repeat must fit in int32, got %r * %r' % (T, K))
        poses = cfg['poses']
        tables = poses if isinstance(poses, (list, tuple)) else [poses]
        for t in tables:
            a = np.asarray(t.cpu() if torch.is_tensor(t) else t, dtype=np.float64)
            if a.ndim != 2 or a.shape[1] != 3 or a.shape[0] < 1 or not np.all(np.isfinite(a)):
                raise ValueError('autoreset poses must be (K, 3) finite start poses, or a list of them (one per map)')
        to_dev = lambda t: torch.as_tensor(np.asarray(t.cpu() if torch.is_tensor(t) else t, dtype=np.float64))
        table = [to_dev(t) for t in poses] if isinstance(poses, (list, tuple)) else to_dev(poses)
        return {'poses': table, 'max_episode_steps': int(T), 'seed': int(cfg.get('seed', 12345)),
                'pose_gap': int(cfg.get('pose_gap', 23)), 'action_repeat': int(K)}

    def _obstacle_obs(self, obs):
        if self._obstacles is not None:
            obs['obstacles'], obs['obstacle_active'] = self.sim.obstacle_boxes, self.sim.obstacle_active

    @staticmethod
    def _obstacle_settings(cfg, batched):
        """obstacles kwarg -> (candidates, (lo, hi), clearance, seed), or None; ValueError before any device work."""
        if cfg is None:
            return None
        if not batched:
            raise ValueError('obstacles need the batched mode (num_envs)')
        if not isinstance(cfg, dict) or 'candidates' not in cfg or set(cfg) - {'candidates', 'count', 'clearance', 'seed'}:
            raise ValueError("obstacles must be a dict with 'candidates' and optionally 'count', 'clearance', 'seed', got %r"
                             % (cfg,))
        try:
            lo, hi = (int(v) for v in cfg.get('count', (1, 1)))
        except (TypeError, ValueError):
            raise ValueError('obstacles count must be (lo, hi), got %r' % (cfg.get('count'),))
        if not 0 <= lo <= hi or not 1 <= hi <= 16:
            raise ValueError('obstacles count must satisfy 0 <= lo <= hi, 1 <= hi <= 16, got %r' % (cfg.get('count'),))
        clearance = float(cfg.get('clearance', 1.0))
        if not (np.isfinite(clearance) and clearance >= 0.0):
            raise ValueError('obstacles clearance must be finite and >= 0, got %r' % clearance)
        return cfg['candidates'], (lo, hi), clearance, int(cfg.get('seed', 0))

    def update_map(self, map_path, map_ext, env_map_ids=None, mixed_resolution=None, rotated_origins=None, centerline=None):
        """f110_env.py:351-362.  Batch extension: lists of map paths (and extensions) as in the constructor;
        env_map_ids / mixed_resolution / rotated_origins None keep the current setting.  centerline: the new map's table(s) as in
        the constructor; None turns progress tracking off (the old tables belong to the old map; ValueError with
        reward='progress')."""
        if centerline is None and self.reward_kind == 'progress':
            raise ValueError("reward='progress' needs the new map's centerline=")
        if env_map_ids is not None:
            self.env_map_ids = env_map_ids
        if mixed_resolution is not None:
            self.mixed_resolution = bool(mixed_resolution)
        if rotated_origins is not None:
            self.rotated_origins = bool(rotated_origins)
        self.centerline = centerline
        self._set_map(map_path, map_ext)

    def _set_map(self, map_path, map_ext):
        """One map, or (batched mode) a list of maps stacked into one DeviceMap; env e drives on map env_map_ids[e]
        (default e % L) and auto-resets from that map's start table when Simulator.tick gets one table per map.  Then the
        centerline table(s), if any, for progress tracking."""
        self._load_map(map_path, map_ext)
        if self.centerline is not None:
            self.sim.set_centerlines(self.centerline)

    def _load_map(self, map_path, map_ext):
        if not isinstance(map_path, (list, tuple)):
            self.sim.set_map(map_path, map_ext)
            return
        if not self.batched:
            raise ValueError('a list of maps needs the batched mode (num_envs)')
        exts = list(map_ext) if isinstance(map_ext, (list, tuple)) else [map_ext] * len(map_path)
        if len(exts) != len(map_path) or len(map_path) < 1:
            raise ValueError('map_ext must be one extension or one per map')
        from .simulator import DeviceMap
        layers = [DeviceMap.from_yaml(p, e, self.sim.device) for p, e in zip(map_path, exts)]
        ids = self.env_map_ids
        if ids is None:
            ids = np.arange(self.num_envs) % len(layers)
        if len(layers) == 1:
            if np.any(np.asarray(ids) != 0):
                raise ValueError('env_map_ids must index the list of maps')
            self.sim.set_device_map(layers[0])
        else:
            self.sim.set_device_map(DeviceMap.stack(layers, mixed_resolution=self.mixed_resolution,
                                                    rotated_origins=self.rotated_origins),
                                   env_map_ids=ids)

    def update_params(self, params, index=-1):
        """f110_env.py:364-375"""
        self.sim.update_params(params, agent_idx=index)

    def add_render_callback(self, callback_func):
        """f110_env.py:377-385 (kept for API compatibility; rendering itself is out of scope)."""
        F110Env.render_callbacks.append(callback_func)

    @staticmethod
    def _local_map_settings(cfg):
        """local_map kwarg -> (size, metres_per_pixel, forward_offset), or None; ValueError for what render_views refuses."""
        if cfg is None:
            return None
        unknown = set(cfg) - {'size', 'metres_per_pixel', 'forward_offset'}
        if unknown or 'size' not in cfg or 'metres_per_pixel' not in cfg:
            raise ValueError("local_map needs 'size' and 'metres_per_pixel' (and optionally 'forward_offset'), got %r" % (cfg,))
        size = Simulator._view_size(cfg['size'])
        s, f = float(cfg['metres_per_pixel']), float(cfg.get('forward_offset', 0.0))
        if not (np.isfinite(s) and s > 0.0) or not np.isfinite(f):
            raise ValueError('local_map metres_per_pixel must be finite and > 0, forward_offset finite, got %r' % (cfg,))
        return size, s, f

    def _render_local_map(self):
        """Every agent's heading-up view into one persistent buffer, (N, A, H, W), overwritten by every step."""
        (H, W), s, f = self._local_map
        N, A = self.num_envs, self.num_agents
        if self._local_map_buf is None:
            self._local_map_buf = torch.empty((N * A, H, W), dtype=torch.uint8, device=self.sim.device)
        self.sim.render_views(None, (H, W), s, f, heading_up=True, out=self._local_map_buf)
        return self._local_map_buf.view(N, A, H, W)

    def render(self, mode='human', env_ids=None, size=(800, 1000), metres_per_pixel=0.024):
        """mode='rgb_array': each env's ego, world-aligned, as RGB uint8 (Simulator.render_views classes through the reference
        window's palette, one device gather).  size = (H, W); the defaults are the reference window (1000 x 800 pixels at
        50 px/m, zoom 1.2).  Batched mode: (K, H, W, 3) CUDA tensor for env_ids (default [0]); single env: numpy (H, W, 3)
        (env_ids None or [0]).
        'human' / 'human_fast' (the reference's pyglet window) raise NotImplementedError."""
        assert mode in self.metadata['render.modes']
        if mode != 'rgb_array':
            raise NotImplementedError('f1tenth_gym_b200 has no window renderer (pyglet/OpenGL GUI is out of scope); '
                                      "use render(mode='rgb_array').")
        envs = np.arange(1) if env_ids is None else np.asarray(env_ids).reshape(-1)
        if envs.dtype.kind not in 'iu' or envs.size < 1 or int(envs.min()) < 0 or int(envs.max()) >= self.num_envs:
            raise ValueError('env_ids must be env indices in [0, %d)' % self.num_envs)
        if not self.batched and envs.size != 1:
            raise ValueError('a single env renders one frame: env_ids must be None or [0]')
        cls = self.sim.render_views(envs * self.num_agents + self.ego_idx, size, metres_per_pixel, 0.0, heading_up=False)
        if self._palette is None:
            self._palette = torch.from_numpy(RENDER_PALETTE).to(self.sim.device)
        # an int32 index (4 bytes per pixel, not the 8 of an int64 one) into the (256, 3) palette
        rgb = torch.index_select(self._palette, 0, cls.view(-1).to(torch.int32)).view(*cls.shape, 3)
        return rgb if self.batched else rgb[0].cpu().numpy()


# class code -> RGB: the reference window's colours (rendering.py): background for off-map and free, walls, other cars, the
# followed car; an invalid view (255) is black
RENDER_PALETTE = np.zeros((256, 3), dtype=np.uint8)
RENDER_PALETTE[0] = RENDER_PALETTE[1] = (9, 32, 87)
RENDER_PALETTE[2] = (183, 193, 222)
RENDER_PALETTE[3] = (99, 52, 94)
RENDER_PALETTE[4] = (172, 97, 185)
RENDER_PALETTE[5] = (236, 146, 38)      # static obstacles
