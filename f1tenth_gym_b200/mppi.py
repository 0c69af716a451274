"""Model-predictive path integral control of any set of cars of a Simulator, on the device (C ABI include/f110_mppi.h).

One planning step is three launches and no host synchronisation, so it can be captured in a CUDA graph with the tick:
  1. f110_mppi_sample: K noisy copies of each agent's nominal action sequence (sample 0 is the nominal itself), clamped to the
     bounds; an agent whose env restarted since the last step starts again from a zero nominal;
  2. f110_predict_scored: the K futures of H ticks of every agent and their costs along the map's centerline;
  3. f110_mppi_update: the softmin-weighted mean of the samples, its first step written to the agent's row of the action
     tensor, the rest shifted into the nominal.

    sim.set_centerlines(f1tenth_gym_b200.maps.load_waypoints()[:, :2])    # (x, y) of the raceline
    ego = MPPIPlanner(sim, agent_ids=np.arange(N) * A, horizon=30, samples=256)
    pp = PurePursuitPlanner(...)
    actions = torch.zeros((N * A, 2), dtype=torch.float64, device=sim.device)
    pp.plan_into(x, y, yaw, 0.82, 1.0, actions)     # every row; the ego rows are then overwritten
    ego.plan_into(actions)
    sim.tick(actions.view(N, A, 2), autoreset_poses=starts)

With F110Env, pass env.sim.
"""
import ctypes as C

import numpy as np
import torch

from . import _native as nat
from .simulator import COST_DEFAULTS, _stream_ptr

# noise std (steer rad, speed m/s) and temperature of MPPIPlanner when none are given
NOISE_DEFAULT = (0.2, 1.5)
TEMPERATURE_DEFAULT = 1.0


class MPPIPlanner(object):
    def __init__(self, sim, agent_ids, horizon, samples, noise_std=NOISE_DEFAULT, temperature=TEMPERATURE_DEFAULT,
                 weights=None, bounds=None, seed=0, diagnostics=False):
        """A planner for the M agents agent_ids (flat ids e*A + slot, distinct) of sim, over `horizon` ticks with `samples`
        candidate sequences each.  noise_std = (steer, speed) std; temperature: lambda of the softmin weights; weights: a
        cost dict as Simulator.predict(cost=) takes (missing keys: COST_DEFAULTS); bounds = (steer_lo, steer_hi, speed_lo,
        speed_hi), None for s_min, s_max, v_min, v_max of sim.params; seed: of the sampling noise.  diagnostics=True keeps
        the weights (M, K) and argmin (M,) of every update.  The sim needs a map the predict path can run on and
        set_centerlines (its window and reacquire_dist are the tracker's).  ValueError before any device work for a bad
        shape, size, weight or id."""
        self.sim = sim
        if sim.map is None:
            raise ValueError('MPPIPlanner needs a map: call set_map or set_device_map first')
        self._cost_c = sim._cost_struct({} if weights is None else weights)
        NA = sim.num_envs * sim.num_agents
        ids = np.asarray(agent_ids.cpu() if torch.is_tensor(agent_ids) else agent_ids)
        if ids.dtype.kind not in 'iu' or ids.ndim != 1 or ids.size < 1:
            raise ValueError('agent_ids must be a non-empty 1-d sequence of integers')
        if int(ids.min()) < 0 or int(ids.max()) >= NA:
            raise ValueError('agent_ids must lie in [0, %d), got [%d, %d]' % (NA, int(ids.min()), int(ids.max())))
        if np.unique(ids).size != ids.size:
            raise ValueError('agent_ids must be distinct: each planner row writes its own action row')
        M, K, H = int(ids.size), int(samples), int(horizon)
        if K != samples or H != horizon or not 2 <= K <= nat.MPPI_MAX_K or not 1 <= H <= nat.MPPI_MAX_H or M * K * H > 0x7fffffff:
            raise ValueError('MPPIPlanner needs 2 <= samples <= %d, 1 <= horizon <= %d and agents * samples * horizon < 2^31, '
                             'got samples=%r horizon=%r' % (nat.MPPI_MAX_K, nat.MPPI_MAX_H, samples, horizon))
        try:
            sig = [float(v) for v in noise_std]
        except (TypeError, ValueError):
            raise ValueError('noise_std must be (steer, speed), got %r' % (noise_std,))
        if len(sig) != 2 or not all(np.isfinite(v) and v >= 0.0 for v in sig):
            raise ValueError('noise_std must be two finite values >= 0, got %r' % (noise_std,))
        lam = float(temperature)
        if not (np.isfinite(lam) and lam > 0.0):
            raise ValueError('temperature must be finite and > 0, got %r' % (temperature,))
        if bounds is None:
            p = sim.params
            bounds = (p['s_min'], p['s_max'], p['v_min'], p['v_max'])
        try:
            b = [float(v) for v in bounds]
        except (TypeError, ValueError):
            raise ValueError('bounds must be (steer_lo, steer_hi, speed_lo, speed_hi), got %r' % (bounds,))
        if len(b) != 4 or not all(np.isfinite(b)) or b[0] > b[1] or b[2] > b[3]:
            raise ValueError('bounds must be four finite values with lo <= hi, got %r' % (bounds,))
        mc, bc = sim._map_struct, sim.beams.c
        if not (sim.march_rec is not None and mc.sincos2 and mc.dt_min_positive > mc.eps and 0.0 < bc.side_max < mc.max_range):
            raise ValueError('MPPIPlanner needs the predict path: the lean ray march and side distances below max_range')
        self.M, self.K, self.H = M, K, H
        dev = sim.device
        f64 = dict(dtype=torch.float64, device=dev)
        self.agent_ids = torch.from_numpy(ids.astype(np.int32)).to(dev)
        self._nominal = torch.zeros((M, H, 2), **f64)
        self.iteration = torch.zeros((1,), dtype=torch.int64, device=dev)
        self.no_finite = torch.zeros((M,), dtype=torch.int32, device=dev)
        self.samples_actions = torch.zeros((M, K, H, 2), **f64)
        self.cost = torch.zeros((M, K), **f64)
        self._final_state = torch.empty((M, K, 7), **f64)
        self._wall_step = torch.empty((M, K), dtype=torch.int32, device=dev)
        self._seg0 = torch.empty((M,), dtype=torch.int32, device=dev)
        self._s0 = torch.empty((M,), **f64)
        self.weights = torch.zeros((M, K), **f64) if diagnostics else None
        self.argmin = torch.zeros((M,), dtype=torch.int32, device=dev) if diagnostics else None
        self._out = torch.zeros((NA, 2), **f64)
        self._mppi_c = nat.F110Mppi(M, K, H, nat.ptr(self.agent_ids), nat.ptr(self._nominal), nat.ptr(self.iteration),
                                    nat.ptr(self.no_finite), sig[0], sig[1], b[0], b[1], b[2], b[3], lam, int(seed) & (2 ** 64 - 1))
        c = self._cost_c
        c.prev_action, c.cost, c.seg0, c.s0 = None, nat.ptr(self.cost), nat.ptr(self._seg0), nat.ptr(self._s0)
        self._args = nat.F110PredictArgs(nat.ptr(self.agent_ids), nat.ptr(self.samples_actions), M, K, H,
                                         nat.ptr(self._final_state), nat.ptr(self._wall_step), None, None)
        self.bounds, self.noise_std, self.temperature = tuple(b), tuple(sig), lam

    @property
    def nominal(self):
        """(M, H, 2) the nominal action sequences (steer, speed); read it, do not write it (reset() does)."""
        return self._nominal

    def plan_into(self, actions):
        """One planning step: writes each agent's action into its row of actions ((N*A, 2) or (N, A, 2) fp64 CUDA tensor) and
        leaves every other row alone.  No host synchronisation: capturable in a CUDA graph with the tick."""
        sim = self.sim
        NA = sim.num_envs * sim.num_agents
        if not (torch.is_tensor(actions) and actions.is_cuda and actions.dtype == torch.float64 and actions.is_contiguous()
                and actions.numel() == 2 * NA and actions.shape[-1] == 2 and actions.device == sim.state.device):
            raise ValueError('actions must be a contiguous float64 (N*A, 2) or (N, A, 2) tensor on %s' % sim.state.device)
        if sim.centerlines is None:
            raise ValueError('MPPIPlanner needs the centerlines of set_centerlines')
        L = nat.lib()
        st = _stream_ptr(sim.device)
        ep = C.byref(sim._episodes) if sim._episodes is not None else None
        nat.check(L.f110_mppi_sample(C.byref(sim.c), C.byref(self._mppi_c), ep, nat.ptr(self.samples_actions), st))
        nat.check(L.f110_predict_scored(C.byref(sim.c), C.byref(sim._map_struct), C.byref(sim._march_tables),
                                        C.byref(sim.beams.c), C.byref(sim.centerlines.c), C.byref(self._args),
                                        C.byref(self._cost_c), st))
        nat.check(L.f110_mppi_update(C.byref(self._mppi_c), nat.ptr(self.samples_actions), nat.ptr(self.cost),
                                     nat.ptr(actions), NA, nat.ptr(self.weights), nat.ptr(self.argmin), st))
        return actions

    def plan(self):
        """One planning step -> (M, 2) actions (steer, speed) of the planner's agents, in agent_ids order."""
        self.plan_into(self._out)
        return self._out[self.agent_ids.long()]

    def reset(self, env_mask=None):
        """Zero the nominals of the agents in the envs of env_mask ((N,) bools; None: every agent), on the device."""
        if env_mask is None:
            self._nominal.zero_()
            return
        m = torch.as_tensor(env_mask).to(self.sim.device).reshape(-1).bool()
        if m.numel() != self.sim.num_envs:
            raise ValueError('env_mask must hold one flag per env (%d)' % self.sim.num_envs)
        hit = m[self.agent_ids.long() // self.sim.num_agents]
        self._nominal.masked_fill_(hit[:, None, None], 0.0)
