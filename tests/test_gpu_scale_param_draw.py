"""Per-episode parameter draws against the CPU oracle at benchmark batch sizes.

The episode cases of test_gpu_scale_features (a captured episode tick) and test_gpu_scale_episode_repeat (a captured
tick_repeat(a, 4) episode call) at 16384 x 2 (on 132 SMs), run again with set_param_draw on mu, C_Sf, C_Sr, m, I, a_max and
v_max drawn wide (m and I in one group).  Their drivers are reused as they are; this file wraps three of their helpers:
  * make_sim also sets the draw and draws every env once (redraw_params), as F110Env.reset does;
  * make_world writes that table into each OracleSim's parameter rows;
  * restart_env, the oracle's restart of an ended env at the device's tick counter, also writes the restated draw
    (param_draw.draw_env) into the env's rows before the oracle's zero-action step.
Everything the drivers compare (every env after every call, at the tolerances of test_gpu_scale.run_vs_oracle) therefore checks
that the restarted envs drive their new cars from the first tick, and that the zero-action restart tick does not depend on the
drawn keys.  After the run the device table must equal the restated one bit for bit, thousands of envs must have restarted,
and the drawn rows must differ across envs.
"""
import numpy as np
import pytest

import test_gpu_scale_episode_repeat as ser
import test_gpu_scale_features as sf
from test_gpu_scale import default_launch_settings, dev, example_map, f110, sms  # noqa: F401

pytestmark = pytest.mark.gpu

DRAW = {'mu': (0.5, 1.5), 'C_Sf': (3.0, 6.5), 'C_Sr': (3.5, 7.5), 'm': (2.8, 4.8), 'I': (0.03, 0.065), 'a_max': (5.0, 13.0),
        'v_max': (10.0, 26.0)}


def with_draw(monkeypatch, module):
    """Wrap module's make_sim, make_world and restart_env so that the run draws on the device and the oracle follows."""
    from f1tenth_gym_b200 import param_draw as pd
    state = dict(restarts=0)
    make_sim, make_world, restart_env = module.make_sim, module.make_world, module.restart_env

    def make_sim_draw(*a, **kw):
        sim = make_sim(*a, **kw)
        sim.set_param_draw(DRAW, groups=[['m', 'I']], seed=77)
        sim.redraw_params()
        state['sim'], state['table'] = sim, sim.param_table.cpu().numpy()
        return sim

    def make_world_draw(*a, **kw):
        world = make_world(*a, **kw)
        for e, s in enumerate(world.sims):
            s.params[:world.A] = state['table'][e]
        return world

    def restart_env_draw(f110, world, tables, ids, tick, e):
        restart_env(f110, world, tables, ids, tick, e)
        row = pd.draw_env(state['table'][e], state['sim'].param_draw, tick, e)
        state['table'][e] = row
        world.sims[e].params[:world.A] = row
        state['restarts'] += 1

    monkeypatch.setattr(module, 'make_sim', make_sim_draw)
    monkeypatch.setattr(module, 'make_world', make_world_draw)
    monkeypatch.setattr(module, 'restart_env', restart_env_draw)
    return state


def check_table(state):
    got = state['sim'].param_table.cpu().numpy()
    assert np.array_equal(got.view(np.int64), state['table'].view(np.int64)), 'device table != restated draws'
    N = got.shape[0]
    print('restarts with a draw: %d over %d envs' % (state['restarts'], N))
    assert state['restarts'] >= 2000, state['restarts']
    assert len(np.unique(got[:, 0, 0])) > N // 2
    assert len(np.unique(got[:, 1, 6])) > N // 2


def test_episode_tick_draws_at_bench_size(f110, dev, sms, example_map, monkeypatch):
    state = with_draw(monkeypatch, sf)
    sf.test_episodes_graph_with_bulk_restarts(f110, dev, sms, example_map, 'mask_boxes')
    check_table(state)


def test_repeat_episode_draws_at_bench_size(f110, dev, sms, example_map, monkeypatch):
    state = with_draw(monkeypatch, ser)
    ser.test_repeat_episodes_graph_with_boxes_and_mask_at_bench_size(f110, dev, sms, example_map)
    check_table(state)
