/*
 * f110_param_draw.h — per-episode dynamics randomisation (libf110_b200.so, ABI v6): redraw the per-env parameter table
 * (f110_sim.params with params_per_env = 1) of the envs that start a new episode, on the device.  An addition to the ABI of
 * f110_b200.h, whose conventions it follows; kept in a header of its own so that the headers it builds on keep their
 * entry-point sets.
 */
#ifndef F110_PARAM_DRAW_H
#define F110_PARAM_DRAW_H

#include "f110_episodes.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- per-episode parameter draws (batch extension; csrc/param_draw.cuh) ---- */
/* The counter-based draw.  When env e is drawn at tick counter t (*f110_sim.tick_counter, read on the device when the draw
 * runs), every key k whose bit is set in keys[i] gets, for agent slot i < A,
 *     v = lo[i][k] + u * (hi[i][k] - lo[i][k])          (fp64, no FMA)
 *     u = (h >> 11) 2^-53,   h = mix64(seed + C1 (t+1) + C2 (e+1) + C3 (s+1) + C4 (g+1))  mod 2^64
 * with s = per_env ? 0 : i (per_env: every car of an env shares its draws, as a surface friction would), g = group[k] (keys of
 * one group share u: m and I scale together), mix64 the finaliser of the auto-reset's start-pose draw and the constants below.
 * Keys whose bit is clear keep their table value.  width and length (keys 16 and 17) are not drawable: the opponent ray-cast
 * reads them while GJK and the views read sim_length / sim_width, so a draw would split one car into two bodies.
 *
 * The caller's obligations (lo / hi are device memory; the library does not read them on the host):
 *   - finite lo <= hi for every drawn key;
 *   - on every drawn range and on the undrawn values of a slot that has a drawn key:  mu, C_Sf, C_Sr, lf, lr, m, I, v_switch,
 *     a_max, v_max > 0;  h >= 0;  s_min, sv_min <= 0;  s_max, sv_max >= 0;  v_min < 0.
 * Under them a car at rest with an empty steer FIFO stays at rest under the action (0, 0) whatever the drawn values: pid gives
 * sv = accl = 0 and the kinematic branch returns zero derivatives.  That is why a draw issued after the zero-action tick of an
 * episode restart is exact: the new episode runs on the drawn values from its first tick on. */
#define F110_PARAM_DRAW_C1 0xC2B2AE3D27D4EB4Full   /* tick  */
#define F110_PARAM_DRAW_C2 0x165667B19E3779F9ull   /* env   */
#define F110_PARAM_DRAW_C3 0x27D4EB2F165667C5ull   /* slot  */
#define F110_PARAM_DRAW_C4 0x85EBCA77C2B2AE63ull   /* group */
#define F110_PARAM_DRAW_KEYS 16                    /* keys 0..15 are drawable */

typedef struct {
    const double *lo, *hi;          /* [A][F110_NPARAM] device: the range of every key of every slot */
    uint32_t keys[32];              /* bit k of keys[i]: key k of slot i is drawn (by value: a captured graph keeps it) */
    int32_t group[F110_NPARAM];     /* draw group of each key, in [0, F110_NPARAM); k itself = every key its own draw */
    int32_t per_env;                /* 1: the slots of an env share their draws (s = 0) */
    uint64_t seed;
    double *final_params;           /* [N*A][F110_NPARAM] device or NULL: f110_params_draw_episodes first copies an ended env's
                                       rows here (the parameters its final observation was produced with) */
} f110_param_draw;

/* Every call: one launch on `stream`, a thread per (env, slot); no allocation, no host synchronisation, capturable in a CUDA
 * graph (the tick counter is read on the device, so graph replays draw afresh).  None of them writes the launch record
 * (f110_debug_last_launch).  F110_ERR_INVALID before anything is enqueued for: sim, draw, draw->lo or draw->hi NULL;
 * sim->params_per_env == 0; more than 32 agents per env; a NULL sim->tick_counter; a bit at or above F110_PARAM_DRAW_KEYS in
 * keys[i] for i < A; a group outside [0, F110_NPARAM); no envs or agents, or a NULL sim->params (or, for the auto-reset rule,
 * sim->collisions or an ego_idx outside [0, A)). */

/* The envs whose env_mask byte is non-zero (device [N]; NULL: all): for a host reset (f110_env_reset). */
int f110_params_draw(const f110_sim *sim, const f110_param_draw *draw, const uint8_t *env_mask, void *stream);
/* The envs with collisions[e*A + ego_idx] != 0: the predicate of the plain auto-reset, which leaves collisions in place.
 * Issue it after every tick that had start_poses (f110_tick*, f110_autoreset*); under a held action with the in-call
 * auto-reset, after each tick, with the ranges of f110_tick_repeat_ticks_lidar (the short path's tail writes collisions
 * before its auto-reset too). */
int f110_params_draw_autoreset(const f110_sim *sim, const f110_param_draw *draw, void *stream);
/* The envs with ep->terminated[e] | ep->truncated[e]: after f110_tick_episodes, or after the range of
 * f110_tick_repeat_episodes_ticks that holds the last tick.  With draw->final_params set, an ended env's rows are copied
 * there first.  Also F110_ERR_INVALID for ep, ep->terminated or ep->truncated NULL. */
int f110_params_draw_episodes(const f110_sim *sim, const f110_param_draw *draw, const f110_episodes *ep, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* F110_PARAM_DRAW_H */
