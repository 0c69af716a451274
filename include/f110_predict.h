/*
 * f110_predict.h — batched single-agent rollouts for sampling-based control (libf110_b200.so, ABI v6): K candidate futures of
 * M agents, H ticks each, in one launch.  An addition to the ABI of f110_b200.h, whose conventions it follows; kept in a
 * header of its own so that the headers it builds on keep their entry-point sets.
 */
#ifndef F110_PREDICT_H
#define F110_PREDICT_H

#include "f110_param_draw.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- predicted futures (batch extension; csrc/predict.cuh) ---- */
/* Sample (m, k), m < M, k < K, starts from agent a = agent_ids[m] (flat id e*A + slot; repeats allowed): its state[.][a],
 * steer_buf[.][a], steer_cnt[a], its parameter row (params_per_env ? a : a % A) and its env's map layer (env_layer[a / A] when
 * the map is a stack).  Step h < H runs one tick of that agent alone under actions[m][k][h] = (steer, speed):
 *   - the steering FIFO of depth 2                              (reference base_classes.py:270-278)
 *   - pid                                                       (dynamic_models.py:178-221)
 *   - RK4 or Euler with sim->integrator and sim->timestep       (base_classes.py:282-404)
 *   - the single-shot yaw wrap                                  (base_classes.py:400-404)
 *   - the scan pose with lidar_dist                             (base_classes.py:406-409)
 *   - the iTTC wall check on the wall-only scan, with the tick's threshold, beam tables and predicate
 *                                                               (laser_models.py:188-217, base_classes.py:428-449, :229-243)
 *   - on a hit, state[3:] = 0, the yaw included                 (base_classes.py:229-254 RaceCar.check_ttc)
 * No scan noise, opponents, boxes, lap, time, done, auto-reset, episode or progress logic: on a simulator with noise_std == 0
 * the state after step h is bit-identical to that agent's state after h + 1 ticks of f110_tick* from the same buffers under
 * the same actions (no auto-reset), and the wall check fires on the same ticks.  An agent's own future does not depend on its
 * opponents or boxes: they only clip scans and set collisions, and the wall check reads the wall-only scan.
 *
 * Reads state, steer_buf, steer_cnt, params, env_layer, the map and the beams; writes only the outputs below; keeps no global
 * state, allocates nothing and does not synchronise (capturable in a CUDA graph, safe on two streams).  One launch, a thread
 * per sample; output offsets are 64-bit.  An agent id outside [0, N*A) gives NaN states, wall_step -1 and NaN clearance for its
 * samples and reads nothing. */
typedef struct {
    const int32_t *agent_ids;       /* [M] device: flat source agent ids */
    const double *actions;          /* [M][K][H][2] device: (steer, speed) per step, the tick's action layout */
    int32_t M, K, H;                /* M >= 1, K >= 1, M * K <= 2^31 - 1, 1 <= H <= F110_PREDICT_MAX_H */
    double *final_state;            /* [M][K][7] device: the state after step H - 1 (x, y, steer, v, yaw, yaw_rate, slip) */
    int32_t *wall_step;             /* [M][K] device: the first step whose wall check fired, -1 for none */
    double *states;                 /* [M][K][H][7] device, or NULL: the state after every step */
    float *clearance;               /* [M][K][H] device, or NULL: fp32 of the metre distance transform at each step's scan pose
                                       (the reference's distance_transform value there, the first lookup of every beam) */
} f110_predict_args;

#define F110_PREDICT_MAX_H 4096

/* F110_ERR_INVALID before anything is enqueued for: sim, args, agent_ids, actions, final_state or wall_step NULL; M < 1,
 * K < 1, M * K > 2^31 - 1, H outside [1, F110_PREDICT_MAX_H]; what f110_step refuses of the sim, map and beams; and a map and
 * beam setup on which f110_tick_repeat's short path cannot run (the tick's march is not a lean kernel -- no march record
 * buffer, no doubled LUT, dt_min_positive <= eps, ... -- or beams->side_max is unknown or not below max_range).  The sim's
 * noise_std and its agent count do not matter.  F110_ERR_NO_MAP without a table. */
int f110_predict(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                 const f110_predict_args *args, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* F110_PREDICT_H */
