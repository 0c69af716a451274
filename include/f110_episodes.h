/*
 * f110_episodes.h — episode mode of the batched F1TENTH hot path (libf110_b200.so, ABI v6): the end of an episode and its
 * restart as F110Env.reset does, for every env of a batch on the device.  An addition to the ABI of f110_b200.h, whose
 * conventions it follows; kept in a header of its own so that f110_b200.h keeps the entry-point set of its own features.
 */
#ifndef F110_EPISODES_H
#define F110_EPISODES_H

#include "f110_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- episodes: the end of an episode and its restart as F110Env.reset does (batch extension; csrc/episodes.cuh) ---- */
/* An episode tick is the plain tick -- f110_tick_lidar with env_level = 1 and without auto-reset: dynamics, march, tail, lap
 * logic, done, obstacles and lidar mask as there -- followed by, per env:
 *   - the end decision: ticks[e] += 1; terminated[e] = done[e] (ego collision, or every agent checkpoint-done: _check_done,
 *     f110_env.py:204-246); truncated[e] = !terminated[e] && max_ticks > 0 && ticks[e] >= max_ticks.  The env ends when either
 *     is set, and length[e] then gets ticks[e].  Both flags are overwritten on every episode tick.
 *   - the final observation of an ended env: its agents' rows of state (7 rows), collisions, collision_idx, lap_times,
 *     lap_counts and scans are copied to the final_* buffers, bit for bit what the plain tick left, before anything is
 *     overwritten.  Rows of envs that did not end keep their contents; the scan row of a slot without a lidar (f110_lidar) is
 *     never written.
 *   - the restart of an ended env: the start poses of f110_autoreset's draw on this tick (the same hash of seed, tick counter
 *     and env, the per-layer tables and pose_gap), the env counters and start frame, the steer FIFO and wall_flag emptied, the
 *     march_cost history marked unknown, the obstacle respawn draw (with candidates; the tick counter of the draw of
 *     f110_tick_obst's auto-reset), track_seg = -1 (when given) and ticks[e] = 0.
 *   - the zero-action tick of the restarted envs alone (f110_env.py:306-349: reset places the agents, then steps once under
 *     zero actions): the tick's dynamics under the action (0, 0), a full scan of every restarted agent whose scan exists with
 *     the arithmetic of the tick's march for the map kind (cell units, metres, canvas stacks, rotated origins, the literal path
 *     for absurd poses), the iTTC predicate, GJK against the env's agents and boxes, the opponent ray-cast and the obstacle
 *     clip, and the lap logic.  The tick counter does not advance and done keeps the plain tick's value, so the tick that ended
 *     the episode reports done = 1.  With scan noise the restart scans take the draw a plain tick at counter t | 2^63 makes
 *     (t: the counter of the tick that ended the episode), independent of the crash scan's noise.
 * A restarted env is then, bit for bit, what f110_env_reset + f110_reset at its drawn start poses, the tick counter set to
 * (t | 2^63) - 1, f110_step_lidar under zero actions and f110_env_post_step leave, except done, tick_counter and the march
 * queue.  Every other env is exactly the plain tick's.  The restart list is built on the device; no result depends on its
 * order.  No allocation, no host synchronisation: capturable in a CUDA graph. */
typedef struct {
    int32_t max_ticks;              /* time limit in ticks, 0 = none */
    int32_t *ticks;                 /* [N] ticks of the running episode */
    uint8_t *terminated;            /* [N] */
    uint8_t *truncated;             /* [N] */
    int32_t *length;                /* [N] ticks of the last ended episode */
    double *final_state;            /* [F110_NSTATE][N*A] */
    float *final_scans;             /* [N*A][num_beams] */
    double *final_collisions;       /* [N*A] */
    int32_t *final_collision_idx;   /* [N*A] */
    double *final_lap_times, *final_lap_counts;   /* [N*A] */
    uint32_t *list;                 /* [N] device scratch: the restarted envs */
    uint32_t *list_count;           /* [1] device scratch, zeroed by the call on `stream` */
    int32_t *track_seg;             /* [N*A] f110_progress.seg, or NULL: set to -1 for the restarted envs' agents */
} f110_episodes;

/* One episode tick.  F110_ERR_INVALID before anything is enqueued for: ep or any of its buffers NULL (track_seg may be),
 * max_ticks < 0, more than 32 agents per env, start_poses NULL, a tick whose ray march is not one of the lean kernels (the
 * restart march shares their arithmetic), and what f110_tick_lidar rejects.  The launch record (f110_debug_last_launch) gains
 * " episodes restart=<kernels> restart_grid=<blocks of k_restart_march>". */
int f110_tick_episodes(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                       const double *actions, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
                       const f110_obstacles *obst, const f110_lidar *lidar, const f110_episodes *ep, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* F110_EPISODES_H */
