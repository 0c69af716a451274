/*
 * f110_episode_repeat.h — episodes under a held action (libf110_b200.so, ABI v6): f110_tick_repeat's K ticks under one action,
 * in episode mode, where an env's episode stops at the first tick that ends it.  An addition to the ABI of f110_episodes.h,
 * whose conventions it follows; kept in a header of its own so that the two headers it builds on keep their entry-point sets.
 */
#ifndef F110_EPISODE_REPEAT_H
#define F110_EPISODE_REPEAT_H

#include "f110_episodes.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- episodes under a held action (batch extension; csrc/episode_repeat.cuh) ---- */
/* Episode mode; one call runs `repeat` = K ticks under one action -- the ticks of f110_tick_repeat_ticks_lidar with
 * env_level = 1 and without auto-reset, so the short path of its intermediate ticks and the lidar mask apply as there -- and
 * decides after every tick j,
 * for every env whose episode is still running in the call, what f110_tick_episodes decides after its tick: ticks[e] += 1,
 * terminated = done, truncated = !terminated && max_ticks > 0 && ticks >= max_ticks.  Let j_e be the first tick at which env e's
 * episode ends.
 *   - An env that does not end: every buffer is bit for bit what f110_tick_repeat (without auto-reset) leaves, scans included;
 *     ticks grows by K; terminated = truncated = 0; end_tick = -1.
 *   - An env that ends at j: its episode stops there, as if its K-tick loop had stopped.  final_state, final_collisions,
 *     final_collision_idx, final_lap_times and final_lap_counts are what plain tick j left; final_scans of its lidar slots is
 *     the scan plain tick j produced -- also on an intermediate tick of the short path, which computes no scans: the call
 *     snapshots that tick's scan inputs and computes the scan once, after the K ticks (k_restart_march's march, the opponent
 *     ray-cast and the box clip).  length = ticks at j, the flags as decided at j, end_tick = j, done = done at j, and
 *     done_any / done_tick count ticks <= j only.  Nothing that happens to the env after j inside the call is visible.
 *   - After the K ticks every env that ended is restarted as f110_tick_episodes restarts it, at the tick counter of the call's
 *     last tick: the start-pose draw and the box respawn draw, track_seg = -1, ticks = 0, then one zero-action tick of those
 *     envs alone with the restart noise of counter t | 2^63.  track_delta_sum (when given) is 0 for their agents.
 * K = 1 is f110_tick_episodes bit for bit, plus done_any, done_tick and end_tick.  Rows of sensorless slots in scans and
 * final_scans are written only where f110_tick_episodes writes them.  Lists are built on the device and no result depends on
 * their order; no allocation, no host synchronisation: capturable in a CUDA graph. */
typedef struct {
    int32_t *end_tick;              /* [N] the tick 0..K-1 of the call at which the env's episode ended, -1 = none */
    double *snap_rec;               /* [N*A][8] device scratch: march_rec of the end tick (short path) */
    double *snap_poses;             /* [N*A][5] device scratch: agent_poses of the end tick */
    int32_t *snap_wall_flag;        /* [N*A] device scratch: wall_flag of the end tick */
    uint32_t *scan_list;            /* [N] device scratch: the envs whose final scan is computed after the K ticks */
    uint32_t *scan_count;           /* [1] device scratch, zeroed by the call on `stream` */
    double *track_delta_sum;        /* [N*A] f110_track_progress_sum's sum, or NULL: set to 0 for the restarted envs' agents */
} f110_episode_repeat;

/* One call.  F110_ERR_INVALID before anything is enqueued for what f110_tick_repeat_ticks_lidar rejects (with env_level = 1),
 * what f110_tick_episodes rejects, and er or any of its buffers NULL (track_delta_sum may be).  The launch record
 * (f110_debug_last_launch) is the last plain tick's, then " repeat=... sub=... UNITS=... grid=... episodes restart=<kernels>
 * restart_grid=<blocks of k_restart_march> final_scan=<kernels|none>". */
int f110_tick_repeat_episodes(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                              const double *actions, int32_t repeat, const f110_repeat *rep, const double *start_poses,
                              int32_t num_start, int32_t pose_gap, uint64_t seed, const f110_obstacles *obst,
                              const f110_lidar *lidar, const f110_episodes *ep, const f110_episode_repeat *er, void *stream);
/* Ticks first_tick .. first_tick + num_ticks - 1 of such a call, for a caller that has launches of its own to put between the
 * ticks (f110_track_progress_sum after every tick): issuing the ranges of one call in order, with the same arguments, is the
 * call.  first_tick == 0 zeroes the scratch counts; the final scans and the restart run with the range that holds the last
 * tick.  F110_ERR_INVALID for a range outside [0, repeat). */
int f110_tick_repeat_episodes_ticks(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables,
                                    const f110_beams *beams, const double *actions, int32_t repeat, int32_t first_tick,
                                    int32_t num_ticks, const f110_repeat *rep, const double *start_poses, int32_t num_start,
                                    int32_t pose_gap, uint64_t seed, const f110_obstacles *obst, const f110_lidar *lidar,
                                    const f110_episodes *ep, const f110_episode_repeat *er, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* F110_EPISODE_REPEAT_H */
