/*
 * f110_b200.h — C ABI of the batched F1TENTH hot path for the H100 (libf110_b200.so).
 *
 * The reference (f1tenth/f1tenth_gym) is pure Python + numba and has no FFI of its own; its
 * boundary for this path is the Python surface  F110Env -> Simulator -> @njit kernels.  Each entry
 * point below replaces one of those Python-level interfaces (cited file:line, paths relative to
 * gym/f110_gym/envs/ of the reference).  INTEGRATION.md shows the ctypes stub a maintainer of the
 * reference would add to bind them.
 *
 * Conventions
 *   - plain C types only; every pointer inside the structs is a DEVICE pointer owned by the caller
 *     (the Python host side allocates them as torch CUDA tensors), except in the *_host entry points.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *   - every function returns 0 on success or a negative f110_status; nothing is printed or thrown.
 *   - all arithmetic is IEEE fp64 without FMA contraction (the reference's numba path emits none);
 *     scans are written as fp32 (= fp32(reference fp64 value), <= 1.9e-6 m at 30 m).
 *   - agents are indexed a = env * num_agents + agent ("flat agent index"), SoA over a.
 */
#ifndef F110_B200_H
#define F110_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define F110_ABI_VERSION 6
#define F110_NPARAM 18     /* mu C_Sf C_Sr lf lr h m I s_min s_max sv_min sv_max v_switch a_max v_min v_max width length
                              (key order of the default dict, f110_env.py:130) */
#define F110_NSTATE 7      /* x y steer v yaw yaw_rate slip   (base_classes.py:97) */
#define F110_MAX_START_TABLES 64   /* per-layer auto-reset start tables (f110_sim.start_offsets) */

typedef enum {
    F110_OK = 0,
    F110_ERR_INVALID = -1,      /* bad argument (NULL pointer, non-positive size, ...)            */
    F110_ERR_NO_MAP = -2,       /* scan before a map is set (laser_models.py:445-446 ValueError)  */
    F110_ERR_CUDA = -3,         /* a CUDA runtime call failed; see f110_last_cuda_error()          */
    F110_ERR_INTEGRATOR = -4,   /* integrator not RK4(1)/Euler(2) (base_classes.py:397-398)       */
    F110_ERR_POSE_COUNT = -5,   /* reset pose count mismatch (base_classes.py:625-626 ValueError) */
    F110_ERR_AGENT_INDEX = -6   /* update_params index out of range (base_classes.py:534)         */
} f110_status;

/* ScanSimulator2D state after set_map (laser_models.py:348-427). */
typedef struct {
    int32_t height, width;
    double resolution, orig_x, orig_y, orig_c, orig_s;
    double eps, max_range;          /* 1e-4, 30.0 (laser_models.py:360) */
    int32_t theta_dis;              /* 2000 */
    int32_t fast_path;              /* 1 iff resolution is a power of two and orig_c==1, orig_s==0:
                                       x/res == x*(1/res) exactly and the rotation is the identity */
    double dt_oob;                  /* dt[-1,-1]: what an off-map ray reads (laser_models.py:79-81); also read where
                                       x_rot / resolution rounds up to width (or y_rot to height), where the
                                       reference reads past its row or table (DESIGN.md §4) */
    const double *dt;               /* [height*width] fp64 distance transform, row 0 = image bottom */
    const double *dt_cells;         /* [height*width] dt / resolution (exact when fast_path), or NULL: enables
                                       the cell-unit march; ignored unless fast_path */
    const uint8_t *dt_codes;        /* [height*width] rank of dt_cells among the map's 255 smallest distinct values,
                                       255 = escape (read dt_cells); NULL disables the coded march */
    const double *dt_lut;           /* [256] code -> dt_cells value (bit-exact) */
    const double *sines, *cosines;  /* [theta_dis]  sin/cos(linspace(0, 2pi, theta_dis)) (:379-381) */
    const double *sincos;           /* [theta_dis][2] the same values interleaved (sin, cos), or NULL */
    const double *dt_cells_pad;     /* [(height+1)*(width+1)] dt_cells with one extra row and column that hold dt[-1,-1]/resolution
                                       (the off-map value): lets the lean march clamp instead of branch; NULL = round-1 kernels */
    const uint8_t *dt_codes_pad;    /* [(height+1)][codes_pitch] rank codes of dt_cells_pad (same code book as dt_lut; columns beyond
                                       width hold the off-map code too), or NULL */
    uint32_t codes_pitch;           /* row pitch of dt_codes_pad in bytes: >= width+1 and a multiple of 16 (TMA global stride) */
    const double *sincos2;          /* [2*theta_dis][2] the interleaved LUT stored twice back to back (index k and k + theta_dis
                                       hold the same pair), or NULL: lets the march index it without the wrap branch */
    double dt_min_positive;         /* smallest value > 0 in dt (= resolution for an exact EDT), or 0 if unknown.  When it
                                       exceeds eps, `d > eps` (laser_models.py:134) is the same predicate as `d != 0` and the
                                       lean march kernel (csrc/march_lean.cuh) may be used */
    int32_t num_layers;             /* 0/1: one map.  L > 1: dt and dt_cells hold L stacked [H][W] tables that share size,
                                       resolution and origin (multi-map batches); f110_sim.env_layer picks one per env */
    /* ABI v3 */
    const double *layer_geom;       /* [num_layers][6] (orig_x, orig_y, x_max = W_l*res, y_max = H_l*res, W_l, H_l) of each layer
                                       of a canvas stack, or NULL (every layer has the geometry above).  When set, height / width
                                       are the canvas (max H_l, max W_l); layer l's table sits in the low corner of its canvas
                                       slice and every other cell of the slice (and of the extra row / column of dt_cells_pad)
                                       holds that layer's dt[-1,-1].  Unrotated origins (or layer_rot) and one resolution (or
                                       layer_res); needs the lean march kernels (F110_ERR_INVALID otherwise) */
    double layer_orig_max;          /* with layer_geom: max over the layers of max(|orig_x|, |orig_y|), a host copy for the
                                       launch-time bound on absurd coordinates (the table itself is device memory) */
    /* ABI v4 */
    const double *layer_res;        /* [num_layers][2] (res_l, RN(1/res_l)) of each layer of a canvas stack whose layers differ in
                                       resolution, or NULL (every layer has `resolution`).  Needs layer_geom (whose x_max / y_max
                                       are then W_l*res_l, H_l*res_l) and the metre table: fast_path 0, every layer marched in
                                       metres by the lean canvas-stack kernel; F110_ERR_INVALID on any other path.  Device memory */
    double layer_res_min, layer_res_max;   /* with layer_res: the finest and coarsest res_l, host copies for the launch-time
                                       bounds (the 2^31-cell floor and the absurd-coordinate reach use the finest, the
                                       extents the coarsest) */
    /* ABI v5 */
    const double *layer_rot;        /* [num_layers][2] (orig_c_l, orig_s_l) of each layer of a canvas stack that holds maps with a
                                       rotated origin, or NULL (every layer unrotated).  Needs layer_geom and layer_res (the rotated
                                       canvas is metre-only and always carries per-layer resolutions, also when there is only one):
                                       fast_path 0, every layer marched by k_march_lean_rot; F110_ERR_INVALID without those tables,
                                       with fast_path or on any other path.  One map with a rotated origin needs no table: its
                                       orig_c / orig_s above are used.  Device memory */
} f110_map;

/* Beam tables RaceCar.__init__ builds once (base_classes.py:122-158) + ScanSimulator2D.__init__ (:360-368). */
typedef struct {
    int32_t num_beams;
    double fov, angle_increment, theta_index_increment;
    const double *scan_angles, *cosines, *side_distances;   /* [num_beams] */
    const double *cos_side;         /* [num_beams][2] (cosines[i], side_distances[i]) interleaved, or NULL */
    double side_max;                /* max(side_distances), or 0 if unknown: bound used by the per-agent iTTC pre-test */
} f110_beams;

/* Simulator / RaceCar / F110Env state for N envs x A agents, SoA, caller-owned device memory. */
typedef struct {
    int32_t num_envs, num_agents;
    int32_t integrator;             /* 1 = RK4, 2 = Euler (base_classes.py:40-42) */
    int32_t ego_idx;
    int32_t params_per_env;         /* 0: params is [A][18]; 1: params is [N*A][18] */
    double timestep, lidar_dist, ttc_thresh;   /* 0.01, 0.0, 0.005 (base_classes.py:115) */
    double sim_length, sim_width;   /* Simulator.params['length'/'width'] used by check_collision (:549) */
    const double *params;           /* [A][F110_NPARAM] per agent slot (update_params, base_classes.py:514-534), or
                                       [N*A][F110_NPARAM] per env and slot when params_per_env != 0 (dynamics randomisation) */
    double *state;                  /* [F110_NSTATE][N*A] */
    double *steer_buf;              /* [2][N*A]   steering delay FIFO, row 0 = newest (base_classes.py:270-278) */
    int32_t *steer_cnt;             /* [N*A] */
    double *scan_pose;              /* [N*A][4]   (scan_x, scan_y, first DT lookup in cells | yaw, theta_index0): dynamics -> march */
    double *agent_poses;            /* [N*A][5]   Simulator.agent_poses snapshot (base_classes.py:574): x, y, yaw, cos yaw, sin yaw */
    float *scans;                   /* [N*A][num_beams] */
    int32_t *wall_flag;             /* [N*A]      RaceCar.in_collision (iTTC) */
    double *collisions;             /* [N*A]      obs['collisions'] (0./1.) */
    int32_t *collision_idx;         /* [N*A]      Simulator.collision_idx (-1 = none) */
    /* F110Env level (f110_env.py:165-189); may be NULL if f110_env_post_step is never called */
    double *current_time;           /* [N] */
    double *lap_times, *lap_counts, *toggle_list;   /* [N*A] */
    int32_t *near_starts;           /* [N*A] */
    double *start_xs, *start_ys, *start_thetas;     /* [N*A] */
    double *start_rot;              /* [N][4] */
    uint8_t *done;                  /* [N] */
    uint8_t *checkpoint_done;       /* [N*A]  info['checkpoint_done'] */
    int32_t *env_arrivals;          /* reserved (ABI v1 used it as a per-env arrival counter of f110_tick); may be NULL */
    const int32_t *env_layer;       /* [N] map layer of each env for stacked maps (f110_map.num_layers > 1), or NULL */
    unsigned long long *lookup_counter;   /* optional [1]: total DT lookups (roofline denominator); NULL = off */
    unsigned long long *tick_counter;     /* optional [1]: incremented by every f110_step; keys the noise stream
                                             and the auto-reset draw so that CUDA-graph replays stay distinct */
    /* optional work queue of the persistent ray-march kernel (csrc/march.cuh): 32-beam items, last tick's
       heavy items first.  Results never depend on it.  All NULL/0 = off (one block per 64-beam tile instead).
       I = N*A*march_ipa items; march_ipa = ceil(num_beams/32) (32-beam items) or ceil(num_beams/64) (64-beam items), <= 256. */
    uint32_t *march_cost;           /* [N*A*256] indexed by (agent << 8 | item); initialised to 0xFFFFFFFF (= unknown) */
    uint32_t *march_order;          /* [3][I]  */
    uint32_t *march_count;          /* [4]     zero-initialised by the caller */
    int32_t march_ipa;
    double *march_rec;              /* [N*A][8] per-agent record k_dynamics hands to the lean march kernel (scan position in
                                       cell units, first lookup, fixed-point LUT index, iTTC threshold, map-layer offset;
                                       csrc/march_lean.cuh), or NULL: round-1 kernels */
    /* scan noise (laser_models.py:429,450-452): N(0, noise_std^2) per beam, added before iTTC; 0 = off */
    double noise_std;
    uint64_t noise_seed;
    /* ABI v3 */
    const int32_t *start_offsets;   /* [num_start_tables + 1] in HOST memory (read when the auto-reset is enqueued, so a captured
                                       CUDA graph keeps the values it was captured with), or NULL: with env_layer set, an env on
                                       layer l auto-resets from rows [start_offsets[l], start_offsets[l+1]) of start_poses (one start
                                       table per map).  start_offsets[0] == 0, num_start == start_offsets[num_start_tables], every
                                       range non-empty, at most F110_MAX_START_TABLES tables, and f110_step / f110_tick need
                                       num_start_tables == the map's num_layers: F110_ERR_INVALID otherwise */
    int32_t num_start_tables;       /* number of ranges in start_offsets (= num_layers of the map) */
} f110_sim;

int f110_abi_version(void);
const char *f110_status_string(int status);
const char *f110_last_cuda_error(void);

/* Optional copies of a map's tables in other layouts, read only by the ray march of the tick.  Held apart from f110_map so
 * that its layout stays that of ABI v6; every pointer may be NULL (the tick then reads the f110_map tables alone). */
typedef struct {
    const double *dt_cells_brick;   /* f110_map.dt_cells_pad stored in 4x4-cell bricks (one 128-byte line each), built by
                                       f110_map_brick: element (r, c) at ((r/4)*BW + c/4)*16 + (r%4)*4 + c%4 with
                                       BW = ceil((width+1)/4); the rows are padded to a multiple of 4 and every cell beyond the
                                       padded table holds dt[-1,-1]/resolution.  Read by the ray march of a single fast-path map
                                       (num_layers <= 1, no layer_geom) at up to 1080 beams in place of dt_cells_pad; ignored
                                       on any other map and at more beams */
} f110_march_tables;

/* Size in elements of the brick table of `map`: ceil((height+1)/4)*4 * ceil((width+1)/4)*4, or 0 when the map has no brick
 * table (no dt_cells_pad, not a fast-path map, or a stack of layers) or it would hold 2^32 elements or more. */
int64_t f110_map_brick_elems(const f110_map *map);
/* Write the brick table of `map` (f110_march_tables.dt_cells_brick) into `out` (device, f110_map_brick_elems(map) fp64)
 * from map->dt_cells_pad on `stream`: a copy, bit for bit.  F110_ERR_INVALID when f110_map_brick_elems(map) is 0. */
int f110_map_brick(const f110_map *map, double *out, void *stream);

/* ---- the per-tick hot path -------------------------------------------------------------------- */
/* Each of f110_step, f110_step_profile, f110_tick and f110_step_host_async has an *_ex sibling that also takes the optional
 * tables (`tables` may be NULL: same as the plain entry point).  Results never depend on the tables; only speed does. */

/* Simulator.step (base_classes.py:553-612): pid + RK4/Euler dynamics -> 1080-beam ray-march (+fused
 * iTTC) -> GJK, wall-hit state zeroing, opponent ray-cast.  actions: device [N*A][2] = (steer, speed).
 * Launches 3 kernels on `stream`; no host synchronisation. */
int f110_step(const f110_sim *sim, const f110_map *map, const f110_beams *beams,
              const double *actions, void *stream);
int f110_step_ex(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                 const double *actions, void *stream);

/* f110_step with CUDA events recorded on `stream` around each of its three kernels; synchronises and
 * returns their durations in milliseconds: kernel_ms[0..2] = dynamics, ray-march, finalize (host array).
 * Measurement aid for bench.py's roofline figure; not for the hot loop. */
int f110_step_profile(const f110_sim *sim, const f110_map *map, const f110_beams *beams,
                      const double *actions, float *kernel_ms, void *stream);
int f110_step_profile_ex(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables,
                         const f110_beams *beams, const double *actions, float *kernel_ms, void *stream);

/* Simulator.reset / RaceCar.reset (base_classes.py:183-204, 614-630) for the envs whose env_mask
 * byte is non-zero (env_mask == NULL: all).  poses: device [N*A][3].  No tick is executed. */
int f110_reset(const f110_sim *sim, const double *poses, const uint8_t *env_mask, void *stream);

/* The counters/start-frame part of F110Env.reset (f110_env.py:319-331) for masked envs. */
int f110_env_reset(const f110_sim *sim, const double *poses, const uint8_t *env_mask, void *stream);

/* F110Env.step tail: time, _check_done lap logic (f110_env.py:204-246, 294-302) -> done, lap arrays. */
int f110_env_post_step(const f110_sim *sim, void *stream);

/* Benchmark/RL convenience (no reference equivalent; SURVEY.md 8d policy): every env whose ego has
 * collisions != 0 is reset (Simulator.reset + env counters) to start_poses[k], k drawn from a
 * counter-based hash of (seed, tick, env); agent i takes start_poses[(k - pose_gap*i) mod K].
 * What the caller sees after a tick that ended an episode: done[env] = 1 and collisions / scans of the crash
 * (the finished episode's last observation), while state, steer FIFO, lap counters, toggles and current_time are
 * those of the NEW episode (a car at rest on its start pose, time 0); done is recomputed by the next tick.
 * At most 32 agents per env (F110_ERR_INVALID otherwise; stepping itself has no such limit).
 * Per-map start tables (sim->start_offsets set, sim->env_layer set): the same draw inside the env's layer range,
 * k = min(floor(u * K_l), K_l - 1), agent i takes start_poses[start_l + (k - pose_gap*i) mod K_l]. */
int f110_autoreset(const f110_sim *sim, const double *start_poses, int32_t num_start, int32_t pose_gap,
                   uint64_t seed, uint64_t tick, void *stream);

/* One whole tick in three launches: f110_step + (env_level != 0) f110_env_post_step + (start_poses != NULL)
 * f110_autoreset, with the finalize kernel of the step, the lap logic and the auto-reset fused into one kernel (a
 * block owns whole envs; with more than 32 agents per env they run as separate launches).  Same results as calling
 * the three entry points in that order.  This is what a training loop / CUDA graph should replay. */
int f110_tick(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const double *actions,
              int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
              void *stream);
int f110_tick_ex(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                 const double *actions, int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap,
                 uint64_t seed, void *stream);

/* ---- action repeat: one action held for `repeat` ticks in one call ---- */
#define F110_MAX_REPEAT 64
/* Outputs and scratch of f110_tick_repeat, caller-owned device memory. */
typedef struct {
    uint8_t *done_any;                    /* [N] or NULL: OR of done[env] over the ticks of the call (overwritten, not accumulated) */
    int32_t *done_tick;                   /* [N] or NULL: index 0..repeat-1 of the first tick of the call that set done, -1 = none */
    uint32_t *list;                       /* [N*A] scratch: flat ids of the agents marched on an intermediate tick */
    uint32_t *list_count;                 /* [repeat] scratch, zeroed by the call on `stream` */
    unsigned long long *marched_agents;   /* [1] or NULL: += agents marched on intermediate ticks (measurement) */
} f110_repeat;

/* `repeat` whole ticks under one action (the "action repeat" / "frame skip" of a policy that runs slower than the physics):
 * what `repeat` calls of f110_tick_ex with the same arguments do, except that only the LAST tick's scans exist.
 *   - Enqueues everything on `stream`: no host synchronisation, no allocation, no global device state; capturable in a CUDA
 *     graph.  1 <= repeat <= F110_MAX_REPEAT; that, `rep` or its two scratch pointers NULL, done_any / done_tick without
 *     env_level, and everything f110_tick_ex rejects, return an error before anything is enqueued.
 *   - After the call every buffer of f110_sim except scans, march_cost / march_order / march_count and *lookup_counter holds,
 *     bit for bit, what the `repeat` plain ticks leave: state, steer FIFO and count (the FIFO sees the action once per tick),
 *     scan_pose, agent_poses, march_rec, wall_flag, collisions, collision_idx, time, lap arrays, toggles, done,
 *     checkpoint_done and tick_counter (advanced `repeat` times: the auto-reset draws and the noise stream are the plain
 *     ticks').  scans holds the last tick's scans, bit-identical to the plain run's; between launches it is unspecified.
 *   - An env that ends inside the call auto-resets on that tick (when start_poses is given) and keeps ticking in its new
 *     episode under the same action, as the plain ticks do; done is the last tick's, done_any / done_tick report the
 *     earlier ones.  repeat == 1 is f110_tick_ex plus done_any = done.
 *   - On ticks 0 .. repeat-2 the reference's only remaining use of the scan is the iTTC wall check (laser_models.py:188-217).
 *     An agent whose first distance-table lookup already exceeds the iTTC pre-test threshold of its speed cannot fire it and is
 *     not marched at all; the others are marched for the flag alone (csrc/march_ttc.cuh).  That path is taken when the tick's
 *     ray march is one of the lean kernels, the scan noise is off, beams->side_max is known and below max_range, and there
 *     are at most 32 agents per env; otherwise every tick of the call is the plain tick and the contract above still holds.
 *   - *lookup_counter counts the lookups actually performed.  The queue history (march_cost) is written by the last tick
 *     alone, so its queue is ordered by costs that are `repeat` ticks old; results never depend on the queue. */
int f110_tick_repeat(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                     const double *actions, int32_t repeat, const f110_repeat *rep, int32_t env_level,
                     const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed, void *stream);
/* Ticks first_tick .. first_tick + num_ticks - 1 of such a call, for a caller that has launches of its own to put between the
 * ticks (f110_track_progress after every tick): issuing the ranges of one call in order, with the same arguments, is the
 * call.  first_tick == 0 zeroes list_count.  F110_ERR_INVALID for a range outside [0, repeat). */
int f110_tick_repeat_ticks(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                           const double *actions, int32_t repeat, int32_t first_tick, int32_t num_ticks, const f110_repeat *rep,
                           int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
                           void *stream);

/* ---- static box obstacles (batch extension; csrc/obstacles.cuh) ---- */
/* An obstacle is a parked car of its env that has no sensor and never moves: an oriented box in env e, slot k.  With boxes of
 * the size of the agents' bodies (sim_length x sim_width, and the params length / width the opponent ray-cast uses), an env
 * with K boxes gives its A agents exactly what the reference gives agents 0..A-1 of a Simulator with A + K agents whose agents
 * A..A+K-1 start at the boxes' poses and receive the action (0, 0) every tick (pid then gives accl = sv = 0, and the RK4 step of
 * a resting car is the identity):
 *   - lidar: every agent's scan is clipped against every present box of its env by ray_cast_agents (laser_models.py:206-227,
 *     :282-346): the blocked-view window, get_range, min(scan, fp32(range)), from the same pose snapshot and with the yaw an
 *     iTTC hit zeroed (base_classes.py:246-249); scan noise is not applied to the box returns, as to opponent returns;
 *   - contact: GJK (collision_models.py:113-212) of the agent's body against the box sets collisions[a] = 1 and
 *     collision_idx[a] = max(.., A + k), the index a parked agent in slot A + k would get.  Contact zeroes no state (neither does
 *     opponent contact); an ego contact sets done and triggers the auto-reset like any other collision;
 *   - iTTC: boxes are invisible to it, as opponents are in the reference (check_ttc runs on the wall-only scan).
 * A slot that is inactive, or whose pose is not finite or whose length or width is not finite and > 0, is absent; with no slot
 * present every output equals the call without obstacles bit for bit.  The buffers are read afresh by every tick: a caller may
 * move boxes between ticks, also under a captured CUDA graph. */
#define F110_MAX_OBSTACLES 16
typedef struct {
    int32_t per_env;                /* K, 1 <= K <= F110_MAX_OBSTACLES */
    double *boxes;                  /* [N][K][5] (x, y, yaw, length, width), device */
    uint8_t *active;                /* [N][K] device, 0 = absent */
    int32_t *hit;                   /* [N*A] i32 device, or NULL: the highest slot the agent's body touches this tick, -1 = none */
    /* the respawn draw: when the auto-reset restarts an env, its boxes are redrawn from these candidates (NULL: boxes stay) */
    const double *candidates;       /* [C][5] device, rows of the layout of boxes */
    const int32_t *cand_offsets;    /* [num_cand_tables + 1] HOST memory (read at enqueue, as f110_sim.start_offsets), or NULL:
                                       an env on layer l draws from rows [cand_offsets[l], cand_offsets[l+1]); needs env_layer,
                                       offsets from 0 to C rising strictly, num_cand_tables == the map's num_layers
                                       (checked by the calls that take the map; f110_autoreset_obst and
                                       f110_obstacles_respawn have none: there an env whose layer has no table gets
                                       every slot inactive) */
    int32_t num_candidates;         /* C >= 1 */
    int32_t num_cand_tables;
    int32_t count_min, count_max;   /* the active count of a respawn, uniform in [count_min, count_max], 0 <= min <= max <= K */
    double clearance;               /* a drawn box whose centre is closer than this to an agent's new position stays inactive */
    uint64_t seed;
} f110_obstacles;

/* The entry points below take `obst`; NULL is exactly the call without _obst (f110_step_ex, f110_tick_ex,
 * f110_tick_repeat_ticks, f110_autoreset), which are these with NULL.  With obstacles the tail of a tick runs without its
 * env-level part, then k_obstacles (warp per agent: GJK against the env's boxes, then the scan clip) and, with env_level or
 * start_poses, k_env_tail_obst (thread per env: lap logic, repeat bookkeeping, auto-reset, respawn).  F110_ERR_INVALID before
 * anything is enqueued for K outside [1, 16], NULL boxes or active, count_min > count_max or count_max > K (or count_min < 0),
 * a clearance that is negative or not finite, candidate tables that do not match the map's layers, and what the call without
 * obstacles rejects.  No allocation, no host synchronisation: capturable in a CUDA graph. */
int f110_step_obst(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                   const double *actions, const f110_obstacles *obst, void *stream);
int f110_tick_obst(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                   const double *actions, int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap,
                   uint64_t seed, const f110_obstacles *obst, void *stream);
/* The intermediate ticks run the contact part of k_obstacles alone (their scans do not exist); the march and the marched
 * subset of the short path are unchanged, since the iTTC check does not see boxes. */
int f110_tick_repeat_ticks_obst(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                                const double *actions, int32_t repeat, int32_t first_tick, int32_t num_ticks, const f110_repeat *rep,
                                int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
                                const f110_obstacles *obst, void *stream);
/* f110_autoreset, and the respawn of the boxes of every env it restarts (with candidates). */
int f110_autoreset_obst(const f110_sim *sim, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
                        uint64_t tick, const f110_obstacles *obst, void *stream);
/* The respawn draw for the envs whose env_mask byte is non-zero (NULL: all), at tick counter `tick`, after the agents are placed
 * (a host reset).  For slot k of env e at tick t, with base = seed + 0xA0761D6478BD642F (t+1) + 0xE7037ED1A0B428DB (e+1) (mod
 * 2^64) and u(h) = (h >> 11) 2^-53:  the active count c = count_min + min(floor(u(mix64(base + 0x589965CC75374CC3)) S), S - 1),
 * S = count_max - count_min + 1; row j = min(floor(u(mix64(base + 0x8EBC6AF09C88C6E3 (k+1))) C_l), C_l - 1) of the env's table
 * is copied to the slot; the slot is active iff k < c and dx^2 + dy^2 >= clearance^2 for every agent of the env (positions from
 * sim->state).  mix64 is the finaliser of the auto-reset's start-pose draw.  The tick's auto-reset uses the tick counter it
 * draws its start poses with.  F110_ERR_INVALID also without candidates and with more than 32 agents per env. */
int f110_obstacles_respawn(const f110_sim *sim, const f110_obstacles *obst, const uint8_t *env_mask, uint64_t tick, void *stream);

/* ---- agents without a lidar (batch extension; csrc/march_ttc.cuh) ---- */
/* A lidar mask says which agent slots have a lidar: bit i covers slot i in every env.  A sensorless agent is simulated exactly
 * as one with a lidar -- dynamics, steer FIFO, the iTTC wall check on its wall-only scan (state[3:] zeroed on a hit), GJK,
 * collisions / collision_idx, lap logic, done, auto-reset and obstacle contact -- and the other agents still see its body in
 * their scans; only its own scan is never computed.
 * Short path: when the tick's ray march is a lean kernel, the scan noise is off, beams->side_max is known and below max_range,
 * dt_min_positive > eps and A <= 32 (the conditions of the short path of f110_tick_repeat), the march queue holds the items of
 * the slots that have a lidar only, the sensorless agents a wall could stop are listed and marched for the iTTC flag alone, and
 * no kernel writes a sensorless agent's scan row.  Every buffer of f110_sim then equals, bit for bit, what the call without a
 * mask leaves, except the scan rows of sensorless agents, march_cost / march_order / march_count and *lookup_counter; the scans
 * of the agents that have a lidar are bit-identical, opponent ray-cast and obstacle clip included.
 * Full path: otherwise the mask is ignored and the call equals the call without it, scans included. */
#define F110_LIDAR_ALL 0xFFFFFFFFu
typedef struct {
    uint32_t mask;                  /* bit i: slot i has a lidar; F110_LIDAR_ALL = every slot (any A) */
    uint32_t *list;                 /* [N*A] device scratch: sensorless agents listed for the iTTC-only march */
    uint32_t *list_count;           /* [1] device scratch, zeroed by the call on `stream` */
    unsigned long long *listed;     /* [1] or NULL: += sensorless agents listed (measurement) */
} f110_lidar;

/* The _obst calls with a lidar mask.  lidar == NULL or mask == F110_LIDAR_ALL is exactly the _obst call.  F110_ERR_INVALID
 * before anything is enqueued for any other mask with more than 32 agents per env, a bit set at or above num_agents, and NULL
 * list or list_count with a mask other than F110_LIDAR_ALL (on either path).  f110_tick_repeat_ticks_lidar applies the mask
 * to the last tick of the call; the ticks before it run as in f110_tick_repeat_ticks_obst.  No allocation, no host
 * synchronisation: capturable in a CUDA graph. */
int f110_step_lidar(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                    const double *actions, const f110_obstacles *obst, const f110_lidar *lidar, void *stream);
int f110_tick_lidar(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                    const double *actions, int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap,
                    uint64_t seed, const f110_obstacles *obst, const f110_lidar *lidar, void *stream);
int f110_tick_repeat_ticks_lidar(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables,
                                 const f110_beams *beams, const double *actions, int32_t repeat, int32_t first_tick,
                                 int32_t num_ticks, const f110_repeat *rep, int32_t env_level, const double *start_poses,
                                 int32_t num_start, int32_t pose_gap, uint64_t seed, const f110_obstacles *obst,
                                 const f110_lidar *lidar, void *stream);

/* Same tick through HOST buffers: copies actions H2D, runs f110_step (+ f110_env_post_step when the
 * lap arrays are bound), copies the observation D2H and synchronises the stream.
 * Any output pointer may be NULL to skip that copy.  Host buffers should be pinned. */
typedef struct {
    float *scans;           /* [N*A][B] */
    double *state;          /* [7][N*A] */
    double *collisions;     /* [N*A] */
    uint8_t *done;          /* [N] */
    double *lap_times, *lap_counts;   /* [N*A] */
    uint8_t *scans_u24;     /* [N*A][B][3] optional narrow scan block for PCIe-bound host consumers (f110_step_host_async only,
                               used when `scans` is NULL): each range as 24-bit fixed point, little endian, value = q * 2^-19 m
                               (step 1.9e-6 m = the fp32 scan's own resolution at 30 m; |error| <= 9.6e-7 m; a noisy range
                               below 0 clamps to 0).  3 bytes per beam instead of 4: see f110_pack_scans_u24. */
} f110_host_obs;
int f110_step_host(const f110_sim *sim, const f110_map *map, const f110_beams *beams,
                   const double *actions_host, double *actions_dev_scratch, const f110_host_obs *out,
                   void *stream);

/* Pipelined variant for host-side consumers: the tick runs on `compute_stream`, its observation is
 * snapshotted into the DEVICE staging buffers `stage` (same layout as f110_host_obs), and the D2H copies
 * into `out` run on `copy_stream`, so that the copy of tick t overlaps the compute of tick t+1.  No host
 * synchronisation: the caller alternates between two (stage, out, event) sets and, before reusing a set or
 * reading its host buffers, waits for `ev_copy_done` (cudaEventSynchronize).  `ev_tick_done` and
 * `ev_copy_done` are cudaEvent_t created by the caller.  Before overwriting `stage` the compute stream
 * waits for the previous copy out of it (the event's last record). */
int f110_step_host_async(const f110_sim *sim, const f110_map *map, const f110_beams *beams,
                         const double *actions_host, double *actions_dev_scratch, const f110_host_obs *stage,
                         const f110_host_obs *out, void *compute_stream, void *copy_stream, void *ev_tick_done,
                         void *ev_copy_done);
int f110_step_host_async_ex(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables,
                            const f110_beams *beams, const double *actions_host, double *actions_dev_scratch,
                            const f110_host_obs *stage, const f110_host_obs *out, void *compute_stream, void *copy_stream,
                            void *ev_tick_done, void *ev_copy_done);

/* scans [count] fp32 (device) -> out [count][3] bytes (device): q = round(range * 2^19) clamped to [0, 2^24-1], little endian.
 * No reference counterpart (the reference hands numpy arrays to a policy in the same process); batch extension for host-side
 * consumers behind PCIe.  Decode: (b0 | b1 << 8 | b2 << 16) * 2^-19.
 * The clamp: every range at or above 32 - 2^-19 m decodes to 32 - 2^-19 m, so the block only holds scans of a map whose
 * max_range plus the noise head-room stays below 32 m (the Python pipeline refuses any other map). */
int f110_pack_scans_u24(const float *scans, int64_t count, uint8_t *out, void *stream);

/* ---- standalone kernels (unit-parity surface; device pointers) ------------------------------- */

/* ScanSimulator2D.scan without noise / get_scan (laser_models.py:148-186, 429-454): M poses -> [M][B].
 * Two deliberate deviations where the reference reads outside its arrays (DESIGN.md §4): a first LUT index of
 * exactly theta_dis reads entry 0, and a cell index that rounds up to width or height reads dt[-1,-1].
 * One map only: on a same-size [L][H][W] stack it scans layer 0 for every pose, and a canvas stack (layer_geom,
 * layer_res or layer_rot) returns F110_ERR_INVALID.  f110_scan_layers scans each pose on a layer of its own, on any map. */
int f110_scan(const f110_map *map, const f110_beams *beams, const double *poses /* [M][3] */, int32_t M,
              float *out_f32 /* [M][B] or NULL */, double *out_f64 /* [M][B] or NULL */,
              unsigned long long *lookup_counter /* [1] or NULL */, void *stream);
/* ScanSimulator2D.scan without noise (laser_models.py:148-186, 429-454) for M poses, each on its own layer of `map`.
 * Batch extension.  poses [M][3] device; layer_ids [M] i32 device, or NULL when the map has one layer.
 * Accepts every map f110_step accepts: one map (rotated origin or not, any resolution), a same-size [L][H][W] stack, and a
 * canvas stack in cell units or metres, with layer_res or layer_rot.  Every beam equals the reference's get_scan on that
 * pose's own map in fp64, with the two deviations of f110_scan; *lookup_counter (optional) gets the reference's lookup
 * count added.  A layer id outside [0, num_layers) (checked on the device) gives NaN for every beam of its pose and no
 * lookups.  F110_ERR_INVALID before anything is enqueued: the table rules of f110_step, layer_ids NULL on a map of more
 * than one layer, sincos2 NULL, dt_min_positive <= eps, fov >= 2 pi, or M * num_beams >= 2^32; F110_ERR_NO_MAP without a
 * table.  No global state and no host synchronisation: calls on different streams may run at once.  Kernel k_scan_lean
 * (csrc/scan_lean.cuh), one warp per 32 beams of one pose. */
int f110_scan_layers(const f110_map *map, const f110_beams *beams, const double *poses, const int32_t *layer_ids, int32_t M,
                     float *out_f32 /* [M][B] or NULL */, double *out_f64 /* [M][B] or NULL */,
                     unsigned long long *lookup_counter /* [1] or NULL */, void *stream);
/* Top-down views of the simulation (batch extension; the reference draws its pyglet window in rendering.py instead): V views
 * of height x width pixels, row 0 at the top, metres_per_pixel each, view k following agent agent_ids[k] (flat index, i32
 * device) from its state pose (x, y, yaw), centred forward_offset metres ahead of it, with its heading up (heading_up != 0)
 * or world-aligned.  out [V][height][width] u8 (device) gets one class per pixel centre: 0 off-map, 1 free, 2 wall (dt == 0,
 * what the lidar sees), 3 another agent of the env, 4 the followed agent (cars are the get_vertices quads of check_collision,
 * base_classes.py:549); 255 fills a view whose agent id is outside [0, N*A), whose env layer is outside [0, num_layers) or
 * whose pose is not finite.  The map class is xy_2_rc (laser_models.py:55-104) on the env's layer, with the deviation of
 * f110_scan; the exact operation order is in csrc/render.cuh.  Accepts every map f110_step accepts (a stack needs
 * sim->env_layer).  F110_ERR_INVALID before anything is enqueued: a NULL pointer, V < 1, height or width outside
 * [1, 8192], metres_per_pixel not finite or <= 0, forward_offset not finite, more than 64 agents per env, a stack without
 * env_layer or the table rules of f110_scan_layers; F110_ERR_NO_MAP without a table.  Writes nothing but `out`; no global
 * state, no allocation and no host synchronisation (graph-capturable; calls on two streams may run at once). */
int f110_render_views(const f110_sim *sim, const f110_map *map, const int32_t *agent_ids, int32_t V, int32_t height,
                      int32_t width, double metres_per_pixel, double forward_offset, int32_t heading_up, uint8_t *out,
                      void *stream);
/* f110_render_views with the env's static box obstacles (f110_obstacles) drawn as class 5: every present slot is the quad
 * get_vertices_cs(x, y, cos, sin, length, width) with (sin, cos) = sincos(yaw), tested as the car quads; priority
 * 4 > 3 > 5 > 2 > 1 / 0.  obst == NULL is f110_render_views; F110_ERR_INVALID for the structs the _obst tick entry points
 * reject (the candidate tables are not read). */
int f110_render_views_obst(const f110_sim *sim, const f110_map *map, const f110_obstacles *obst, const int32_t *agent_ids, int32_t V,
                           int32_t height, int32_t width, double metres_per_pixel, double forward_offset, int32_t heading_up,
                           uint8_t *out, void *stream);
/* vehicle_dynamics_st (dynamic_models.py:123-176): x [M][7], u [M][2], params [18] -> f [M][7]. */
int f110_vehicle_dynamics_st(const double *x, const double *u, const double *params, int32_t M, double *f,
                             void *stream);
/* vehicle_dynamics_ks (dynamic_models.py:90-121): x [M][5] (x, y, steer, v, yaw), u [M][2], params [18] -> f [M][5]. */
int f110_vehicle_dynamics_ks(const double *x, const double *u, const double *params, int32_t M, double *f,
                             void *stream);
/* pid (dynamic_models.py:178-221): in [M][4] = (speed, steer, current_speed, current_steer) -> out [M][2] = (accl, sv). */
int f110_pid(const double *in, const double *params, int32_t M, double *out, void *stream);
/* get_vertices (collision_models.py:237-260): poses [M][3] -> [M][4][2] (rl, rr, fr, fl). */
int f110_get_vertices(const double *poses, double length, double width, int32_t M, double *out, void *stream);
/* collision (GJK, collision_models.py:113-182): va, vb [M][4][2] -> out [M] 0/1. */
int f110_collision(const double *va, const double *vb, int32_t M, int32_t *out, void *stream);
/* collision_multiple (collision_models.py:184-212): verts [M][n][4][2] -> collisions [M][n], collision_idx [M][n]. */
int f110_collision_multiple(const double *verts, int32_t M, int32_t n, double *collisions, double *collision_idx,
                            void *stream);
/* check_ttc_jit (laser_models.py:188-217): scans [M][B] fp64, vel [M] -> out [M] 0/1. */
int f110_check_ttc(const f110_beams *beams, const double *scans, const double *vel, double ttc_thresh, int32_t M,
                   int32_t *out, void *stream);
/* ray_cast (laser_models.py:318-346): pose [M][3], opponent vertices [M][4][2], scans [M][B] fp32 modified in
 * place; window [M][2] (min_ind, max_ind of get_blocked_view_indices :282-315) optional. */
int f110_ray_cast(const f110_beams *beams, const double *poses, const double *opp_vertices, int32_t M,
                  float *scans, int32_t *window, void *stream);
/* Seeded scan noise (laser_models.py:450-452; N(0, std^2) per beam).  Counter-based Philox-4x32 +
 * Box-Muller; statistical, not bit, parity with numpy's PCG64 stream. */
int f110_scan_noise(float *scans, int64_t count, double std_dev, uint64_t seed, uint64_t offset, void *stream);

/* Batched pure-pursuit policy (reference examples/waypoint_follow.py:15-217, PurePursuitPlanner.plan):
 * waypoint columns wx, wy, wv [num_waypoints] and poses pose_x/y/theta [M] (device) -> actions_out [M][2] =
 * (steering angle, speed), the layout f110_step consumes.  max_reacquire is 20.0 in the reference (:154). */
int f110_pure_pursuit(const double *wx, const double *wy, const double *wv, int32_t num_waypoints, const double *pose_x,
                      const double *pose_y, const double *pose_theta, int32_t M, double lookahead_distance, double vgain,
                      double wheelbase, double max_reacquire, double *actions_out, void *stream);

/* The same policy over several waypoint tables (one per track of a multi-map batch; batch extension, no reference
 * counterpart): the tables are concatenated in wx/wy/wv, table t occupies rows [table_start[t], table_start[t+1])
 * (table_start [num_tables+1] i32, device, every table >= 2 rows) and pose a follows table pose_table[a]
 * (i32 [M], device, values in [0, num_tables) -- not range-checked on the device). */
int f110_pure_pursuit_tables(const double *wx, const double *wy, const double *wv, const int32_t *table_start,
                             int32_t num_tables, const int32_t *pose_table, const double *pose_x, const double *pose_y,
                             const double *pose_theta, int32_t M, double lookahead_distance, double vgain, double wheelbase,
                             double max_reacquire, double *actions_out, void *stream);

/* ---- centerline progress (batch extension: the reference's reward is the constant timestep, f110_env.py:263-304) ---- */

/* Closed centerlines, one table per map layer.  Table t holds segments [table_start[t], table_start[t+1]) of `segments`; segment
 * i of a table of n points runs from point i to point (i + 1) mod n, and its record is 8 fp64 values (x_i, y_i, dx, dy, l2,
 * s_i, len_i, h_i): dx, dy = next point - point, l2 = dx*dx + dy*dy, len_i = sqrt(l2), s_i = arc length at point i
 * (np.cumsum of len, 0 for point 0), h_i = atan2(dy, dx).  A table's length L is s_{n-1} + len_{n-1}. */
typedef struct {
    int32_t num_tables;
    int32_t min_segments;           /* host copy: the fewest segments of any table (>= 3) */
    const int32_t *table_start;     /* [num_tables + 1] i32, device */
    const double *segments;         /* [table_start[num_tables]][8] fp64, device */
} f110_track;

/* Per-agent tracker state and outputs, [N*A] device buffers each (flat agent index). */
typedef struct {
    int32_t *seg;                   /* state: segment of the last projection, -1 = not acquired */
    double *s;                      /* arc length of the last projection (also the previous s of the next update) */
    double *d;                      /* signed lateral offset, positive left of the direction of travel */
    double *heading_error;          /* yaw - h_i wrapped to [-pi, pi) */
    double *progress;               /* arc length travelled since the agent was acquired */
    double *delta;                  /* progress made by the last update */
    int32_t back, fwd;              /* the tracking window: segments seg - back .. seg + fwd (1 <= back + fwd + 1 <= 1024) */
    double reacquire_dist;          /* a window whose best distance exceeds this falls back to the global projection */
} f110_progress;

/* nearest_point_on_trajectory (reference examples/waypoint_follow.py:16-47) on the closed table vstack(T, T[0]) in its operation
 * order, fp64, the first minimum by segment index; its np.dot is BLAS ddot, dot = fma(py - y, dy, (px - x) * dx), and no other
 * operation is fused (csrc/progress.cuh): poses [M][3] (x, y, yaw, device), table_ids [M] i32 (device), or
 * NULL with a single table -> out [M][5] = (seg, t, d, s, e): segment, t in [0, 1], signed distance (+ left of travel),
 * s = s_i + t * len_i, heading error yaw - h_i wrapped by e - 2pi * floor((e + pi) / 2pi).  A non-finite pose or a table id
 * outside [0, num_tables) gives a NaN row.  F110_ERR_INVALID before anything is enqueued: NULL pointers, M < 1, no table,
 * min_segments < 3, table_ids NULL with more than one table.  No global state, allocation or host synchronisation. */
int f110_track_project(const f110_track *track, const double *poses, const int32_t *table_ids, int32_t M, double *out,
                       void *stream);

/* One update of every agent's progress along its map's centerline (table env_layer[env], or table 0 when sim->env_layer is
 * NULL), from the pose in sim->state.  Acquire when seg < 0 or sim->steer_cnt == 0 (the agent was reset since its last step:
 * f110_reset and the auto-reset zero it, every step increments it): the projection of f110_track_project, progress = delta = 0.
 * Otherwise track: the first minimum over the window k = 0 .. back + fwd, segment (seg - back + k) mod n, in window order
 * (clipped to n segments); a best distance above reacquire_dist falls back to the global projection and keeps the progress;
 * delta = s - s_prev, minus L if above L/2, plus L if below -L/2, and progress += delta.  On the tick that auto-resets an env
 * the update already sees the new episode, so that tick's delta is 0 and the crash tick's last partial delta is lost.
 * A non-finite pose or a bad table id gives NaN outputs and seg = -1.  F110_ERR_INVALID before anything is enqueued: NULL
 * pointers, no table, min_segments < 3, a bad window, reacquire_dist not finite or <= 0.  No global state, allocation or
 * host synchronisation: capturable in a CUDA graph after f110_tick.  Kernel k_track_progress (csrc/progress.cuh). */
int f110_track_progress(const f110_sim *sim, const f110_track *track, f110_progress *progress, void *stream);

/* f110_track_progress, then delta_sum[a] = (restart ? 0 : delta_sum[a]) + progress->delta[a] for every agent (delta_sum [N*A]
 * fp64, device): the progress of a policy step that spans several ticks, summed in tick order (restart != 0 on its first tick).
 * F110_ERR_INVALID for a NULL delta_sum and for what f110_track_progress rejects. */
int f110_track_progress_sum(const f110_sim *sim, const f110_track *track, f110_progress *progress, double *delta_sum,
                            int32_t restart, void *stream);

/* Exact Euclidean distance transform on the device (load-time; reference laser_models.py:40-53 get_dt =
 * resolution * scipy.ndimage.distance_transform_edt(bitmap)): occupied [H][W] u8 (1 where the thresholded image
 * is 0), scratch [H][W] i32, dt_out [H][W] f64 = resolution * sqrt(k) with k the exact squared cell distance
 * (optionally written to k_out [H][W] i64).  Bit-identical to the scipy table. */
int f110_edt(const uint8_t *occupied, int32_t height, int32_t width, double resolution, int32_t *scratch, double *dt_out,
             int64_t *k_out, void *stream);

/* Walls of a generated track (reference unittest/random_trackgen.py:156-165 shapely buffer(+-WIDTH) of the closed
 * centerline, :167-178 the two offset curves drawn 3 pt wide): segments [num_segments][5] (device) = ax, ay, bx-ax,
 * by-ay, 1/|b-a|^2 of the closed centerline in PIXEL units (pixel (r, c) has its centre at (c+0.5, r+0.5), row 0 =
 * bottom of the map like the flipped image of laser_models.py:399); occupied [H][W] u8 = 1 where the pixel centre's
 * distance d to the centerline satisfies wall_inner <= d <= wall_outer (the input f110_edt takes); dist2_out
 * (optional) [H][W] f64 = d^2 in pixels^2 (d < wall_inner = on the track). */
int f110_rasterize_track(const double *segments, int32_t num_segments, double wall_inner, double wall_outer, int32_t height,
                          int32_t width, uint8_t *occupied, double *dist2_out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* F110_B200_H */
