/*
 * f110_mppi.h — scored rollouts and a device MPPI planner (libf110_b200.so, ABI v6): the cost of every predicted future along
 * the map's centerline, computed inside f110_predict's rollout, and the sample / update steps of model-predictive path
 * integral control on top of it.  An addition to the ABI of f110_b200.h and f110_predict.h, whose conventions it follows;
 * kept in a header of its own so that the headers it builds on keep their entry-point sets.
 */
#ifndef F110_MPPI_H
#define F110_MPPI_H

#include "f110_predict.h"
#include "f110_episodes.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- scored rollouts (batch extension; csrc/predict.cuh k_scored_rollout, k_scored_acquire) ---- */
/* The weights, tracker settings, optional input, output and scratch of f110_predict_scored.  cost[m][k], fp64, accumulated in
 * step order h = 0 .. H-1 and within a step in the order written:
 *   c = sum_h [ w_lat * d_h^2 + w_head * e_h^2 + w_clear * max(0, clear_min - clr_h)^2
 *               + w_dsteer * (u_h.steer - u_{h-1}.steer)^2 + w_dspeed * (u_h.speed - u_{h-1}.speed)^2 ]
 *       - w_prog * P_{H-1} + (wall_step >= 0 ? w_wall : 0)
 * each term as c = c + w * (x * x) (the library builds with -fmad=false: every operation rounds on its own).
 *   - d_h, e_h: the signed lateral offset (+ left of travel) and heading error of the state after step h, from the tracker below;
 *   - P_{H-1}: the tracker's progress after the last step (metres along the centerline, the deltas of f110_track_progress);
 *   - clr_h: the first distance-transform lookup in metres at step h's scan pose, fp64 (the value clearance rounds to fp32);
 *   - u_h = actions[m][k][h]; u_{-1} = prev_action[m], or, with prev_action NULL, the two rate terms of h = 0 are 0.
 * The tracker is f110_track_progress's, per sample: one acquiring update at the source agent's pose (k_scored_acquire, a warp
 * per m: f110_track_project's global projection on its layer's table, progress 0), then one tracking update after every step
 * (the window seg - back .. seg + fwd in window order, clipped to n segments; a best distance above reacquire_dist, or none,
 * falls back to the global projection; delta unwrapped by half a lap), in one thread with track_search's per-segment
 * statements.  Fill back, fwd and reacquire_dist from the f110_progress the simulator tracks with, so that the sequence is the
 * one f110_track_progress would run over the predicted states.
 * NaN propagates: an agent id outside [0, N*A), a non-finite source pose or a bad table id (seg0 = -1), and a step whose state
 * is not finite or whose tracker finds no segment make the sample's cost NaN. */
typedef struct {
    double w_lat, w_head, w_clear, w_dsteer, w_dspeed, w_prog, w_wall;   /* finite, >= 0 */
    double clear_min;               /* metres, finite */
    int32_t back, fwd;              /* the tracking window (1 <= back + fwd + 1 <= 1024) */
    double reacquire_dist;          /* finite, > 0 */
    const double *prev_action;      /* [M][2] device (steer, speed), or NULL */
    double *cost;                   /* [M][K] device: the output */
    int32_t *seg0;                  /* [M] device scratch: the source pose's segment (-1: not acquired) */
    double *s0;                     /* [M] device scratch: the source pose's arc length */
} f110_cost;

/* f110_predict, and cost->cost.  final_state, wall_step, states and clearance are bit-identical to f110_predict's on the same
 * inputs (the rollout is k_predict's; the cost is computed beside it).  Two launches: k_scored_acquire, then the rollout.
 * F110_ERR_INVALID before anything is enqueued for what f110_predict refuses; track or cost NULL; cost->cost, seg0 or s0 NULL;
 * track->num_tables other than the map's layer count (1 for a single map), no table or min_segments < 3; a bad window; a
 * weight that is not finite or is negative, a non-finite clear_min; reacquire_dist not finite or <= 0.  No allocation, no
 * global state, no host synchronisation: capturable in a CUDA graph. */
int f110_predict_scored(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                        const f110_track *track, const f110_predict_args *args, const f110_cost *cost, void *stream);

/* ---- MPPI (batch extension; csrc/mppi.cuh) ---- */
/* The planner state of M agents over a horizon of H steps with K samples per agent.  Device buffers: nominal, iteration,
 * no_finite; the rest are values read when a call is enqueued (a captured graph keeps them). */
typedef struct {
    int32_t M, K, H;                /* 1 <= M, 2 <= K <= F110_MPPI_MAX_K, 1 <= H <= F110_MPPI_MAX_H, M * K * H < 2^31 */
    const int32_t *agent_ids;       /* [M] device: the flat agent id e*A + slot each planner row drives */
    double *nominal;                /* [M][H][2] device: the nominal action sequence (steer, speed) */
    int64_t *iteration;             /* [1] device: the noise counter, incremented by every f110_mppi_update */
    int32_t *no_finite;             /* [M] device: updates in which no sample of the agent had a finite cost */
    double sigma_steer, sigma_speed;        /* noise std, finite, >= 0 */
    double steer_lo, steer_hi, speed_lo, speed_hi;   /* clamp bounds, finite, lo <= hi */
    double lambda;                  /* the temperature, finite, > 0 */
    uint64_t seed;
} f110_mppi;

#define F110_MPPI_MAX_K 4096
#define F110_MPPI_MAX_H 1000     /* with F110_MPPI_MAX_K: f110_mppi_update's shared memory within 48 KiB */

/* actions[m][k][h][c] = clamp(nominal[m][h][c] + sigma_c * z, lo_c, hi_c), c = 0 steer, 1 speed, a thread per (m, k, h);
 * z = normal_sample(seed, 2^63 | iteration, ((m * K + k) * H + h) * 2 + c), the Philox stream of the scan noise (csrc/lidar.cuh)
 * under stream numbers with the top bit set, which neither the per-tick scan noise (the tick counter) nor f110_scan_noise
 * (2^32 - 1) uses.  Sample k = 0 is the clamped nominal without noise.
 * Before sampling, the nominal of an agent that restarted since the planner's last update is reset to (0, 0): an agent whose
 * steer_cnt is 0 (f110_reset, the auto-reset of f110_tick*), or, with ep given, whose env has terminated or truncated set (the
 * episode restart, whose zero-action tick leaves steer_cnt at 1).  Call it once per tick: the episode flags hold until the next
 * episode tick.  An agent id outside [0, N*A) is never reset.  F110_ERR_INVALID before anything is enqueued for NULL pointers
 * (ep may be NULL; its terminated / truncated may not), sizes or values outside the ranges above. */
int f110_mppi_sample(const f110_sim *sim, const f110_mppi *mppi, const f110_episodes *ep, double *actions, void *stream);

/* A block per agent m, over the samples' actions [M][K][H][2] and costs [M][K] (f110_predict_scored):
 *   beta = min over k of the finite costs;  w_k = exp(-(c_k - beta) / lambda), 0 for a cost that is NaN or infinite;
 *   U[h] = sum_k w_k * A[k][h] / sum_k w_k, both sums in k order (repeated calls are bit-identical);
 *   action_out[agent_ids[m]] = U[0] (rows [num_rows][2] fp64 device; an id outside [0, num_rows) writes nothing, and every
 *   other row is left alone, so several planners and other controllers can fill one action tensor);
 *   nominal[h] = U[h + 1] for h < H - 1, nominal[H - 1] = U[H - 1].
 * No finite cost: U is the nominal clamped to the bounds, shifted the same way, and no_finite[m] += 1.  weights [M][K] and
 * argmin [M] (the first k of the smallest finite cost, -1 for none) are optional outputs.  Then iteration += 1, so that the
 * next sample draws fresh noise.  F110_ERR_INVALID before anything is enqueued for NULL pointers (weights and argmin may be),
 * num_rows < 1, and what f110_mppi_sample refuses of the planner. */
int f110_mppi_update(const f110_mppi *mppi, const double *actions, const double *cost, double *action_out, int32_t num_rows,
                     double *weights, int32_t *argmin, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* F110_MPPI_H */
