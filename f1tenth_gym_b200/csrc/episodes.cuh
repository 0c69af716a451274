// episodes.cuh — the episode tick (f110_tick_episodes, include/f110_b200.h): every env whose episode ends on a tick keeps its
// final observation and restarts as F110Env.reset does -- the placement, then one zero-action tick of that env alone.
// Included by f110_b200.cu after obstacles.cuh, whose device functions it reuses.
//
// After the plain tick (f110_tick_lidar with env_level and without auto-reset):
//   k_episode_end        thread per env      counters, terminated / truncated / length; for an ended env the final_* copies,
//                                            the start-pose draw of the auto-reset, the respawn draw, track_seg = -1, and its
//                                            id appended to the restart list (one atomic per ended env)
//   k_episode_dyn        thread per agent    the listed envs' agents: k_dynamics' per-agent statements under the action (0, 0)
//   k_restart_march      fixed grid          a warp per 32-beam item of a listed agent: k_march_ttc's beam arithmetic marched
//                                            to completion, the noise of counter t | 2^63, the tick's iTTC predicate, and for
//                                            an agent that has a lidar the crash scan to final_scans, then the new range
//   k_episode_cast       warp per ego        the opponent ray-cast of the listed egos that have a lidar (k_lidar_cast's body)
//   k_episode_tail       thread per env      wall-hit zeroing, GJK and collisions of the listed envs' agents, then the lap
//                                            logic of the zero tick; `done` keeps the plain tick's value
//   k_episode_obstacles  warp per agent      with obstacles: box contact and the scan clip (k_obstacles' body)
// Every kernel of the restart reads the list and its count on the device; the grids are sized for every env.  An env's
// results never depend on its position in the list.
#pragma once

namespace f110 {

struct EpisodeK {
    int32_t *ticks, *length;
    uint8_t *terminated, *truncated;
    double *final_state, *final_collisions, *final_lap_times, *final_lap_counts;
    int32_t *final_collision_idx;
    uint32_t *list, *count;
    int32_t *track_seg;          // [N*A] or NULL
    int max_ticks;
};

// The start-pose draw and placement of autoreset_one for env `env`, unconditionally: a copy of its statements, kept apart from
// it because calling this from autoreset_one would change the code of the tuned tails.
__device__ __forceinline__ void episode_place(const f110_sim &s, int env, const AutoResetArgs &ar) {
    const int A = s.num_agents, NA = s.num_envs * s.num_agents;
    const double *__restrict__ start_poses = ar.start_poses;
    int num_start = ar.num_start;
    const int pose_gap = ar.pose_gap;
    if (ar.num_tables) {         // the start table of the env's own map: rows [start_off[l], start_off[l + 1])
        const int l = s.env_layer[env];
        start_poses += 3 * (size_t)ar.start_off[l];
        num_start = ar.start_off[l + 1] - ar.start_off[l];
    }
    const uint64_t tick = s.tick_counter ? (uint64_t)*s.tick_counter : ar.tick_host;
    uint64_t h = mix64(ar.seed + 0x9E3779B97F4A7C15ull * (tick + 1) + 0xD1B54A32D192ED03ull * (uint64_t)(env + 1));
    int k = (int)((double)(h >> 11) * (1.0 / 9007199254740992.0) * num_start);
    if (k >= num_start) k = num_start - 1;
    double pose3[3 * 32];
    for (int i = 0; i < A; i++) {
        const int kk = ((k - pose_gap * i) % num_start + num_start) % num_start;
        const size_t a = (size_t)env * A + i;
        const double x = start_poses[3 * kk], y = start_poses[3 * kk + 1], th = start_poses[3 * kk + 2];
        pose3[3 * i] = x; pose3[3 * i + 1] = y; pose3[3 * i + 2] = th;
#pragma unroll
        for (int q = 0; q < 7; q++) s.state[(size_t)q * NA + a] = 0.0;
        s.state[a] = x;
        s.state[(size_t)NA + a] = y;
        s.state[(size_t)4 * NA + a] = th;
        s.steer_cnt[a] = 0;
        s.steer_buf[a] = 0.0;
        s.steer_buf[(size_t)NA + a] = 0.0;
        s.wall_flag[a] = 0;
        mark_march_cost_unknown(s, a);
    }
    env_counters_reset(s, env, pose3, false);
}

__global__ void k_episode_end(f110_sim s, AutoResetArgs ar, EpisodeK ep, ObstDraw d) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= s.num_envs) return;
    const int A = s.num_agents, NA = s.num_envs * A;
    const int t = ep.ticks[env] + 1;
    const bool term = s.done[env] != 0;
    const bool trunc = !term && ep.max_ticks > 0 && t >= ep.max_ticks;
    ep.terminated[env] = term ? 1 : 0;
    ep.truncated[env] = trunc ? 1 : 0;
    if (!term && !trunc) {
        ep.ticks[env] = t;
        return;
    }
    ep.length[env] = t;
    ep.ticks[env] = 0;            // the zero-action tick does not count, as F110Env.reset's does not
    for (int i = 0; i < A; i++) {
        const size_t a = (size_t)env * A + i;
#pragma unroll
        for (int q = 0; q < 7; q++) ep.final_state[(size_t)q * NA + a] = s.state[(size_t)q * NA + a];
        ep.final_collisions[a] = s.collisions[a];
        ep.final_collision_idx[a] = s.collision_idx[a];
        ep.final_lap_times[a] = s.lap_times[a];
        ep.final_lap_counts[a] = s.lap_counts[a];
        if (ep.track_seg) ep.track_seg[a] = -1;
    }
    episode_place(s, env, ar);
    if (d.cand) obst_respawn_one(s, env, d, s.tick_counter ? (uint64_t)*s.tick_counter : ar.tick_host);
    ep.list[atomicAdd(ep.count, 1u)] = (uint32_t)env;
}

// the agents of the listed envs, thread per agent: k_dynamics' per-agent statements under the action (0, 0), copied from it so
// that k_dynamics keeps its code; the tick counter stays
__global__ void __launch_bounds__(128) k_episode_dyn(f110_sim s, double fov, double theta_dis_f, FirstLookup fl,
                                                     const uint32_t *__restrict__ list, const uint32_t *__restrict__ count) {
    const int NA = s.num_envs * s.num_agents;
    const unsigned t = blockIdx.x * blockDim.x + threadIdx.x, k = t / (unsigned)s.num_agents;
    if (k >= *count) return;
    const int a = (int)(list[k] * (unsigned)s.num_agents + (t - k * (unsigned)s.num_agents));
    const double *p = s.params + (size_t)(s.params_per_env ? a : a % s.num_agents) * F110_NPARAM;
    double st[7];
#pragma unroll
    for (int k = 0; k < 7; k++) st[k] = s.state[(size_t)k * NA + a];
    // steering delay FIFO (base_classes.py:270-278): depth 2, zeros until two commands are queued
    const double raw_steer = 0.0, speed = 0.0;
    int cnt = s.steer_cnt[a];
    double b0 = s.steer_buf[a], b1 = s.steer_buf[(size_t)NA + a];
    double steer = (cnt < 2) ? 0. : b1;
    s.steer_buf[(size_t)NA + a] = b0;
    s.steer_buf[a] = raw_steer;
    if (cnt < 2) s.steer_cnt[a] = cnt + 1;

    integrate_tick(st, steer, speed, p, s.timestep, s.integrator);

#pragma unroll
    for (int k = 0; k < 7; k++) s.state[(size_t)k * NA + a] = st[k];
    // scan pose (base_classes.py:406-409) and the first beam's LUT index (laser_models.py:167-172)
    double sx = st[0], sy = st[1];
    if (s.lidar_dist != 0.0) {
        sx = st[0] + s.lidar_dist * cos(st[4]);
        sy = st[1] + s.lidar_dist * sin(st[4]);
    }
    // slot 2: on fast-path maps the DT value of the scan-pose cell in cell units — the first lookup of every
    // beam of this agent (laser_models.py:129), done once here; otherwise the yaw
    double slot2 = st[4];
    const size_t lo = fl.env_layer ? (size_t)fl.env_layer[a / s.num_agents] * (size_t)fl.layer_stride : (size_t)0;
    if (fl.layer_geom) {
        // canvas stack: the env's own origin and extent; the canvas cells beyond the layer hold its dt[-1,-1], so a column
        // (row) index up to the canvas width (height) reads what the reference reads off that map
        const double *__restrict__ g = fl.layer_geom + 6 * (size_t)fl.env_layer[a / s.num_agents];
        if (!fl.metres) {
            CellConsts k;
            k.ox = g[0] * fl.inv_res; k.oy = g[1] * fl.inv_res; k.eps = 0; k.tmax = 0;
            k.width = fl.width; k.height = fl.height; k.last = fl.last;
            slot2 = __ldg(fl.cells + lo + cell_index(sx * fl.inv_res, sy * fl.inv_res, k));
        } else {
            double tx = sx - g[0], ty = sy - g[1];
            // the layer's own resolution when the layers differ in it (the reference's IEEE division by that map's res)
            const double res = fl.layer_res ? fl.layer_res[2 * (size_t)fl.env_layer[a / s.num_agents]] : fl.res;
            if (fl.layer_rot) {      // the layer's rotated frame: x_rot, y_rot of xy_2_rc (laser_models.py:75-76)
                const double *__restrict__ rt = fl.layer_rot + 2 * (size_t)fl.env_layer[a / s.num_agents];
                const double xr = tx * rt[0] + ty * rt[1];
                ty = -tx * rt[1] + ty * rt[0];
                tx = xr;
            }
            unsigned idx = fl.last;
            if (!(tx < 0 || tx >= g[2] || ty < 0 || ty >= g[3])) {
                const unsigned c = (unsigned)(int)(tx / res), r = (unsigned)(int)(ty / res);
                if (c < fl.width && r < fl.height) idx = r * fl.width + c;
            }
            slot2 = __ldg(fl.cells + lo + idx);
        }
    } else if (fl.cells && !fl.metres) {
        CellConsts k;
        k.ox = fl.ox; k.oy = fl.oy; k.eps = 0; k.tmax = 0; k.width = fl.width; k.height = fl.height; k.last = fl.last;
        slot2 = __ldg(fl.cells + lo + cell_index(sx * fl.inv_res, sy * fl.inv_res, k));
    } else if (fl.cells) {          // literal xy_2_rc (laser_models.py:55-86)
        double tx = sx - fl.orig_x, ty = sy - fl.orig_y;
        if (fl.rotated) {
            const double xr = tx * fl.orig_c + ty * fl.orig_s;
            ty = -tx * fl.orig_s + ty * fl.orig_c;
            tx = xr;
        }
        unsigned idx = fl.last;
        if (!(tx < 0 || tx >= fl.x_max || ty < 0 || ty >= fl.y_max)) {
            // a quotient that rounds up to width / height is off-map, like every other lookup (lidar.cuh dt_lookup)
            const unsigned c = (unsigned)(int)(tx / fl.res), r = (unsigned)(int)(ty / fl.res);
            if (c < fl.width && r < fl.height) idx = r * fl.width + c;
        }
        slot2 = __ldg(fl.cells + lo + idx);
    }
    double2 *sp = reinterpret_cast<double2 *>(s.scan_pose) + 2 * (size_t)a;
    const double ti0 = theta_index0(st[4], fov, theta_dis_f);
    sp[0] = make_double2(sx, sy);
    sp[1] = make_double2(slot2, ti0);
    if (fl.rec) {
        // everything the march needs per agent, computed once here instead of once per 32-beam work item
        // the march takes floor() through the low word of a magic-number add: cell coordinates must stay below 2^31.
        // Unrotated: |x| / res < 1e9 here and, along a ray, |x - orig| / res < 1e9 + reach / res < 1.5e9 (reach: step_impl).
        // Rotated: |x_rot| <= (|tx| + |ty|)(1 + 2^-51), and along a ray |tx| + |ty| <= |sx| + |sy| + sqrt(2) (max_range +
        // the largest DT value) + |ox| + |oy| <= |sx| + |sy| + 2 reach, so (|sx| + |sy|) / res < 1e9 and reach < 0.5e9 res
        // give |x_rot| / res < 2e9 (1 + 2^-50) < 2^31; likewise y_rot.  Anything else takes march_generic_rot, which has the
        // full row / column checks and needs no bound.
        const bool sane = (fl.rotated || fl.layer_rot) ? (fabs(sx) + fabs(sy)) * fl.inv_res < 1e9
                                                       : fabs(sx) * fl.inv_res < 1e9 && fabs(sy) * fl.inv_res < 1e9;
        const bool cells = !fl.metres;
        double2 *rp = fl.rec + 4 * (size_t)a;
        rp[0] = (sane && cells) ? make_double2(sx * fl.inv_res, sy * fl.inv_res) : make_double2(sx, sy);
        // LUT index of beam 0 as Q16.48 (ti0 in [0, theta_dis], theta_dis < 2^15); all ones = absurd coordinates
        const unsigned long long tfx = sane ? __double2ull_rd(ti0 * 281474976710656.0) : ~0ull;
        rp[1] = make_double2(slot2, __longlong_as_double((long long)tfx));
        // iTTC (laser_models.py:188-217) can only fire for |range - side_i| <= margin * |v cos_i|, i.e. never for
        // range > max(side) + margin * |v| (1e-9 of slack covers the roundings); v == 0 never fires
        const double v = st[3];
        const double thr = (v != 0.0) ? (fl.side_max + fl.ttc_margin * fabs(v)) * (1.0 + 1e-9) : -INFINITY;
        rp[2] = make_double2(thr, v);
        const unsigned long long lo_rec = fl.env_layer ? (unsigned long long)fl.env_layer[a / s.num_agents] * fl.rec_layer_stride : 0ull;
        rp[3] = make_double2(__longlong_as_double((long long)lo_rec), ti0);
    }
    // pose snapshot (Simulator.agent_poses, base_classes.py:574) + cos/sin of the yaw: every vertex / heading
    // computation of the finalize kernel reuses them instead of re-evaluating fp64 trig per opponent
    double *ap = s.agent_poses + 5 * (size_t)a;
    ap[0] = st[0]; ap[1] = st[1]; ap[2] = st[4];
    sincos(st[4], ap + 4, ap + 3);
    s.wall_flag[a] = 0;
}

struct RestartK {
    const uint32_t *__restrict__ list;      // restarted envs
    const uint32_t *__restrict__ count;
    float *scans, *final_scans;
    const unsigned long long *tick_counter; // or NULL (counter 0)
    double noise_std;
    unsigned long long noise_seed;
    uint32_t lidar;                         // bit i: slot i's scan row exists and is written
    uint32_t final_slots;                   // bit i: slot i has a lidar (its crash scan goes to final_scans)
};

// One beam i of agent a (its k_dynamics record r0, r1, r3) marched to completion, the range exactly as the tick's kernel of the
// map kind computes it: the statements of k_march_ttc's loop without the stop at the iTTC threshold, kept apart from it so
// that k_march_ttc keeps its code.  n: lookups.
template <int UNITS>
__device__ __forceinline__ double restart_beam_range(const TtcK &p, unsigned a, int i, const double2 r0, const double2 r1,
                                                     const double2 r3, unsigned &n) {
    const unsigned long long ti0fx = (unsigned long long)__double_as_longlong(r1.y);
    // the agent's map layer: origin, extent, resolution and rotation (warp-uniform loads, once per item)
    double2 lorig = p.orig, lmax = p.ext, lres = p.res, lrot = p.rot;
    if (p.layer_geom) {
        const unsigned l = (unsigned)__ldg(p.env_layer + a / p.num_agents);
        lorig = __ldg(reinterpret_cast<const double2 *>(p.layer_geom + 6 * (size_t)l));
        lmax = __ldg(reinterpret_cast<const double2 *>(p.layer_geom + 6 * (size_t)l) + 1);
        if (p.layer_res) lres = __ldg(reinterpret_cast<const double2 *>(p.layer_res) + l);
        if (UNITS == F110_SCAN_UNITS_ROT && p.layer_rot) lrot = __ldg(reinterpret_cast<const double2 *>(p.layer_rot) + l);
    }
    const unsigned long long off = (unsigned long long)__double_as_longlong(r3.x);
    double range;
    n = 1;
    if (ti0fx != ~0ull) {
        const unsigned long long vfx = ti0fx + (unsigned long long)(unsigned)i * p.inc_fx;
        unsigned ti = (unsigned)(vfx >> F110_FX_SHIFT);
        const unsigned fr = (unsigned)(vfx >> (F110_FX_SHIFT - 32));
        if (fr + p.guard32 <= 2u * p.guard32) ti = (unsigned)replay_theta_index(r3.y, i, p.inc, p.theta_dis_f);
        const double2 sc = __ldg(p.sincos2 + ti);
        const double *__restrict__ table = p.table + off;
        const double MAGIC = 6755399441055744.0;   // 2^52 + 2^51: round-down add == floor in the low word
        double X = r0.x, Y = r0.y, T = r1.x, D = r1.x;
        if (UNITS == F110_SCAN_UNITS_CELLS) {
            const double ox = lorig.x * p.res.y, oy = lorig.y * p.res.y;     // exact: res = 2^-k
            while (__double2hiint(D) != 0 && T <= p.tmax) {
                X = X + D * sc.y;
                Y = Y + D * sc.x;
                const unsigned c = (unsigned)__double2loint(__dadd_rd(X - ox, MAGIC));
                const unsigned r = (unsigned)__double2loint(__dadd_rd(Y - oy, MAGIC));
                // off the layer -> its padding on the canvas (or the extra row / column), which holds dt[-1,-1]
                D = __ldg(table + min(r, p.height) * (p.width + 1u) + min(c, p.width));
                T = T + D;
                n++;
            }
            range = ((T > p.tmax) ? p.tmax : T) * p.res.x;
        } else {
            while (__double2hiint(D) != 0 && T <= p.tmax) {
                X = X + D * sc.y;
                Y = Y + D * sc.x;
                double tx = X - lorig.x, ty = Y - lorig.y;
                if (UNITS == F110_SCAN_UNITS_ROT) {
                    // x_rot, y_rot as the reference rounds them: two products and a sum each, never fused
                    const double xr = __dadd_rn(__dmul_rn(tx, lrot.x), __dmul_rn(ty, lrot.y));
                    ty = __dadd_rn(__dmul_rn(-tx, lrot.y), __dmul_rn(ty, lrot.x));
                    tx = xr;
                }
                double qx = tx * lres.y, qy = ty * lres.y;
                qx = __fma_rn(__fma_rn(-qx, lres.x, tx), lres.y, qx);     // RN(t / res_l), see march.cuh
                qy = __fma_rn(__fma_rn(-qy, lres.x, ty), lres.y, qy);
                const int c = __double2loint(__dadd_rd(qx, MAGIC));
                const int r = __double2loint(__dadd_rd(qy, MAGIC));
                unsigned idx = (unsigned)r * p.width + (unsigned)c;
                if ((unsigned)c >= p.width || (unsigned)r >= p.height || tx >= lmax.x || ty >= lmax.y) idx = p.last;
                D = __ldg(table + idx);
                T = T + D;
                n++;
            }
            range = (T > p.tmax) ? p.tmax : T;
        }
    } else {
        // absurd coordinates: the literal reference arithmetic on the layer's geometry, out of line, as in the tick's kernel
        const size_t lo = (size_t)(off / p.layer_stride_lean * p.layer_stride);
        const int ti = beam_theta_index(r3.y, i, p.inc, p.theta_dis_f, 1e-6);
        const double2 sc = __ldg(p.sincos2 + ti);
        if (UNITS == F110_SCAN_UNITS_ROT)
            range = march_generic_rot(p.dt + lo, lorig, lrot, lmax, lres.x, __ldg(p.dt + lo + p.last), p.eps, p.max_range,
                                      (int)p.width, (int)p.height, r0.x, r0.y, sc.x, sc.y);
        else
            range = march_generic(p.dt + lo, lorig.x, lorig.y, lmax.x, lmax.y, lres.x, __ldg(p.dt + lo + p.last), p.eps,
                                  p.max_range, (int)p.width, r0.x, r0.y, sc.x, sc.y);
    }
    return range;
}

template <int UNITS, bool COUNT>
__global__ void __launch_bounds__(F110_TTC_THREADS) k_restart_march(const TtcK p, const RestartK r) {
    const unsigned lane = threadIdx.x & 31u;
    const unsigned per_env = p.num_agents * p.ipa;
    const unsigned long long items = (unsigned long long)__ldg(r.count) * per_env;
    const unsigned long long stride = (unsigned long long)gridDim.x * (F110_TTC_THREADS / 32);
    // the noise of a plain tick at counter t | 2^63, t the counter of the tick that ended the episode
    const unsigned long long tick = (r.tick_counter ? *r.tick_counter : 0ull) | (1ull << 63);
    unsigned looks = 0u;
    for (unsigned long long item = (unsigned long long)blockIdx.x * (F110_TTC_THREADS / 32) + (threadIdx.x >> 5); item < items;
         item += stride) {
        const unsigned e = (unsigned)(item / per_env), rem = (unsigned)(item - (unsigned long long)e * per_env);
        const unsigned slot = rem / p.ipa;
        const unsigned a = __ldg(r.list + e) * p.num_agents + slot;
        const int i = (int)((rem - slot * p.ipa) * 32u + lane);
        if (i >= p.B) continue;
        const double2 *__restrict__ rp = p.rec + 4 * (size_t)a;
        const double2 r0 = __ldg(rp), r1 = __ldg(rp + 1), r2 = __ldg(rp + 2), r3 = __ldg(rp + 3);
        unsigned n;
        double range = restart_beam_range<UNITS>(p, a, i, r0, r1, r3, n);
        if (r.noise_std > 0.0) range = range + r.noise_std * normal_sample(r.noise_seed, tick, (uint64_t)a * (uint64_t)p.B + (uint64_t)i);
        if (range <= r2.x) {
            const double2 cs2 = __ldg(p.cos_side + i);
            ttc_exact(range, r2.y, cs2.x, cs2.y, p.ttc_thresh, p.ttc_margin, p.wall_flag + a);
        }
        if ((r.lidar >> slot) & 1u) {
            const size_t at = (size_t)a * (size_t)p.B + (size_t)i;
            if ((r.final_slots >> slot) & 1u) r.final_scans[at] = r.scans[at];
            r.scans[at] = (float)range;
        }
        if (COUNT) looks += n;
    }
    if (COUNT) {
        const unsigned nsum = __reduce_add_sync(0xffffffffu, looks);
        if (lane == 0 && nsum) atomicAdd(p.lookup_counter, (unsigned long long)nsum);
    }
}

// warp per (listed env, slot whose scan exists): k_lidar_cast's statements on the listed egos, copied from it so that
// k_lidar_cast keeps its code (without its end_of_tick_housekeeping: the plain tick's tail consumed the queue counters)
__global__ void __launch_bounds__(32 * F110_LIDAR_CAST_WARPS) k_episode_cast(f110_sim s, BeamView bv, LidarOrder lo,
                                                                              const uint32_t *__restrict__ list,
                                                                              const uint32_t *__restrict__ count, double max_scan_range) {
    __shared__ TailTask tasks_all[F110_LIDAR_CAST_WARPS][31];
    const int A = s.num_agents;
    const int opp = A - 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned r = blockIdx.x * F110_LIDAR_CAST_WARPS + (unsigned)warp;
    if (opp < 1 || r >= *count * lo.slots) return;       // warp-uniform
    const unsigned e = r / lo.slots;
    const int a = (int)(list[e] * (unsigned)A + (lidar_agent(r, lo, (unsigned)A) - e * (unsigned)A));
    const int env = a / A, slot = a - env * A;
    TailTask *tasks = tasks_all[warp];
    const int hit = s.wall_flag[a];
    const double *pa = s.agent_poses + 5 * (size_t)a;
    const double px = pa[0], py = pa[1];
    // check_ttc zeroes state[3:] -- including the yaw -- before the opponent ray-cast reads it (:246-249, :225)
    const double yaw = hit ? 0.0 : pa[2];
    const double cyaw = hit ? 1.0 : pa[3], syaw = hit ? 0.0 : pa[4];
    const double *p = s.params + (size_t)(s.params_per_env ? a : slot) * F110_NPARAM;
    const double length = p[P_LENGTH], width = p[P_WIDTH];
    const double half_diag = 0.5 * sqrt(length * length + width * width);
    if (lane < opp) {
        const int oj = lane, j = oj < slot ? oj : oj + 1;     // opponents in ascending index, skipping the ego itself
        const double *pb = s.agent_poses + 5 * (size_t)(env * A + j);
        TailTask &k = tasks[oj];
        const double ddx = pb[0] - px, ddy = pb[1] - py;
        const double far = max_scan_range + half_diag;
        int active = 1;
        if (ddx * ddx + ddy * ddy > far * far) active = 0;     // cannot shorten any beam (see finalize_agent)
        k.active = active;
        if (active) {
            double v[8];
            get_vertices_cs(pb[0], pb[1], pb[3], pb[4], length, width, v);
            int lo_i, hi_i;
            double phi;
            blocked_view_indices_cs(px, py, cyaw, syaw, v, bv.scan_angles, bv.num_beams, bv.fov, bv.angle_increment, pb[0], pb[1],
                                    lo_i, hi_i, phi);
            double cone = 4.0;
            if (hi_i - lo_i >= 96) {
                const double dist = sqrt(ddx * ddx + ddy * ddy);
                if (dist > 1.25 * half_diag) cone = asin(half_diag / dist) + 0.05;
            }
            k.px = px; k.py = py; k.yaw = yaw; k.phi = phi; k.cone = cone; k.lo = lo_i; k.hi = hi_i;
#pragma unroll
            for (int q = 0; q < 8; q++) k.v[q] = v[q];
        }
    }
    __syncwarp();
    float *scan = s.scans + (size_t)a * bv.num_beams;
    for (int oj = 0; oj < opp; oj++) {
        const TailTask &k = tasks[oj];
        if (!k.active) continue;
        const double kpx = k.px, kpy = k.py, kyaw = k.yaw, phi = k.phi, cone = k.cone;
        const int lo_i = k.lo, hi_i = k.hi;
        double v[8];
#pragma unroll
        for (int q = 0; q < 8; q++) v[q] = k.v[q];
        auto cast_beams = [&](int i0, int i1) {
            for (int i = i0 + lane; i <= i1; i += 32) {
                const float cur = scan[i];
                double bt = kyaw + bv.scan_angles[i];
                double dl = bt - phi;
                dl = dl - (2 * M_PI) * rint(dl * (1.0 / (2 * M_PI)));
                const double adl = fabs(dl);
                if (adl > cone && (M_PI - adl) > cone) continue;
                double v3x, v3y;
                sincos(bt + M_PI / 2., &v3y, &v3x);
                const double curd = (double)cur;
                double rr = INFINITY;
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    int e2 = (e + 1) & 3;
                    double d = get_range_below(kpx, kpy, v3x, v3y, v[2 * e], v[2 * e + 1], v[2 * e2], v[2 * e2 + 1], curd);
                    if (d < rr) rr = d;
                }
                float rf = (float)rr;
                if (rf < cur) scan[i] = rf;
            }
        };
        if (cone < 3.5 && hi_i - lo_i >= 96) {
            const double base = wrap_2pi_diff(phi - kyaw), half = bv.fov / 2., inv_inc = 1.0 / bv.angle_increment;   // (see finalize_agent)
            const int m0 = max(-3, (int)floor((-half - cone - 0.02 - base) * (1.0 / M_PI))),
                      m1 = min(5, (int)ceil((half + cone + 0.02 - base) * (1.0 / M_PI)));
            for (int m = m0; m <= m1; m++) {
                const double c = base + (double)m * M_PI;
                const double f0 = (c - cone + half) * inv_inc - 2.0, f1 = (c + cone + half) * inv_inc + 2.0;
                if (f1 < (double)lo_i || f0 > (double)hi_i) continue;
                const int i0 = max(lo_i, (int)floor(fmax(f0, (double)lo_i))), i1 = min(hi_i, (int)ceil(fmin(f1, (double)hi_i)));
                cast_beams(i0, i1);
            }
        } else {
            cast_beams(lo_i, hi_i);
        }
        __syncwarp();
    }
}

// thread per listed env: the agent duties of the tail (after the cast, whose yaw comes from wall_flag), then the zero tick's
// lap logic with the plain tick's `done` kept
__global__ void k_episode_tail(f110_sim s, const uint32_t *__restrict__ list, const uint32_t *__restrict__ count) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= *count) return;
    const int env = (int)list[k], A = s.num_agents;
    for (int slot = 0; slot < A; slot++) {
        const int a = env * A + slot;
        agent_duties(s, env, slot, a, s.wall_flag[a], s.agent_poses + 5 * (size_t)a);
    }
    const uint8_t done = s.done[env];
    env_post_step_one(s, env);
    s.done[env] = done;
}

// warp per agent of a listed env: k_obstacles' body (contact, and the clip of the scans of the slots that have a lidar)
__global__ void __launch_bounds__(128) k_episode_obstacles(f110_sim s, BeamView bv, ObstK o, double max_scan_range,
                                                           const uint32_t *__restrict__ list, const uint32_t *__restrict__ count) {
    const unsigned w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, A = (unsigned)s.num_agents;
    const unsigned k = w / A;
    if (k >= *count) return;
    obstacles_agent<true, true>(s, bv, o, max_scan_range, (int)(list[k] * A + (w - k * A)), (int)(threadIdx.x & 31));
}

}  // namespace f110
