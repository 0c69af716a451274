// predict.cuh — f110_predict (include/f110_predict.h): K candidate futures of M agents, H ticks each, in one launch; and
// f110_predict_scored (include/f110_mppi.h): the same rollout with each sample's cost along its map's centerline.
//
// k_predict<UNITS>  thread per sample (m, k), consecutive lanes on the samples of one agent (the KS/ST branch and the map region
//                   are then mostly shared).  State and steer FIFO stay in registers for all H steps.  Per step:
//   1. k_dynamics' per-agent statements: FIFO, integrate_tick, scan pose, the first DT lookup d0 at the scan pose and the iTTC
//      pre-test threshold thr, exactly as k_dynamics builds them for the march record (march_lean.cuh);
//   2. k_ttc_select's pre-test: d0 > thr and max_range > thr means no beam can fire (a NaN or absurd coordinates fail it);
//   3. the lanes that fail it are marched by their whole warp, one after another (ballot loop): lane j takes beams j, j + 32, ...
//      with k_march_ttc's per-beam arithmetic for the map kind, stopping a beam once its running total exceeds thr, and the
//      warp stops at the first 32-beam round in which a beam fires.  Exact: the wall check is an OR over the beams;
//   4. a hit zeroes state[3:] (agent_duties, the tail's wall-hit zeroing).
// Opponents and boxes play no part: in the tick they only clip scans (after the wall check, which reads the wall-only scan) and
// set collisions; neither changes state (DESIGN §3.14).
// The statements below are copies of k_dynamics', k_march_ttc's and agent_duties' (each block names its origin): calling shared
// functions out of those kernels would change their code.  integrate_tick, cell_index, theta_index0, replay_theta_index,
// beam_theta_index and march_generic(_rot) are called as they are.
#pragma once

namespace f110 {

#define F110_PREDICT_THREADS 128

struct PredictK {
    const int32_t *__restrict__ agent_ids;  // [M]
    const double2 *__restrict__ actions;    // [M][K][H] (steer, speed)
    double *__restrict__ final_state;       // [M][K][7]
    int32_t *__restrict__ wall_step;        // [M][K]
    double *__restrict__ states;            // [M][K][H][7] or NULL
    float *__restrict__ clearance;          // [M][K][H] or NULL
    unsigned long long samples;             // M * K
    unsigned K;
    int H;
    double d0_scale;                        // metres per unit of d0 (resolution on cell-unit tables, else 1)
    double fov, theta_dis_f;
};

// The first DT lookup at the scan pose (sx, sy) of agent a, in the units of fl.cells: k_dynamics' `slot2` statements.
__device__ __forceinline__ double predict_first_lookup(const f110_sim &s, const FirstLookup &fl, int a, double sx, double sy) {
    double slot2 = 0.0;
    const size_t lo = fl.env_layer ? (size_t)fl.env_layer[a / s.num_agents] * (size_t)fl.layer_stride : (size_t)0;
    if (fl.layer_geom) {
        const double *__restrict__ g = fl.layer_geom + 6 * (size_t)fl.env_layer[a / s.num_agents];
        if (!fl.metres) {
            CellConsts k;
            k.ox = g[0] * fl.inv_res; k.oy = g[1] * fl.inv_res; k.eps = 0; k.tmax = 0;
            k.width = fl.width; k.height = fl.height; k.last = fl.last;
            slot2 = __ldg(fl.cells + lo + cell_index(sx * fl.inv_res, sy * fl.inv_res, k));
        } else {
            double tx = sx - g[0], ty = sy - g[1];
            const double res = fl.layer_res ? fl.layer_res[2 * (size_t)fl.env_layer[a / s.num_agents]] : fl.res;
            if (fl.layer_rot) {
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
    } else if (!fl.metres) {
        CellConsts k;
        k.ox = fl.ox; k.oy = fl.oy; k.eps = 0; k.tmax = 0; k.width = fl.width; k.height = fl.height; k.last = fl.last;
        slot2 = __ldg(fl.cells + lo + cell_index(sx * fl.inv_res, sy * fl.inv_res, k));
    } else {
        double tx = sx - fl.orig_x, ty = sy - fl.orig_y;
        if (fl.rotated) {
            const double xr = tx * fl.orig_c + ty * fl.orig_s;
            ty = -tx * fl.orig_s + ty * fl.orig_c;
            tx = xr;
        }
        unsigned idx = fl.last;
        if (!(tx < 0 || tx >= fl.x_max || ty < 0 || ty >= fl.y_max)) {
            const unsigned c = (unsigned)(int)(tx / fl.res), r = (unsigned)(int)(ty / fl.res);
            if (c < fl.width && r < fl.height) idx = r * fl.width + c;
        }
        slot2 = __ldg(fl.cells + lo + idx);
    }
    return slot2;
}

// ttc_exact's predicate (check_ttc_jit, laser_models.py:188-217) as a value: passing ttc_exact a flag in shared memory would turn
// its global reduction into a generic atomic in every kernel that calls it
__device__ __forceinline__ bool predict_ttc_fires(double range, double v, double cos_i, double side_i, double thresh, double margin) {
    const double pv = v * cos_i;
    const double d = range - side_i;
    if (fabs(d) <= margin * fabs(pv)) {
        const double ttc = d / pv;
        return (ttc < thresh) && (ttc >= 0.0);
    }
    return false;
}

// Does any beam of the agent whose record is (r0, r1, r2, r3) fire?  Called by the whole warp with the same record; lane j takes
// beams j, j + 32, ...  The per-beam statements are k_march_ttc's.
template <int UNITS>
__device__ __forceinline__ bool predict_wall_hit(const TtcK &p, unsigned a, unsigned lane, const double2 r0, const double2 r1,
                                                 const double2 r2, const double2 r3) {
    const unsigned long long ti0fx = (unsigned long long)__double_as_longlong(r1.y);
    double2 lorig = p.orig, lmax = p.ext, lres = p.res, lrot = p.rot;
    if (p.layer_geom) {
        const unsigned l = (unsigned)__ldg(p.env_layer + a / p.num_agents);
        lorig = __ldg(reinterpret_cast<const double2 *>(p.layer_geom + 6 * (size_t)l));
        lmax = __ldg(reinterpret_cast<const double2 *>(p.layer_geom + 6 * (size_t)l) + 1);
        if (p.layer_res) lres = __ldg(reinterpret_cast<const double2 *>(p.layer_res) + l);
        if (UNITS == F110_SCAN_UNITS_ROT && p.layer_rot) lrot = __ldg(reinterpret_cast<const double2 *>(p.layer_rot) + l);
    }
    const unsigned long long off = (unsigned long long)__double_as_longlong(r3.x);
    const double thr = r2.x;
    const bool stops = p.max_range > thr;
    for (int base = 0; base < p.B; base += 32) {
        const int i = base + (int)lane;
        bool fired = false;
        if (i < p.B) {
            double range;
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
                    while (__double2hiint(D) != 0 && T <= p.tmax && !(stops && T * p.res.x > thr)) {
                        X = X + D * sc.y;
                        Y = Y + D * sc.x;
                        const unsigned c = (unsigned)__double2loint(__dadd_rd(X - ox, MAGIC));
                        const unsigned r = (unsigned)__double2loint(__dadd_rd(Y - oy, MAGIC));
                        D = __ldg(table + min(r, p.height) * (p.width + 1u) + min(c, p.width));
                        T = T + D;
                    }
                    range = ((T > p.tmax) ? p.tmax : T) * p.res.x;
                } else {
                    while (__double2hiint(D) != 0 && T <= p.tmax && !(stops && T > thr)) {
                        X = X + D * sc.y;
                        Y = Y + D * sc.x;
                        double tx = X - lorig.x, ty = Y - lorig.y;
                        if (UNITS == F110_SCAN_UNITS_ROT) {
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
                    }
                    range = (T > p.tmax) ? p.tmax : T;
                }
            } else {
                // absurd coordinates: the literal reference arithmetic on the layer's geometry, out of line
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
            if (range <= thr) {
                const double2 cs2 = __ldg(p.cos_side + i);
                fired = predict_ttc_fires(range, r2.y, cs2.x, cs2.y, p.ttc_thresh, p.ttc_margin);
            }
        }
        if (__any_sync(0xffffffffu, fired)) return true;
    }
    return false;
}

template <int UNITS>
__global__ void __launch_bounds__(F110_PREDICT_THREADS) k_predict(const f110_sim s, const FirstLookup fl, const TtcK q,
                                                                  const PredictK p) {
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long smp = (unsigned long long)blockIdx.x * F110_PREDICT_THREADS + threadIdx.x;
    const bool live = smp < p.samples;
    const int NA = s.num_envs * s.num_agents;
    int a = -1;
    if (live) {
        const int id = __ldg(p.agent_ids + smp / p.K);
        if (id >= 0 && id < NA) a = id;
    }
    const bool valid = a >= 0;
    double st[7], b0 = 0.0, b1 = 0.0;
    int cnt = 0;
    const double *prm = nullptr;
#pragma unroll
    for (int k = 0; k < 7; k++) st[k] = __longlong_as_double(0x7ff8000000000000ll);      // NaN: an id outside [0, N*A)
    if (valid) {
        prm = s.params + (size_t)(s.params_per_env ? a : a % s.num_agents) * F110_NPARAM;
#pragma unroll
        for (int k = 0; k < 7; k++) st[k] = s.state[(size_t)k * NA + a];
        cnt = s.steer_cnt[a];
        b0 = s.steer_buf[a]; b1 = s.steer_buf[(size_t)NA + a];
    }
    const double2 *act = p.actions + smp * (unsigned long long)p.H;
    int wall = -1;
    for (int h = 0; h < p.H; h++) {
        bool listed = false;
        double2 r0 = make_double2(0.0, 0.0), r1 = r0, r2 = r0, r3 = r0;
        float clear = __int_as_float(0x7fc00000);
        if (valid) {
            // k_dynamics: steering delay FIFO (base_classes.py:270-278), integrate_tick, scan pose (base_classes.py:406-409)
            const double2 u = __ldg(act + h);
            const double steer = (cnt < 2) ? 0. : b1;
            b1 = b0;
            b0 = u.x;
            if (cnt < 2) cnt = cnt + 1;
            integrate_tick(st, steer, u.y, prm, s.timestep, s.integrator);
            double sx = st[0], sy = st[1];
            if (s.lidar_dist != 0.0) {
                sx = st[0] + s.lidar_dist * cos(st[4]);
                sy = st[1] + s.lidar_dist * sin(st[4]);
            }
            const double slot2 = predict_first_lookup(s, fl, a, sx, sy);
            clear = (float)(slot2 * p.d0_scale);
            const double ti0 = theta_index0(st[4], p.fov, p.theta_dis_f);
            // k_dynamics: the march record (march_lean.cuh), `sane` and the derivation there
            const bool sane = (fl.rotated || fl.layer_rot) ? (fabs(sx) + fabs(sy)) * fl.inv_res < 1e9
                                                           : fabs(sx) * fl.inv_res < 1e9 && fabs(sy) * fl.inv_res < 1e9;
            r0 = (sane && !fl.metres) ? make_double2(sx * fl.inv_res, sy * fl.inv_res) : make_double2(sx, sy);
            const unsigned long long tfx = sane ? __double2ull_rd(ti0 * 281474976710656.0) : ~0ull;
            r1 = make_double2(slot2, __longlong_as_double((long long)tfx));
            const double v = st[3];
            const double thr = (v != 0.0) ? (fl.side_max + fl.ttc_margin * fabs(v)) * (1.0 + 1e-9) : -INFINITY;
            r2 = make_double2(thr, v);
            const unsigned long long lo_rec = fl.env_layer ? (unsigned long long)fl.env_layer[a / s.num_agents] * fl.rec_layer_stride : 0ull;
            r3 = make_double2(__longlong_as_double((long long)lo_rec), ti0);
            // k_ttc_select's pre-test (false for a NaN on either side)
            const bool absurd = tfx == ~0ull;
            const bool clr = slot2 * p.d0_scale > thr && q.max_range > thr;
            listed = absurd || !clr;
        }
        unsigned vote = __ballot_sync(0xffffffffu, listed);
        bool hit = false;
        while (vote) {
            const int src = __ffs(vote) - 1;
            vote &= vote - 1u;
            const double2 w0 = make_double2(__shfl_sync(0xffffffffu, r0.x, src), __shfl_sync(0xffffffffu, r0.y, src));
            const double2 w1 = make_double2(__shfl_sync(0xffffffffu, r1.x, src), __shfl_sync(0xffffffffu, r1.y, src));
            const double2 w2 = make_double2(__shfl_sync(0xffffffffu, r2.x, src), __shfl_sync(0xffffffffu, r2.y, src));
            const double2 w3 = make_double2(__shfl_sync(0xffffffffu, r3.x, src), __shfl_sync(0xffffffffu, r3.y, src));
            const unsigned wa = (unsigned)__shfl_sync(0xffffffffu, a, src);
            const bool f = predict_wall_hit<UNITS>(q, wa, lane, w0, w1, w2, w3);
            if ((int)lane == src) hit = f;
        }
        if (hit) {      // agent_duties: the tail's wall-hit zeroing
#pragma unroll
            for (int k = 3; k < 7; k++) st[k] = 0.0;
            if (wall < 0) wall = h;
        }
        if (live) {
            const unsigned long long o = smp * (unsigned long long)p.H + (unsigned long long)h;
            if (p.states) {
#pragma unroll
                for (int k = 0; k < 7; k++) p.states[7 * o + k] = st[k];
            }
            if (p.clearance) p.clearance[o] = clear;
        }
    }
    if (live) {
#pragma unroll
        for (int k = 0; k < 7; k++) p.final_state[7 * smp + k] = st[k];
        p.wall_step[smp] = wall;
    }
}

// ---- f110_predict_scored (include/f110_mppi.h): the cost of every sample along its map's centerline, beside the rollout
struct CostK {
    const double *__restrict__ segments;      // f110_track
    const int32_t *__restrict__ table_start;
    int num_tables;
    int back, window;                         // window = back + fwd + 1
    double reacquire_dist;
    int32_t *__restrict__ seg0;               // [M] the source pose's segment, -1 = not acquired
    double *__restrict__ s0;                  // [M] its arc length
    const double2 *__restrict__ prev_action;  // [M] or NULL
    double *__restrict__ cost;                // [M][K]
    double w_lat, w_head, w_clear, w_dsteer, w_dspeed, w_prog, w_wall, clear_min;
};

// the table of agent a's layer (k_track_progress' rule), or false for a bad table id
__device__ __forceinline__ bool cost_table(const f110_sim &s, const CostK &c, int a, const double *__restrict__ &rec, int &n) {
    rec = c.segments;
    return track_table(c.table_start, c.num_tables, s.env_layer ? s.env_layer[a / s.num_agents] : 0, rec, n);
}

// The acquiring update of each source agent: a warp per m, f110_track_project's projection of the agent's pose.
__global__ void __launch_bounds__(128) k_scored_acquire(const f110_sim s, const int32_t *__restrict__ agent_ids, int M,
                                                         const CostK c) {
    const int m = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (m >= M) return;
    const int NA = s.num_envs * s.num_agents;
    const int a = agent_ids[m];
    const double *rec = nullptr;
    int n = 0;
    double px = 0.0, py = 0.0, yaw = 0.0;
    bool ok = a >= 0 && a < NA;
    if (ok) {
        px = s.state[a]; py = s.state[(size_t)NA + a]; yaw = s.state[4 * (size_t)NA + a];
        ok = isfinite(px) && isfinite(py) && isfinite(yaw) && cost_table(s, c, a, rec, n);
    }
    TrackHit h;
    h.k = 0x7fffffff;
    if (ok) h = track_search(rec, n, 0, n, px, py, lane);
    if (lane != 0) return;
    if (h.k == 0x7fffffff) {
        c.seg0[m] = -1;
        c.s0[m] = __longlong_as_double(0x7ff8000000000000ll);
        return;
    }
    const TrackOut r = track_outputs(rec, h.k, h.t, px, py, yaw);
    c.seg0[m] = h.k;
    c.s0[m] = r.s;
}

// The per-sample tracker (k_track_progress' tracking update, one thread) and the cost sum of include/f110_mppi.h.  Little is
// held across a step's warp march: the actions are read again from the sample's row, the lap length from the table.
struct Scorer {
    const CostK &c;
    const double *rec;
    const double2 *prev;          // prev_action[m], or NULL
    int n, seg;
    bool lost;
    double s_prev, prog, cost, clr;

    __device__ __forceinline__ explicit Scorer(const CostK &k) : c(k) {}

    __device__ __forceinline__ void begin(const f110_sim &s, bool valid, int a, unsigned long long m) {
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        cost = 0.0; prog = 0.0; clr = nan; n = 0; seg = -1; rec = nullptr; s_prev = nan;
        prev = c.prev_action ? c.prev_action + m : nullptr;
        lost = !valid;
        if (valid) {
            seg = c.seg0[m];
            s_prev = c.s0[m];
            lost = seg < 0 || !cost_table(s, c, a, rec, n);
        }
        if (lost) cost = nan;
    }
    __device__ __forceinline__ void clearance(double metres) { clr = metres; }
    __device__ __forceinline__ void step(int h, const double *st, const double2 *act) {
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        if (lost) return;
        const double px = st[0], py = st[1], yaw = st[4];
        if (!(isfinite(px) && isfinite(py) && isfinite(yaw))) { lost = true; cost = nan; return; }
        int base = (seg - c.back) % n;
        if (base < 0) base += n;
        TrackHit t = track_search_thread(rec, n, base, c.window < n ? c.window : n, px, py);
        int sg;
        if (t.k == 0x7fffffff || !(t.dist <= c.reacquire_dist)) {
            t = track_search_thread(rec, n, 0, n, px, py);
            sg = t.k;
        } else {
            sg = (base + t.k) % n;
        }
        if (t.k == 0x7fffffff) { lost = true; cost = nan; return; }
        const TrackOut r = track_outputs(rec, sg, t.t, px, py, yaw);
        const double *last = rec + (size_t)(n - 1) * F110_TRACK_REC;
        const double L = last[5] + last[6];          // k_track_progress' lap length
        double delta = r.s - s_prev;
        if (delta > L * 0.5) delta -= L;
        else if (delta < -(L * 0.5)) delta += L;
        prog = prog + delta;
        s_prev = r.s;
        seg = sg;
        const double2 u = __ldg(act + h);
        const double2 up = h > 0 ? __ldg(act + h - 1) : (prev ? *prev : u);     // no rate terms at h = 0 without prev_action
        const double gap = c.clear_min - clr;
        const double pen = gap > 0.0 ? gap : 0.0;
        const double ds = u.x - up.x, dv = u.y - up.y;
        cost = cost + c.w_lat * (r.d * r.d);
        cost = cost + c.w_head * (r.e * r.e);
        cost = cost + c.w_clear * (pen * pen);
        cost = cost + c.w_dsteer * (ds * ds);
        cost = cost + c.w_dspeed * (dv * dv);
    }
    __device__ __forceinline__ void finish(unsigned long long smp, int wall) {
        double v = cost - c.w_prog * prog;
        if (wall >= 0) v = v + c.w_wall;
        c.cost[smp] = v;
    }
};

// k_predict with the Scorer calls added (a copy, so that k_predict keeps its code): the rollout statements are k_predict's.
template <int UNITS>
__global__ void __launch_bounds__(F110_PREDICT_THREADS) k_scored_rollout(const f110_sim s, const FirstLookup fl, const TtcK q,
                                                                         const PredictK p, const CostK c) {
    Scorer score(c);
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long smp = (unsigned long long)blockIdx.x * F110_PREDICT_THREADS + threadIdx.x;
    const bool live = smp < p.samples;
    const int NA = s.num_envs * s.num_agents;
    int a = -1;
    if (live) {
        const int id = __ldg(p.agent_ids + smp / p.K);
        if (id >= 0 && id < NA) a = id;
    }
    const bool valid = a >= 0;
    double st[7], b0 = 0.0, b1 = 0.0;
    int cnt = 0;
    const double *prm = nullptr;
#pragma unroll
    for (int k = 0; k < 7; k++) st[k] = __longlong_as_double(0x7ff8000000000000ll);      // NaN: an id outside [0, N*A)
    if (valid) {
        prm = s.params + (size_t)(s.params_per_env ? a : a % s.num_agents) * F110_NPARAM;
#pragma unroll
        for (int k = 0; k < 7; k++) st[k] = s.state[(size_t)k * NA + a];
        cnt = s.steer_cnt[a];
        b0 = s.steer_buf[a]; b1 = s.steer_buf[(size_t)NA + a];
    }
    score.begin(s, valid, a, smp / p.K);
    const double2 *act = p.actions + smp * (unsigned long long)p.H;
    int wall = -1;
    for (int h = 0; h < p.H; h++) {
        bool listed = false;
        double2 r0 = make_double2(0.0, 0.0), r1 = r0, r2 = r0, r3 = r0;
        float clear = __int_as_float(0x7fc00000);
        if (valid) {
            // k_dynamics: steering delay FIFO (base_classes.py:270-278), integrate_tick, scan pose (base_classes.py:406-409)
            const double2 u = __ldg(act + h);
            const double steer = (cnt < 2) ? 0. : b1;
            b1 = b0;
            b0 = u.x;
            if (cnt < 2) cnt = cnt + 1;
            integrate_tick(st, steer, u.y, prm, s.timestep, s.integrator);
            double sx = st[0], sy = st[1];
            if (s.lidar_dist != 0.0) {
                sx = st[0] + s.lidar_dist * cos(st[4]);
                sy = st[1] + s.lidar_dist * sin(st[4]);
            }
            const double slot2 = predict_first_lookup(s, fl, a, sx, sy);
            clear = (float)(slot2 * p.d0_scale);
            score.clearance(slot2 * p.d0_scale);
            const double ti0 = theta_index0(st[4], p.fov, p.theta_dis_f);
            // k_dynamics: the march record (march_lean.cuh), `sane` and the derivation there
            const bool sane = (fl.rotated || fl.layer_rot) ? (fabs(sx) + fabs(sy)) * fl.inv_res < 1e9
                                                           : fabs(sx) * fl.inv_res < 1e9 && fabs(sy) * fl.inv_res < 1e9;
            r0 = (sane && !fl.metres) ? make_double2(sx * fl.inv_res, sy * fl.inv_res) : make_double2(sx, sy);
            const unsigned long long tfx = sane ? __double2ull_rd(ti0 * 281474976710656.0) : ~0ull;
            r1 = make_double2(slot2, __longlong_as_double((long long)tfx));
            const double v = st[3];
            const double thr = (v != 0.0) ? (fl.side_max + fl.ttc_margin * fabs(v)) * (1.0 + 1e-9) : -INFINITY;
            r2 = make_double2(thr, v);
            const unsigned long long lo_rec = fl.env_layer ? (unsigned long long)fl.env_layer[a / s.num_agents] * fl.rec_layer_stride : 0ull;
            r3 = make_double2(__longlong_as_double((long long)lo_rec), ti0);
            // k_ttc_select's pre-test (false for a NaN on either side)
            const bool absurd = tfx == ~0ull;
            const bool clr = slot2 * p.d0_scale > thr && q.max_range > thr;
            listed = absurd || !clr;
        }
        unsigned vote = __ballot_sync(0xffffffffu, listed);
        bool hit = false;
        while (vote) {
            const int src = __ffs(vote) - 1;
            vote &= vote - 1u;
            const double2 w0 = make_double2(__shfl_sync(0xffffffffu, r0.x, src), __shfl_sync(0xffffffffu, r0.y, src));
            const double2 w1 = make_double2(__shfl_sync(0xffffffffu, r1.x, src), __shfl_sync(0xffffffffu, r1.y, src));
            const double2 w2 = make_double2(__shfl_sync(0xffffffffu, r2.x, src), __shfl_sync(0xffffffffu, r2.y, src));
            const double2 w3 = make_double2(__shfl_sync(0xffffffffu, r3.x, src), __shfl_sync(0xffffffffu, r3.y, src));
            const unsigned wa = (unsigned)__shfl_sync(0xffffffffu, a, src);
            const bool f = predict_wall_hit<UNITS>(q, wa, lane, w0, w1, w2, w3);
            if ((int)lane == src) hit = f;
        }
        if (hit) {      // agent_duties: the tail's wall-hit zeroing
#pragma unroll
            for (int k = 3; k < 7; k++) st[k] = 0.0;
            if (wall < 0) wall = h;
        }
        score.step(h, st, act);
        if (live) {
            const unsigned long long o = smp * (unsigned long long)p.H + (unsigned long long)h;
            if (p.states) {
#pragma unroll
                for (int k = 0; k < 7; k++) p.states[7 * o + k] = st[k];
            }
            if (p.clearance) p.clearance[o] = clear;
        }
    }
    if (live) {
#pragma unroll
        for (int k = 0; k < 7; k++) p.final_state[7 * smp + k] = st[k];
        p.wall_step[smp] = wall;
        score.finish(smp, wall);
    }
}

}  // namespace f110
