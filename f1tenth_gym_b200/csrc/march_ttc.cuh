// march_ttc.cuh — the intermediate tick of f110_tick_repeat: ticks whose scans nobody reads.
//
// The reference uses a tick's scan twice: as the observation, and in the iTTC wall check (check_ttc_jit,
// laser_models.py:188-217) that sets RaceCar.in_collision.  On a tick whose observation is withheld only the second use is
// left, and k_dynamics has already written what decides most of it: per agent the first DT lookup d0 at the scan pose and
// thr = (max side distance + margin |v|)(1 + 1e-9), with the proof (f110_b200.cu, k_dynamics) that a beam of range > thr
// cannot fire.  Every beam's range is min(d0 + sum of non-negative steps, max_range) >= min(d0, max_range), so
//     d0 > thr  and  max_range > thr   =>   no beam of the agent can fire: wall_flag stays 0 and nothing is marched.
// k_ttc_select   thread per agent: lists the agents for which that is NOT true (written that way round, a NaN lists the
//                agent) and every agent k_dynamics marked absurd; one global atomic per block.  On a tick with a lidar mask
//                (f110_lidar) only the sensorless agents are candidates: the others are in the tick's full march.
// k_march_ttc    fixed grid, a warp per 32-beam item of a listed agent: the beam's range exactly as the tick's kernel of the
//                map kind computes it -- cell units (k_march_lean<CELLS>, k_march_lean_het<CELLS>), metres (k_march_lean,
//                k_march_lean_het, k_march_lean_het_res) or the rotated frame (k_march_lean_rot); the layer's geometry comes
//                from the per-layer tables when the map has them, else from the launch parameters, as in k_scan_lean -- then
//                the tick's predicate (pre-test against thr, ttc_exact).  A beam stops as soon as its running total exceeds
//                thr: its range can then only be larger.  No scan is stored and no queue cost.
// k_tail_noscan  the tick's tail without the opponent ray-cast, which only edits scans: wall-hit zeroing, GJK, collisions,
//                then per env the lap logic, the done bookkeeping of the repeat call and the auto-reset.
// Results never depend on the list order.
#pragma once
#include "scan_lean.cuh"

namespace f110 {

#define F110_TTC_THREADS 256
#define F110_TTC_SELECT_THREADS 256
#define F110_TAIL_NOSCAN_THREADS 128

struct TtcSelectK {
    const double2 *__restrict__ rec;        // [M][4] per-agent record of k_dynamics (march_lean.cuh)
    uint32_t *__restrict__ list;            // [M] out: flat ids of the agents to march
    uint32_t *count;                        // [1] out: entries of `list` (zeroed before the launch)
    unsigned long long *marched;            // [1] or NULL: += entries (measurement)
    double d0_scale;                        // metres per unit of the record's first lookup (resolution on cell-unit tables, else 1)
    double max_range;
    unsigned agents;
    uint32_t skip;                          // lidar mask of a masked tick (f110_lidar): agents of these slots are marched in full,
    unsigned num_agents;                    // not listed; 0 on the intermediate ticks of f110_tick_repeat
};

__global__ void __launch_bounds__(F110_TTC_SELECT_THREADS) k_ttc_select(const TtcSelectK p) {
    __shared__ unsigned s_cnt, s_base;
    if (threadIdx.x == 0) s_cnt = 0u;
    __syncthreads();
    const unsigned a = blockIdx.x * F110_TTC_SELECT_THREADS + threadIdx.x, lane = threadIdx.x & 31u;
    bool listed = false;
    if (a < p.agents) {
        const double2 r1 = __ldg(p.rec + 4 * (size_t)a + 1), r2 = __ldg(p.rec + 4 * (size_t)a + 2);
        const bool absurd = (unsigned long long)__double_as_longlong(r1.y) == ~0ull;
        const bool clear = r1.x * p.d0_scale > r2.x && p.max_range > r2.x;      // false for a NaN on either side
        listed = (absurd || !clear) && !(p.skip && ((p.skip >> (a % p.num_agents)) & 1u));
    }
    const unsigned vote = __ballot_sync(0xffffffffu, listed);
    unsigned wbase = 0u;
    if (lane == 0 && vote) wbase = atomicAdd(&s_cnt, (unsigned)__popc(vote));
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    __syncthreads();
    if (threadIdx.x == 0 && s_cnt) {
        s_base = atomicAdd(p.count, s_cnt);
        if (p.marched) atomicAdd(p.marched, (unsigned long long)s_cnt);
    }
    __syncthreads();
    if (listed) p.list[s_base + wbase + (unsigned)__popc(vote & ((1u << lane) - 1u))] = a;
}

struct TtcK {
    const double *__restrict__ table;       // CELLS: [L][(H+1)*(W+1)] dt_cells_pad; else [L][H*W] dt in metres
    const double *__restrict__ dt;          // [L][H*W] dt in metres (absurd coordinates)
    const double2 *__restrict__ sincos2;    // [2 * theta_dis] (sin, cos), the LUT stored twice
    const double2 *__restrict__ cos_side;   // [B] (cos(scan_angle_i), side_distance_i)
    const double2 *__restrict__ rec;        // [M][4] per-agent record of k_dynamics
    const uint32_t *__restrict__ list;      // [*count] agents to march
    const uint32_t *__restrict__ count;     // [1]
    int32_t *__restrict__ wall_flag;        // [M]
    unsigned long long *lookup_counter;     // COUNT only
    // canvas stack: per-layer tables (f110_map.layer_geom / layer_res / layer_rot) and the env's layer, or NULL: the values below
    const double *__restrict__ layer_geom;
    const double *__restrict__ layer_res;
    const double *__restrict__ layer_rot;
    const int32_t *__restrict__ env_layer;
    double2 orig, ext, res, rot;            // (orig_x, orig_y), (W res, H res), (res, RN(1 / res)), (orig_c, orig_s)
    double tmax;                            // CELLS: max_range / res; else max_range
    double max_range, eps, ttc_thresh, ttc_margin, inc, theta_dis_f;
    unsigned long long inc_fx;              // theta_index_increment in Q16.48
    unsigned long long layer_stride;        // elements between layers of `dt`
    unsigned long long layer_stride_lean;   // elements between layers of `table`
    unsigned guard32;
    unsigned width, height, last;           // canvas; `last` = width * height - 1 (the metre table's dt[-1,-1])
    unsigned ipa;                           // items per agent: ceil(B / 32)
    unsigned num_agents;
    int B;
};

template <int UNITS, bool COUNT>
__global__ void __launch_bounds__(F110_TTC_THREADS) k_march_ttc(const TtcK p) {
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long items = (unsigned long long)__ldg(p.count) * p.ipa;
    const unsigned long long stride = (unsigned long long)gridDim.x * (F110_TTC_THREADS / 32);
    unsigned looks = 0u;
    for (unsigned long long item = (unsigned long long)blockIdx.x * (F110_TTC_THREADS / 32) + (threadIdx.x >> 5); item < items;
         item += stride) {
        const unsigned a = __ldg(p.list + (unsigned)(item / p.ipa));
        const int i = (int)((unsigned)(item % p.ipa) * 32u + lane);
        if (i >= p.B) continue;
        const double2 *__restrict__ rp = p.rec + 4 * (size_t)a;
        const double2 r0 = __ldg(rp), r1 = __ldg(rp + 1), r2 = __ldg(rp + 2), r3 = __ldg(rp + 3);
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
        // A beam's total only grows and its range is min(total, max_range): once the total exceeds thr (and max_range does),
        // the range will too and the beam cannot fire, so it stops there.  Most beams of a listed agent stop after a lookup or two.
        const double thr = r2.x;
        const bool stops = p.max_range > thr;
        double range;
        unsigned n = 1;
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
                    // off the layer -> its padding on the canvas (or the extra row / column), which holds dt[-1,-1]
                    D = __ldg(table + min(r, p.height) * (p.width + 1u) + min(c, p.width));
                    T = T + D;
                    n++;
                }
                range = ((T > p.tmax) ? p.tmax : T) * p.res.x;
            } else {
                while (__double2hiint(D) != 0 && T <= p.tmax && !(stops && T > thr)) {
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
        if (range <= thr) {
            const double2 cs2 = __ldg(p.cos_side + i);
            ttc_exact(range, r2.y, cs2.x, cs2.y, p.ttc_thresh, p.ttc_margin, p.wall_flag + a);
        }
        if (COUNT) looks += n;
    }
    if (COUNT) {
        const unsigned nsum = __reduce_add_sync(0xffffffffu, looks);
        if (lane == 0 && nsum) atomicAdd(p.lookup_counter, (unsigned long long)nsum);
    }
}

}  // namespace f110
