// march_lean.cuh — k_march_lean: the production ray-march kernel of f110_step / f110_tick (round 2).
//
// Same results as march.cuh's k_march_persistent (bit-identical ranges, same DT lookups), same persistent
// longest-first work queue; what changed is the instruction count.  The round-1 SASS spent
// about half of its warp-instructions per 32-beam work item OUTSIDE the sphere-tracing loop and carried four
// kernel-parameter reloads inside it.  Here:
//   * everything that is constant for an agent is computed once per agent by k_dynamics into a 64-byte record
//     (scan position already in cell units, first lookup, LUT index of beam 0 as Q16.48 fixed point, the iTTC
//     pre-test threshold, the map-layer offset): a work item starts with two 16-byte broadcast loads;
//   * the beam's LUT index is a 64-bit integer multiply-add on that fixed-point value (no I2F / F2I on the XU
//     pipe, no fp64 compare chain); beams whose fractional part is within the proven error bound of an integer
//     replay the reference's sequential recurrence exactly as before (lidar.cuh), out of line;
//   * the sin/cos LUT is stored twice back to back, so the `while theta_index >= theta_dis` wrap is an index, not a
//     branch (needs fov < 2 pi: host-checked);
//   * `d > eps` is an integer test on the high word: every DT value is resolution * sqrt(k) with integer k, so it is
//     either +0.0 or >= resolution > eps (host-checked: resolution > eps >= 0);
//   * the cell-unit tables carry one extra row and column holding dt[-1,-1] (what an off-map lookup reads through
//     numba's negative-index wrap, laser_models.py:79-81): the bounds test is two unsigned min() on the cell
//     coordinates (a negative coordinate is a huge unsigned) instead of two compares, a select and a reload of `last`;
//   * iTTC (laser_models.py:188-217): one compare per beam against a per-agent threshold (range > max side distance
//     + margin * |v| cannot be a hit); the exact test runs out of line for the few beams that are that close;
//   * TABLE = 1: the lookup goes to the 1-byte rank-coded table (32 cells per 32-byte sector instead of 4) and the
//     code is decoded through a 2 KB fp64 LUT in SHARED memory; the escape code decodes to NaN, which ends the loop
//     through the range test, and such a beam (never on a race track) is redone on the fp64 table out of line.
// Behavioural spec: reference laser_models.py:106-217 (trace_ray, get_scan, check_ttc_jit).
#pragma once
#include "march.cuh"

namespace f110 {

struct LeanK {
    const double *__restrict__ table;       // CELLS: [L][(H+1)*(W+1)] dt / res, padded with dt[-1,-1]; else [L][H*W] dt in metres
    const uint8_t *__restrict__ codes;      // [(H+1)*(W+1)] rank codes of the padded table (TABLE = 1), else NULL
    const double *__restrict__ lut;         // [256] code -> table value, lut[255] = NaN
    const double2 *__restrict__ sincos2;    // [2 * theta_dis] (sin, cos), the LUT stored twice
    const double2 *__restrict__ cos_side;   // [B] (cos(scan_angle_i), side_distance_i)
    const double2 *__restrict__ rec;        // [M][4] per-agent record written by k_dynamics (MarchRec)
    float *__restrict__ out;                // [M][B]
    int32_t *__restrict__ wall_flag;        // [M]
    unsigned long long *lookup_counter;     // COUNT only
    const unsigned long long *tick_counter; // NOISE only
    double ox, oy, tmax;                    // CELLS: orig / res, max_range / res; else orig (m), max_range (m)
    double res, inv_res, x_max, y_max;      // metres path (and range scaling of the cell path)
    double ttc_thresh, ttc_margin, noise_std;
    double inc, theta_dis_f;                // replay path
    unsigned long long inc_fx;              // theta_index_increment in Q16.48
    unsigned long long noise_seed;
    unsigned guard32;                       // replay when the fraction (top 32 bits) is within guard32 of an integer
    unsigned width, height, last;           // CELLS: `last` unused, the row stride is width + 1
    unsigned codes_pitch;                   // row pitch of `codes` (>= width + 1, multiple of 16 for TMA)
    int B;
    // literal fallback for absurd coordinates
    const double *__restrict__ dt;
    double orig_x, orig_y;
    unsigned brick_cols1, unused;           // k_march_lean_brick: bricks per row of the brick table, minus one
    double eps_m, max_range;
    unsigned long long layer_stride;        // elements between layers of dt (metres table)
    unsigned long long layer_stride_lean;   // elements between layers of `table`
};

// Element (r, c) of the padded (H+1) x (W+1) cell-unit table in the brick table (f110_march_tables.dt_cells_brick): bricks of
// 4 x 4 cells (128 bytes of fp64, one cache line), row-major over a grid of bw = brick_cols1 + 1 bricks per row, and row-major
// inside a brick: ((r / 4) * bw + c / 4) * 16 + (r % 4) * 4 + c % 4, rearranged to two AND and two multiply-adds
__device__ __forceinline__ unsigned brick_index(unsigned r, unsigned c, unsigned brick_cols1) {
    return ((r & ~3u) * brick_cols1 + r) * 4u + (c & ~3u) * 3u + c;
}

// f110_map_brick: the brick table from the padded row-major table (height + 1 rows of width + 1), thread per element.  Element e
// holds cell (r, c) = ((e / 16) / bw * 4 + e % 16 / 4, (e / 16) % bw * 4 + e % 4); cells beyond the padded table (the rows and
// columns that round it up to whole bricks) hold its last element, dt[-1,-1] / resolution, like the padding itself
__global__ void k_map_brick(const double *__restrict__ pad, unsigned height, unsigned width, unsigned bw, double *__restrict__ out,
                            unsigned n) {
    const unsigned e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const unsigned b = e >> 4;
    const unsigned r = (b / bw) * 4u + ((e >> 2) & 3u), c = (b % bw) * 4u + (e & 3u);
    out[e] = (r <= height && c <= width) ? pad[r * (width + 1u) + c] : pad[height * (width + 1u) + width];
}

// per-agent record, 4 x double2:
//   [0] (X, Y)      scan position: cell units (CELLS) or metres
//   [1] (d0, ti0fx) first DT lookup (same unit), LUT index of beam 0 in Q16.48 (bits), ~0 = absurd coordinates
//   [2] (thr, v)    iTTC pre-test threshold in metres (-inf when v == 0), longitudinal velocity
//   [3] (off, ti0)  element offset of the env's map layer (bits), LUT index of beam 0 as the reference's fp64 value
#define F110_FX_SHIFT 48

__device__ __noinline__ int replay_theta_index(double ti0, int i, double inc, double theta_dis_f) {
    double t = ti0;
    for (int k = 0; k < i; k++) {
        t += inc;
        while (t >= theta_dis_f) t -= theta_dis_f;
    }
    return (int)t;
}

// exact iTTC predicate for one beam (check_ttc_jit, laser_models.py:188-217); v != 0
__device__ __noinline__ void ttc_exact(double range, double v, double cos_i, double side_i, double thresh, double margin,
                                       int32_t *flag) {
    const double pv = v * cos_i;
    const double d = range - side_i;
    if (fabs(d) <= margin * fabs(pv)) {
        const double ttc = d / pv;
        if ((ttc < thresh) && (ttc >= 0.0)) atomicOr(flag, 1);
    }
}

// one beam on the fp64 table, cell units: the escape path of the coded table
__device__ __noinline__ double redo_beam_cells(const double *__restrict__ table, double X, double Y, double d0, double s,
                                               double c, double ox, double oy, double tmax, unsigned width,
                                               unsigned height, unsigned *n_out) {
    const double MAGIC = 6755399441055744.0;
    double T = d0, D = d0;
    unsigned n = 1;
    while (D > 0.0 && T <= tmax) {
        X = X + D * c;
        Y = Y + D * s;
        const int cc = __double2loint(__dadd_rd(X - ox, MAGIC));
        const int rr = __double2loint(__dadd_rd(Y - oy, MAGIC));
        D = __ldg(table + min((unsigned)rr, height) * (width + 1u) + min((unsigned)cc, width));
        T = T + D;
        n++;
    }
    *n_out = n;
    return T;
}

// TABLE: 0 = fp64 table in global memory, 1 = u8 rank codes in global memory + fp64 LUT in shared memory
// DYN: the first mq.static_runs runs (of 2^chunk_shift consecutive queue entries) of every block are dealt statically,
// round-robin, as before; the REST of the queue is handed out dynamically from one global counter (mq.claim).  Static
// dealing gives every block the same number of items but not the same amount of work: some SMs finish early and idle
// until the last block ends.  Claims are prefetched: the warp that draws the first
// ticket of local run r claims the run for r + mq.dyn_ahead and publishes it in a shared-memory ring, so a ticket only reads
// two shared words; the global order of the queue (longest first) is kept.  Two lessons from the A/B measurements:
//   * the ring logic must stay OUT OF LINE (dyn_queue_position): inlined it wrecks the register allocation of the whole item
//     path (a quarter more warp-instructions per launch) and every dynamic flavour loses;
//   * half static / half dynamic was the measured optimum (with 4 x 512 threads per SM, also ahead of the static 2 x 1024
//     shape; a mostly static or a mostly dynamic split is behind): the static half keeps the head of the queue -- the
//     heavy items -- free of claim latency, the dynamic half evens out the blocks.
#define F110_DYN_RING 16u
// common tail of the two ticket -> queue position functions: (local run r, first entry idx of the ticket inside the run,
// log2 entries of the ticket) -> position | (entries - 1) << 29
// RING: how the ring words are handed from the claiming warp to the reading warps -- 0: volatile stores and loads around a
// __threadfence_block (every lane polls: a broadcast read); 1: shared-memory atomics, polled by the elected lane alone (32 lanes
// would be 32 serialized atomics on one word) and broadcast by a shuffle; 2: st.release.cta / ld.acquire.cta.
template <int RING>
__device__ __forceinline__ unsigned dyn_claim_and_locate(unsigned r, unsigned idx, unsigned sh, bool elected, unsigned cs,
                                                         unsigned static_runs, unsigned dyn_ahead, unsigned *claim, unsigned *s_run,
                                                         unsigned *s_seq, unsigned qstride, unsigned qbase, unsigned nblocks) {
    const unsigned nsub1 = ((1u << sh) - 1u) << 29;
    if (idx == 0u && elected && r + dyn_ahead >= static_runs) {
        // first ticket of run r: claim the dynamic run that local run r + dyn_ahead will use
        const unsigned g = atomicAdd(claim, 1u);
        const unsigned nb = (r + dyn_ahead) & (F110_DYN_RING - 1u);
        if (RING == 1) {
            atomicExch(s_run + nb, static_runs * nblocks + g);
            __threadfence_block();
            atomicExch(s_seq + nb, r + dyn_ahead);
        } else if (RING == 2) {
            asm volatile("st.relaxed.cta.shared.u32 [%0], %1;" :: "r"((unsigned)__cvta_generic_to_shared(s_run + nb)), "r"(static_runs * nblocks + g) : "memory");
            asm volatile("st.release.cta.shared.u32 [%0], %1;" :: "r"((unsigned)__cvta_generic_to_shared(s_seq + nb)), "r"(r + dyn_ahead) : "memory");
        } else {
            ((volatile unsigned *)s_run)[nb] = static_runs * nblocks + g;
            __threadfence_block();
            ((volatile unsigned *)s_seq)[nb] = r + dyn_ahead;
        }
    }
    if (r < static_runs) return (r * qstride + qbase + idx) | nsub1;
    const unsigned buf = r & (F110_DYN_RING - 1u);
    // a ring slot is reused 16 runs (>= 32 tickets: the host keeps at least two tickets per run) later: a warp cannot fall that far
    // behind between drawing its ticket and reading the slot; if it ever did, stop loudly instead of marching the wrong items
    unsigned run = 0u, sq;
    if (RING == 1) {
        if (elected) {
            while ((sq = atomicOr(s_seq + buf, 0u)) != r)
                if (sq != 0xFFFFFFFFu && sq > r) __trap();
            __threadfence_block();
            run = atomicOr(s_run + buf, 0u);
        }
        run = __shfl_sync(0xffffffffu, run, __ffs(__ballot_sync(0xffffffffu, elected)) - 1);
    } else if (RING == 2) {
        const unsigned a_seq = (unsigned)__cvta_generic_to_shared(s_seq + buf), a_run = (unsigned)__cvta_generic_to_shared(s_run + buf);
        for (;;) {
            asm volatile("ld.acquire.cta.shared.u32 %0, [%1];" : "=r"(sq) : "r"(a_seq) : "memory");
            if (sq == r) break;
            if (sq != 0xFFFFFFFFu && sq > r) __trap();
        }
        asm volatile("ld.relaxed.cta.shared.u32 %0, [%1];" : "=r"(run) : "r"(a_run) : "memory");
    } else {
        while ((sq = ((volatile unsigned *)s_seq)[buf]) != r)
            if (sq != 0xFFFFFFFFu && sq > r) __trap();
        run = ((volatile unsigned *)s_run)[buf];
    }
    return ((run << cs) + idx) | nsub1;
}
// every ticket covers 2^sh consecutive queue entries (a run of 2^cs entries is 2^(cs - sh) tickets)
template <int RING>
__device__ __noinline__ unsigned dyn_queue_position(unsigned k, bool elected, unsigned cs, unsigned static_runs, unsigned dyn_ahead,
                                                    unsigned *claim, unsigned *s_run, unsigned *s_seq, unsigned qstride,
                                                    unsigned qbase, unsigned nblocks, unsigned sh) {
    const unsigned r = k >> (cs - sh), idx = (k & ((1u << (cs - sh)) - 1u)) << sh;
    return dyn_claim_and_locate<RING>(r, idx, sh, elected, cs, static_runs, dyn_ahead, claim, s_run, s_seq, qstride, qbase, nblocks);
}
// Ticket size by the class of the run (k_march_lean<IPT = 0>).  The queue holds the very heavy entries first, then the heavy,
// then the light ones: a ticket of four consecutive VERY HEAVY entries puts four of the longest marches of the launch on one
// warp, one after the other -- a constant addition to the critical path at every batch size (4 entries per ticket won at
// cfg3 and lost at cfg2x2) -- while for the light entries the pop and this call are a large part of the work.
// zone[] (shared memory, written by thread 0 before the first pop): ticket bounds T1 <= T2 <= T3 of the block's static runs
// that start in the very heavy / heavy / light part of the queue, the run counts rA, rAB behind them, and the four shifts
// (very heavy | heavy << 8 | light << 16 | dynamic tail << 24).
template <int RING>
__device__ __noinline__ unsigned dyn_queue_position_zoned(unsigned k, bool elected, unsigned cs, unsigned static_runs,
                                                          unsigned dyn_ahead, unsigned *claim, unsigned *s_run, unsigned *s_seq,
                                                          unsigned qstride, unsigned qbase, unsigned nblocks, const unsigned *zone) {
    const unsigned shifts = zone[5];
    unsigned sh, r0;
    if (k < zone[0]) { sh = shifts & 255u; r0 = 0u; }
    else if (k < zone[1]) { sh = (shifts >> 8) & 255u; r0 = zone[3]; k -= zone[0]; }
    else if (k < zone[2]) { sh = (shifts >> 16) & 255u; r0 = zone[4]; k -= zone[1]; }
    else { sh = shifts >> 24; r0 = static_runs; k -= zone[2]; }
    const unsigned r = r0 + (k >> (cs - sh)), idx = (k & ((1u << (cs - sh)) - 1u)) << sh;
    return dyn_claim_and_locate<RING>(r, idx, sh, elected, cs, static_runs, dyn_ahead, claim, s_run, s_seq, qstride, qbase, nblocks);
}
// CL > 1: the kernel is launched in thread-block clusters of CL CTAs that share ONE ticket counter (the shared-memory word of
// the cluster's rank-0 CTA, popped through distributed shared memory: mapa + atom.shared::cluster).  The queue is then dealt
// statically to the CLUSTERS and handed out dynamically inside each: a pool of CL x PT/32 warps on several SMs of one GPC
// instead of PT/32 warps on one SM, which evens out the finishing times without the global atomics that made the fully
// dynamic queue lose.
// IPT: queue entries per ticket (1, 2 or 4; 0 = by the class of the run, mq.ipt_shifts, dynamic queue only).  With 2, a warp that
// pops the block's counter marches two consecutive entries of its run before it pops again: the pop, the queue arithmetic and
// the dynamic-queue call are paid once per 64 beams.
// BRICK (k_march_lean_brick): `table` is the same padded cell-unit table stored in 4 x 4-cell bricks (brick_index)
template <int TABLE, bool NOISE, bool COUNT, bool CELLS, bool LAYERED, int PT, int MINB, bool DYN, int CL, int IPT, int RING, bool BRICK>
__device__ __forceinline__ void march_lean_body(const LeanK &p, const MarchQueue &mq) {
    static_assert(!BRICK || (TABLE == 0 && CELLS && !LAYERED), "the brick table is a single fp64 cell-unit map");
    __shared__ unsigned s_next;
    __shared__ unsigned s_run[DYN ? F110_DYN_RING : 1u], s_seq[DYN ? F110_DYN_RING : 1u];
    if (DYN && threadIdx.x < F110_DYN_RING) s_seq[threadIdx.x] = 0xFFFFFFFFu;
    __shared__ double s_lut[TABLE == 1 ? 256 : 1];
    __shared__ unsigned s_zone[(DYN && IPT == 0) ? 6 : 1];
    if (threadIdx.x == 0) s_next = 0u;
    if (TABLE == 1)
        for (unsigned t = threadIdx.x; t < 256u; t += PT) s_lut[t] = p.lut[t];
    // everything above touches only launch constants: under PDL it overlaps the end of k_dynamics.  From here on the
    // kernel reads what k_dynamics wrote (queue, per-agent records).
    pdl_wait();
    pdl_launch_dependents();
    if (DYN && IPT == 0 && threadIdx.x == 0) {
        // ticket sizes by queue class (dyn_queue_position_zoned).  Static run r of this block starts at queue entry
        // (r * gridDim.x + blockIdx.x) << cs: count the runs that start below each class boundary.
        const unsigned zA = min(mq.count[0], mq.items), zAB = zA + min(mq.count[1], mq.items);
        const unsigned zcs = mq.chunk_shift, sr = mq.static_runs;
        const unsigned gA = (zA + (1u << zcs) - 1u) >> zcs, gAB = (zAB + (1u << zcs) - 1u) >> zcs;
        const unsigned rA = gA > blockIdx.x ? min((gA - blockIdx.x + gridDim.x - 1u) / gridDim.x, sr) : 0u;
        const unsigned rAB = gAB > blockIdx.x ? min((gAB - blockIdx.x + gridDim.x - 1u) / gridDim.x, sr) : 0u;
        const unsigned shA = mq.ipt_shifts & 255u, shB = (mq.ipt_shifts >> 8) & 255u, shC = (mq.ipt_shifts >> 16) & 255u;
        unsigned shD = mq.ipt_shifts >> 24;
        if (shD == 255u) {      // by the class the dynamic tail starts in
            const unsigned long long d0 = ((unsigned long long)sr * gridDim.x) << zcs;
            shD = d0 < zA ? shA : d0 < zAB ? shB : shC;
        }
        s_zone[0] = rA << (zcs - shA);
        s_zone[1] = s_zone[0] + ((rAB - rA) << (zcs - shB));
        s_zone[2] = s_zone[1] + ((sr - rAB) << (zcs - shC));
        s_zone[3] = rA;
        s_zone[4] = rAB;
        s_zone[5] = (mq.ipt_shifts & 0xFFFFFFu) | (shD << 24);
    }
    __syncthreads();
    const unsigned lane = threadIdx.x & 31u;
    const unsigned nA = min(mq.count[0], mq.items), nB = min(mq.count[1], mq.items);
    const unsigned nAB = nA + nB;
    const unsigned total = min(nAB + min(mq.count[2], mq.items), mq.items);
    const unsigned cs = mq.chunk_shift;
    const unsigned qstride = (gridDim.x / (unsigned)CL) << cs, qbase = (blockIdx.x / (unsigned)CL) << cs, qmask = (1u << cs) - 1u;
    unsigned s_next_addr = (unsigned)__cvta_generic_to_shared(&s_next);
    if (CL > 1) {
        // every CTA pops the counter of the cluster's rank-0 CTA; it was zeroed before the __syncthreads above, the cluster
        // barrier makes that visible to the other CTAs before their first pop
        asm volatile("mapa.shared::cluster.u32 %0, %0, 0;" : "+r"(s_next_addr));
        asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    }
    unsigned looks = 0u;
    for (;;) {
        // one elected lane pops the block's queue.  (An atomicAdd inside `if (lane == 0)` makes ptxas emit its
        // warp-aggregation sequence -- vote, find-leader, two popc, shuffle: 14 extra instructions per item.)
        unsigned k = 0, leader;
        if (CL > 1)
            asm volatile("{\n\t.reg .pred p;\n\telect.sync %1|p, 0xffffffff;\n\t@p atom.shared::cluster.add.u32 %0, [%2], 1;\n\t}"
                         : "+r"(k), "=r"(leader) : "r"(s_next_addr) : "memory");
        else
            asm volatile("{\n\t.reg .pred p;\n\telect.sync %1|p, 0xffffffff;\n\t@p atom.shared.add.u32 %0, [%2], 1;\n\t}"
                         : "+r"(k), "=r"(leader) : "r"(s_next_addr) : "memory");
        k = __shfl_sync(0xffffffffu, k, leader);
        unsigned q, nsub = (unsigned)IPT;
        if (DYN) {
            // out of line: inlined, the ring logic costs the whole item path its register allocation (ncu: 55.4 M instead of
            // 43.6 M warp-instructions per launch at cfg2 -- the clamp and the store of every beam grew)
            if (IPT == 0) {
                q = dyn_queue_position_zoned<RING>(k, lane == leader, cs, mq.static_runs, mq.dyn_ahead, mq.claim, s_run, s_seq, qstride,
                                             qbase, gridDim.x, s_zone);
                nsub = (q >> 29) + 1u;
            } else
                q = dyn_queue_position<RING>(k, lane == leader, cs, mq.static_runs, mq.dyn_ahead, mq.claim, s_run, s_seq, qstride, qbase,
                                       gridDim.x, IPT == 4 ? 2u : IPT == 2 ? 1u : 0u);
            q &= 0x1FFFFFFFu;
        } else {
            if (IPT == 4) q = (k >> (cs - 2u)) * qstride + qbase + ((k & (qmask >> 2)) << 2);
            else if (IPT == 2) q = (k >> (cs - 1u)) * qstride + qbase + ((k & (qmask >> 1)) << 1);
            else q = (k >> cs) * qstride + qbase + (k & qmask);
        }
        if (q >= total) break;
#pragma unroll 1
        for (unsigned sub = 0; sub < nsub; sub++, q++) {
        if (IPT != 1 && q >= total) break;
        const unsigned it = mq.order[(q < nA) ? q : (q < nAB) ? (mq.items + (q - nA)) : (2u * mq.items + (q - nAB))];
        const unsigned a = it >> 8;
        const int i = (int)((it & 255u) * 32u + lane);
        const double2 *__restrict__ rp = p.rec + 4 * (size_t)a;
        const double2 r0 = __ldg(rp), r1 = __ldg(rp + 1);
        const unsigned long long ti0fx = (unsigned long long)__double_as_longlong(r1.y);
        unsigned n = 0;
        if (i < p.B) {
            double range;
            if (ti0fx != ~0ull) {
                const unsigned long long vfx = ti0fx + (unsigned long long)(unsigned)i * p.inc_fx;
                unsigned ti = (unsigned)(vfx >> F110_FX_SHIFT);
                const unsigned fr = (unsigned)(vfx >> (F110_FX_SHIFT - 32));
                if (fr + p.guard32 <= 2u * p.guard32)
                    ti = (unsigned)replay_theta_index(__ldg(rp + 3).y, i, p.inc, p.theta_dis_f);
                const double2 sc = __ldg(p.sincos2 + ti);
                const double *__restrict__ table = p.table;
                if (LAYERED) table += (unsigned long long)__double_as_longlong(__ldg(rp + 3).x);
                asm volatile("" : "+l"(table));
                const double MAGIC = 6755399441055744.0;   // 2^52 + 2^51: round-down add == floor in the low word
                double X = r0.x, Y = r0.y, T = r1.x, D = r1.x;
                n = 1;
                if (CELLS) {
                    if (__double2hiint(D) != 0 && T <= p.tmax) {
#pragma unroll 1
                        do {
                            X = X + D * sc.y;
                            Y = Y + D * sc.x;
                            const unsigned c = (unsigned)__double2loint(__dadd_rd(X - p.ox, MAGIC));
                            const unsigned r = (unsigned)__double2loint(__dadd_rd(Y - p.oy, MAGIC));
                            // off-map -> the padding row / column, which holds dt[-1,-1]
                            if (TABLE == 1) D = s_lut[__ldg(p.codes + min(r, p.height) * p.codes_pitch + min(c, p.width))];
                            else if (BRICK) D = __ldg(table + brick_index(min(r, p.height), min(c, p.width), p.brick_cols1));
                            else D = __ldg(table + min(r, p.height) * (p.width + 1u) + min(c, p.width));
                            T = T + D;
                            n++;
                        } while (__double2hiint(D) != 0 && T <= p.tmax);
                    }
                    if (TABLE == 1 && T != T) {     // escape code on the way: redo this beam on the fp64 table
                        T = redo_beam_cells(table, r0.x, r0.y, r1.x, sc.x, sc.y, p.ox, p.oy, p.tmax, p.width, p.height, &n);
                    }
                    range = ((T > p.tmax) ? p.tmax : T) * p.res;
                } else {
                    if (__double2hiint(D) != 0 && T <= p.tmax) {
#pragma unroll 1
                        do {
                            X = X + D * sc.y;
                            Y = Y + D * sc.x;
                            const double tx = X - p.ox, ty = Y - p.oy;
                            double qx = tx * p.inv_res, qy = ty * p.inv_res;
                            qx = __fma_rn(__fma_rn(-qx, p.res, tx), p.inv_res, qx);     // RN(tx / res), see march.cuh
                            qy = __fma_rn(__fma_rn(-qy, p.res, ty), p.inv_res, qy);
                            const int c = __double2loint(__dadd_rd(qx, MAGIC));
                            const int r = __double2loint(__dadd_rd(qy, MAGIC));
                            unsigned idx = (unsigned)r * p.width + (unsigned)c;
                            if ((unsigned)c >= p.width || (unsigned)r >= p.height || tx >= p.x_max || ty >= p.y_max) idx = p.last;
                            D = __ldg(table + idx);
                            T = T + D;
                            n++;
                        } while (__double2hiint(D) != 0 && T <= p.tmax);
                    }
                    range = (T > p.tmax) ? p.tmax : T;
                }
            } else {
                // absurd coordinates (|x| >= 1e8 m): the literal reference arithmetic, out of line
                const double2 r3 = __ldg(rp + 3);
                const size_t lo = LAYERED ? (size_t)((unsigned long long)__double_as_longlong(r3.x) / p.layer_stride_lean * p.layer_stride) : (size_t)0;
                const int ti = beam_theta_index(r3.y, i, p.inc, p.theta_dis_f, 1e-6);
                const double2 sc = __ldg(p.sincos2 + ti);
                range = march_generic(p.dt + lo, p.orig_x, p.orig_y, p.x_max, p.y_max, p.res, __ldg(p.dt + lo + p.last), p.eps_m,
                                      p.max_range, (int)p.width, r0.x, r0.y, sc.x, sc.y);
                n = 1;
            }
            if (NOISE) {
                const unsigned long long tick = p.tick_counter ? *p.tick_counter : 0ull;
                range = range + p.noise_std * normal_sample(p.noise_seed, tick, (uint64_t)a * (uint64_t)p.B + (uint64_t)i);
            }
            const double2 r2 = __ldg(rp + 2);
            if (range <= r2.x) {
                const double2 cs2 = __ldg(p.cos_side + i);
                ttc_exact(range, r2.y, cs2.x, cs2.y, p.ttc_thresh, p.ttc_margin, p.wall_flag + a);
            }
            p.out[a * (unsigned)p.B + (unsigned)i] = (float)range;      // M * B < 2^32 (host-checked)
        }
        if (COUNT) looks += n;
        const unsigned mx = __reduce_max_sync(0xffffffffu, n);
        if (lane == 0) mq.cost[it] = mx;
        }
    }
    if (COUNT) {
        const unsigned nsum = __reduce_add_sync(0xffffffffu, looks);
        if (lane == 0 && nsum) atomicAdd(p.lookup_counter, (unsigned long long)nsum);
    }
    // the rank-0 CTA's shared memory must outlive the last pop of every CTA of the cluster
    if (CL > 1) asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

template <int TABLE, bool NOISE, bool COUNT, bool CELLS, bool LAYERED, int PT, int MINB, bool DYN = false, int CL = 1, int IPT = 1, int RING = 0>
__global__ void __launch_bounds__(PT, MINB) k_march_lean(const LeanK p, const MarchQueue mq) {
    march_lean_body<TABLE, NOISE, COUNT, CELLS, LAYERED, PT, MINB, DYN, CL, IPT, RING, false>(p, mq);
}

// k_march_lean on the bricked cell-unit table (f110_march_tables.dt_cells_brick): one fp64 map in cell units, not layered
template <bool NOISE, bool COUNT, int PT, int MINB, bool DYN, int IPT, int RING>
__global__ void __launch_bounds__(PT, MINB) k_march_lean_brick(const LeanK p, const MarchQueue mq) {
    march_lean_body<0, NOISE, COUNT, true, false, PT, MINB, DYN, 1, IPT, RING, true>(p, mq);
}

}  // namespace f110
