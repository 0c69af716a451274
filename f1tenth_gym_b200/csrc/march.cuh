// march.cuh — k_march: the production ray-march kernel of f110_step (fast-path maps).
//
// Same arithmetic as lidar.cuh's cell-unit march (bit-identical ranges), specialised for the tick:
//   * 2-D grid (agent, 64-beam block): no integer division, block-uniform pose / velocity loads
//   * everything that is constant for a launch is precomputed on the host into MarchK (kernel params)
//   * interleaved (sin, cos) and (cos_i, side_i) tables: one 16-byte load each
//   * one loop: T starts at 0 and the first iteration performs the pose-cell lookup (0 + D == D exactly)
//   * CODED: 1-byte rank-coded DT table (L1-resident working set) + 2 KB fp64 LUT, escape as a real branch
//   * fp32 range out, fused iTTC predicate with a division-free pre-test, optional Philox noise
// Behavioural spec: reference laser_models.py:106-217 (trace_ray, get_scan, check_ttc_jit).
#pragma once
#include "lidar.cuh"

namespace f110 {

struct MarchK {
    const uint8_t *__restrict__ codes;      // [H*W] or NULL
    const double *__restrict__ lut;         // [256]
    const double *__restrict__ cells;       // [H*W] dt / res
    const double2 *__restrict__ sincos;     // [theta_dis] (sin, cos)
    const double2 *__restrict__ cos_side;   // [B] (cos(scan_angle_i), side_distance_i)
    const double2 *__restrict__ scan_pose;  // [M][2] (x, y), (first lookup d0 in cells, theta_index0)
    const double *__restrict__ vel;         // [M]
    float *__restrict__ out;                // [M][B]
    int32_t *__restrict__ wall_flag;        // [M]
    unsigned long long *lookup_counter;     // COUNT only
    const unsigned long long *tick_counter; // NOISE only
    double ox, oy, eps, tmax;               // cell units
    double inv_res, res;
    double inc, theta_dis_f, ti_guard;
    double ttc_thresh, ttc_margin;          // thresh, thresh * 1.000001
    double noise_std;
    unsigned long long noise_seed;
    unsigned width, height, last;
    int B;
    const int32_t *__restrict__ env_layer;  // [num_envs] map layer of each env, or NULL (single map)
    unsigned long long layer_stride;        // H*W elements between layers of cells / dt
    unsigned num_agents;
    unsigned long long *trace;              // debug: [blocks][4] (smid, t_start_ns, t_end_ns, warp-max steps) or NULL
    const double *__restrict__ dt;          // fp64 DT in metres + metadata: literal-arithmetic fallback
    double orig_x, orig_y, x_max, y_max, dt_oob, eps_m, max_range;
};

// absurd coordinates (|x| >= 1e8 m): the literal reference arithmetic, out of line, all arguments by value
// (taking the address of the kernel parameter struct would spill the whole struct to local memory)
__device__ __noinline__ double march_generic(const double *dt, double orig_x, double orig_y, double x_max,
                                             double y_max, double res, double dt_oob, double eps, double max_range,
                                             int width, double px, double py, double s, double c) {
    MapView m;
    m.dt = dt; m.orig_x = orig_x; m.orig_y = orig_y; m.orig_c = 1.0; m.orig_s = 0.0; m.resolution = res;
    m.x_max = x_max; m.y_max = y_max; m.dt_oob = dt_oob; m.eps = eps; m.max_range = max_range; m.width = width;
    int n;
    return trace_ray<false>(m, px, py, s, c, n);
}

// escape codes are rare (never on a race-track map): keep them out of line so the march loop carries no
// predicated-off instructions for them
__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ unsigned smid() {
    unsigned r;
    asm volatile("mov.u32 %0, %smid;" : "=r"(r));
    return r;
}

__device__ __noinline__ double escape_load(const double *__restrict__ cells, unsigned idx) { return __ldg(cells + idx); }

// Work queue of the persistent march kernel (exactness never depends on it).
// Lookups per beam are heavy-tailed (p50 5, p99 32, max ~300 under the benchmark policy) and a long
// beam is a serial dependent chain (~150 ns per lookup).  With one block per tile of beams the grid's
// makespan was a throughput phase plus a long tail of a few late-dispatched tiles holding a
// 250-lookup beam, and the block dispatcher could not keep all slots filled.  So:
//   * work items are 32 consecutive beams of one agent (one warp); every item records its maximum lookup
//     count, which changes little from tick to tick (>= 99 % of the items with a >= 100-lookup beam had
//     a >= 24-lookup beam one tick earlier);
//   * extra blocks of k_dynamics sort the items into three classes (very heavy >= 64 or unknown; heavy
//     >= 24 incl. neighbours; light) -> queue = [A | B | C], i.e. longest-processing-time-first;
//   * k_march_persistent keeps 64 warps per SM resident; the queue is dealt round-robin to the blocks and
//     the warps of a block pull from it through a shared-memory counter, so there is no block-dispatch
//     gap and the tail consists of light items only.
#define F110_Q_HEAVY 24u
#define F110_Q_VERY_HEAVY 64u
#define F110_Q_UNKNOWN 0xFFFFFFFFu
struct MarchQueue {
    unsigned *__restrict__ cost;            // [M << 8] max lookups of the item in the last tick, by packed id
    const unsigned *__restrict__ order;     // [3][items] class lists of packed items (agent << 8 | slice)
    const unsigned *__restrict__ count;     // [3]
    unsigned items;                         // M * ipa
    unsigned ipa;                           // 32-beam slices per agent (<= 256)
    unsigned chunk_shift;                   // a block is dealt 2^chunk_shift consecutive queue entries at a time
    unsigned *claim;                        // global run counter of the dynamic queue tail (k_march_lean<DYN>), zeroed every tick
    unsigned static_runs;                   // DYN: runs per block that are dealt statically (>= dyn_ahead)
    unsigned dyn_ahead;                     // DYN: how many local runs ahead a dynamic run is claimed (1..8)
    unsigned uniform_ipt4;                  // DYN: 4 / 2 = the queue is long enough for that many entries per ticket throughout, 0 = ticket size by run class (host's choice)
    unsigned ipt_shifts;                    // DYN: log2(queue entries per ticket): very heavy | heavy << 8 | light << 16 | dynamic tail << 24 (255 = by class)
};

// One beam: LUT heading, sphere tracing in cell units, optional noise, iTTC predicate, fp32 range out.
// xy = scan position (m), ti0 = LUT index of beam 0, v = longitudinal velocity of the agent.
// d0 = DT value (cell units) of the pose cell: the first lookup of every beam of the agent, done once per agent
// by k_dynamics instead of once per beam here.
// CELLS = true : resolution 2^-k — march in cell units (see lidar.cuh), d0 / table in cells.
// CELLS = false: any resolution, unrotated origin — march in metres on the reference's own table; the cell index
//   needs RN(t/res) exactly as the reference's `int(x_rot/resolution)` computes it.  With inv = RN(1/res) from the
//   host, q = t*inv; y = fma(fma(-q, res, t), inv, q) is the correctly rounded quotient (the residual-correction
//   tail of the IEEE division algorithm, 3 instructions instead of the ~10 of a full fp64 divide).
// element offset of agent a's map layer inside the stacked DT tables (multi-map batches share one canvas)
__device__ __forceinline__ size_t layer_offset(const MarchK &p, unsigned a) {
    return p.env_layer ? (size_t)p.env_layer[a / p.num_agents] * (size_t)p.layer_stride : (size_t)0;
}

template <bool CODED, bool NOISE, bool CELLS>
__device__ __forceinline__ void march_beam(const MarchK &p, unsigned a, int i, double2 xy, double d0, double ti0,
                                           double v, size_t lo, unsigned &nlook) {
    // the agent's map layer as ONE opaque register pair: otherwise ptxas re-derives (uniform base + 64-bit layer offset
    // + index) on every lookup, 4 address instructions instead of one IMAD.WIDE (loop 27 -> 23 instructions).
    // Things tried on the remaining 4 parameter re-loads per iteration (ptxas rematerialises them; it sees through
    // moves and uniform shuffles): pinning them in registers via volatile shared-memory reads gives a 20-instruction
    // loop but needs 40 registers = 48 warps/SM, and was slower (occupancy beats instruction count here); unrolling
    // the loop by two (21.5 instructions per lookup) was slower too.
    const double *table = (CELLS ? p.cells : p.dt) + lo;
    asm volatile("" : "+l"(table));
    const int ti = beam_theta_index(ti0, i, p.inc, p.theta_dis_f, p.ti_guard);
    const double2 sc = __ldg(p.sincos + ti);
    double range;
    unsigned n = 0;
    if (!CELLS && fabs(xy.x) < 1e8 && fabs(xy.y) < 1e8) {
        const double MAGIC = 6755399441055744.0;
        double X = xy.x, Y = xy.y, T = d0, D = d0;
        n = 1;
#pragma unroll 1
        while (D > p.eps_m && T <= p.max_range) {
            X = X + D * sc.y;
            Y = Y + D * sc.x;
            const double tx = X - p.orig_x, ty = Y - p.orig_y;
            double qx = tx * p.inv_res, qy = ty * p.inv_res;
            qx = __fma_rn(__fma_rn(-qx, p.res, tx), p.inv_res, qx);
            qy = __fma_rn(__fma_rn(-qy, p.res, ty), p.inv_res, qy);
            const int c = __double2loint(__dadd_rd(qx, MAGIC));     // floor == int() for the in-bounds quotients
            const int r = __double2loint(__dadd_rd(qy, MAGIC));
            unsigned idx = (unsigned)r * p.width + (unsigned)c;
            // laser_models.py:79: x_rot < 0 or x_rot >= width*resolution (the fp64 product) -> dt[-1,-1]
            if ((unsigned)c >= p.width || (unsigned)r >= p.height || tx >= p.x_max || ty >= p.y_max) idx = p.last;
            D = __ldg(table + idx);
            T = T + D;
            n++;
        }
        range = (T > p.max_range) ? p.max_range : T;
    } else if (CELLS && fabs(xy.x) < 1e8 && fabs(xy.y) < 1e8) {
        const double MAGIC = 6755399441055744.0;   // 2^52 + 2^51: round-down add == floor in the low word
        double X = xy.x * p.inv_res, Y = xy.y * p.inv_res, T = d0, D = d0;
        n = 1;
#pragma unroll 1
        while (D > p.eps && T <= p.tmax) {
            X = X + D * sc.y;
            Y = Y + D * sc.x;
            const int c = __double2loint(__dadd_rd(X - p.ox, MAGIC));
            const int r = __double2loint(__dadd_rd(Y - p.oy, MAGIC));
            unsigned idx = (unsigned)r * p.width + (unsigned)c;
            if ((unsigned)c >= p.width || (unsigned)r >= p.height) idx = p.last;   // off-map reads dt[-1,-1]
            if (CODED) {
                const unsigned code = __ldg(p.codes + lo + idx);
                if (code == 255u) D = escape_load(p.cells + lo, idx);
                else D = __ldg(p.lut + code);
            } else {
                D = __ldg(table + idx);
            }
            T = T + D;
            n++;
        }
        range = ((T > p.tmax) ? p.tmax : T) * p.res;
    } else {
        range = march_generic(p.dt + lo, p.orig_x, p.orig_y, p.x_max, p.y_max, p.res, __ldg(p.dt + lo + p.last), p.eps_m, p.max_range,
                              (int)p.width, xy.x, xy.y, sc.x, sc.y);
        n = 1;
    }
    nlook = n;
    if (NOISE) {
        const unsigned long long tick = p.tick_counter ? *p.tick_counter : 0ull;
        range = range + p.noise_std * normal_sample(p.noise_seed, tick, (uint64_t)a * (uint64_t)p.B + (uint64_t)i);
    }
    // check_ttc_jit, one beam: hit iff 0 <= fl(d/pv) < thresh.  |d| <= margin*|pv| is a necessary condition,
    // so the exact IEEE division only runs for beams that are about to touch a wall.
    if (v != 0.0) {
        const double2 cs = __ldg(p.cos_side + i);
        const double pv = v * cs.x;
        const double d = range - cs.y;
        if (fabs(d) <= p.ttc_margin * fabs(pv)) {
            const double ttc = d / pv;
            if ((ttc < p.ttc_thresh) && (ttc >= 0.0)) atomicOr(p.wall_flag + a, 1);
        }
    }
    p.out[(size_t)a * (size_t)p.B + (size_t)i] = (float)range;
}

// grid (agents, 64-beam tiles per agent), 64 threads: one tile of one agent per block (no queue)
template <bool CODED, bool NOISE, bool COUNT, int MINB, bool CELLS>
__global__ void __launch_bounds__(64, MINB) k_march(const MarchK p) {
    unsigned long long t0 = 0;
    if (p.trace) t0 = gtime();
    const unsigned a = blockIdx.x;
    const int i = (int)(blockIdx.y * 64u + threadIdx.x);
    if (i >= p.B) return;
    unsigned nlook;
    {
        const double2 xy = __ldg(p.scan_pose + 2 * (size_t)a);
        const double2 yt = __ldg(p.scan_pose + 2 * (size_t)a + 1);
        march_beam<CODED, NOISE, CELLS>(p, a, i, xy, yt.x, yt.y, __ldg(p.vel + a), layer_offset(p, a), nlook);
    }
    if (p.trace || COUNT) {
        const unsigned act = __activemask();
        if (p.trace) {
            const unsigned mx = __reduce_max_sync(act, nlook);
            if (threadIdx.x == 0) {
                unsigned long long *tr = p.trace + 4ull * ((unsigned long long)blockIdx.y * gridDim.x + blockIdx.x);
                tr[0] = smid(); tr[1] = t0; tr[2] = gtime(); tr[3] = mx;
            }
        }
        if (COUNT) {
            const unsigned n = __reduce_add_sync(act, nlook);
            if ((threadIdx.x & 31) == (unsigned)(__ffs(act) - 1)) atomicAdd(p.lookup_counter, (unsigned long long)n);
        }
    }
}

// persistent: gridDim.x blocks of 512 threads stay resident; queue position q = k * gridDim.x + blockIdx.x.
// cost[] is indexed by the packed item id (agent << 8 | slice), so no multiply/divide is needed per item.
// SUB = 32-beam slices per work item (1 or 2): a wider item halves the per-item queue / pose / cost overhead
template <bool CODED, bool NOISE, bool COUNT, bool TRACE, int PT, int SUB, bool CELLS>
__global__ void __launch_bounds__(PT, 4) k_march_persistent(const MarchK p, const MarchQueue mq) {
    __shared__ unsigned s_next;
    if (threadIdx.x == 0) s_next = 0u;
    __syncthreads();
    const unsigned lane = threadIdx.x & 31u;
    const unsigned nA = min(mq.count[0], mq.items), nB = min(mq.count[1], mq.items);
    const unsigned nAB = nA + nB;
    const unsigned total = min(nAB + min(mq.count[2], mq.items), mq.items);
    unsigned looks = 0u;
    for (;;) {
        unsigned k = 0;
        if (lane == 0) k = atomicAdd(&s_next, 1u);
        k = __shfl_sync(0xffffffffu, k, 0);
        // items < 2^32 / 4 (host-checked): no overflow.  Consecutive entries of a class list are neighbouring
        // slices of one agent, so dealing them in runs of 8 lets the warps of a block share L1 lines (faster at cfg2
        // than runs of 4 or 16; also giving the co-resident blocks of an SM neighbouring runs concentrates the heavy
        // items on few SMs and is slower still).
        const unsigned q = ((((k >> mq.chunk_shift) * gridDim.x + blockIdx.x) << mq.chunk_shift)) +
                           (k & ((1u << mq.chunk_shift) - 1u));
        if (q >= total) break;
        unsigned long long t0 = 0;
        if (TRACE) t0 = gtime();
        const unsigned it = mq.order[(q < nA) ? q : (q < nAB) ? (mq.items + (q - nA)) : (2u * mq.items + (q - nAB))];
        const unsigned a = it >> 8;
        const double2 xy = __ldg(p.scan_pose + 2 * (size_t)a);
        const double2 yt = __ldg(p.scan_pose + 2 * (size_t)a + 1);
        const double v = __ldg(p.vel + a);
        const size_t lo = layer_offset(p, a);
        unsigned nlook = 0;
#pragma unroll 1
        for (int sub = 0; sub < SUB; sub++) {
            const int i = (int)(((it & 255u) * SUB + sub) * 32u + lane);
            unsigned n1 = 0;
            if (i < p.B) march_beam<CODED, NOISE, CELLS>(p, a, i, xy, yt.x, yt.y, v, lo, n1);
            nlook = (SUB == 1) ? n1 : max(nlook, n1);
            if (COUNT) looks += n1;
        }
        const unsigned mx = __reduce_max_sync(0xffffffffu, nlook);
        if (lane == 0) {
            mq.cost[it] = mx;
            if (TRACE) {
                unsigned long long *tr = p.trace + 4ull * q;
                tr[0] = smid(); tr[1] = t0; tr[2] = gtime(); tr[3] = mx;
            }
        }
    }
    if (COUNT) {
        const unsigned n = __reduce_add_sync(0xffffffffu, looks);
        if (lane == 0 && n) atomicAdd(p.lookup_counter, (unsigned long long)n);
    }
}

}  // namespace f110
