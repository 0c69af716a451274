// f110_b200.cu — kernels and C ABI of libf110_b200.so (see include/f110_b200.h).
//
// One tick (reference base_classes.py:553-612 Simulator.step) = three launches on the caller's stream:
//   k_dynamics     thread per agent     steer FIFO, pid, RK4/Euler, yaw wrap, scan pose, pose snapshot, the per-agent record of
//                                       the march (+ extra blocks that sort last tick's work items into the march queue)
//   k_march_lean   persistent, warp per 32-beam item (march_lean.cuh): LUT heading, sphere tracing on the DT grid, fused iTTC
//                                       predicate, optional seeded noise, fp32 range out -- the roofline kernel.  Stand-alone
//                                       scans run the literal k_raymarch (thread per beam); canvas stacks of maps with
//                                       different sizes / origins run k_march_lean_het (march_het.cuh), maps with a rotated
//                                       origin, alone or stacked, k_march_lean_rot (march_rot.cuh).  f110_scan_layers runs
//                                       k_scan_lean (scan_lean.cuh): arbitrary poses, each on its own layer of any map
//   k_tail         warp per agent       GJK vs. the other agents of the env, wall-hit state zeroing, opponent ray-cast inside the
//                                       blocked-view window, collisions obs, then lap logic and auto-reset per env
//                                       (k_finalize = the same without the env-level part, for f110_step)
// f110_tick_repeat holds one action for K ticks: the last is the tick above, the others run k_dynamics, k_ttc_select, k_march_ttc
// (march_ttc.cuh: only the agents a wall could stop, for the iTTC flag alone) and k_tail_noscan.
// Host side of a tick (step_impl): validate -> classify_map (MapGeom: the map-geometry rules, shared with f110_scan_layers and
// f110_render_views) -> plan_march (MarchPlan: kernel family, block shape, queue sizing; the only reader of the debug variant)
// -> k_dynamics -> launch_march_plan (a switch on the family) -> launch_tail -> the launch record, written from the plan.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false (no FMA contraction).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <algorithm>
#include <type_traits>

#include "../../include/f110_b200.h"
#include "../../include/f110_episodes.h"
#include "../../include/f110_episode_repeat.h"
#include "../../include/f110_param_draw.h"
#include "../../include/f110_predict.h"
#include "../../include/f110_mppi.h"
#include "collision.cuh"
#include "dynamics.cuh"
#include "lidar.cuh"
#include "march.cuh"
#include "march_lean.cuh"
#include "march_het.cuh"
#include "march_rot.cuh"
#include "scan_lean.cuh"
#include "march_ttc.cuh"
#include "render.cuh"
#include "march_tile.cuh"
#include "planner.cuh"
#include "progress.cuh"
#include "edt.cuh"
#include "trackgen.cuh"

namespace f110 {

static thread_local char g_cuda_err[256] = "";

static int cuda_fail(cudaError_t e, const char *where) {
    snprintf(g_cuda_err, sizeof(g_cuda_err), "%s: %s", where, cudaGetErrorString(e));
    return F110_ERR_CUDA;
}
#define CUDA_TRY(call)                                                   \
    do {                                                                 \
        cudaError_t e__ = (call);                                        \
        if (e__ != cudaSuccess) return cuda_fail(e__, #call);            \
    } while (0)
#define LAUNCH_CHECK(name)                                               \
    do {                                                                 \
        cudaError_t e__ = cudaGetLastError();                            \
        if (e__ != cudaSuccess) return cuda_fail(e__, name);             \
    } while (0)

static MapView make_view(const f110_map *m) {
    MapView v;
    v.dt = m->dt; v.dt_cells = m->dt_cells; v.dt_codes = m->dt_codes; v.dt_lut = m->dt_lut;
    v.sines = m->sines; v.cosines = m->cosines;
    v.orig_x = m->orig_x; v.orig_y = m->orig_y; v.orig_c = m->orig_c; v.orig_s = m->orig_s;
    v.resolution = m->resolution; v.inv_resolution = 1.0 / m->resolution;
    v.x_max = m->width * m->resolution;    // `width * resolution` (laser_models.py:79)
    v.y_max = m->height * m->resolution;
    v.eps = m->eps; v.max_range = m->max_range; v.dt_oob = m->dt_oob;
    v.theta_dis = m->theta_dis; v.theta_dis_f = (double)m->theta_dis;
    v.height = m->height; v.width = m->width;
    return v;
}

struct BeamView {
    const double *__restrict__ scan_angles;
    const double *__restrict__ cosines;
    const double *__restrict__ side_distances;
    double fov, angle_increment, theta_index_increment;
    int32_t num_beams;
};
static BeamView make_view(const f110_beams *b) {
    BeamView v;
    v.scan_angles = b->scan_angles; v.cosines = b->cosines; v.side_distances = b->side_distances;
    v.fov = b->fov; v.angle_increment = b->angle_increment; v.theta_index_increment = b->theta_index_increment;
    v.num_beams = b->num_beams;
    return v;
}

// Work queue of the persistent march kernel (march.cuh): sort the 32-beam items into [very heavy | heavy |
// light] by the maximum lookup count they recorded in the previous tick.  One thread per item; runs as the
// extra blocks of k_dynamics (it only reads march_cost, which the reset kernels mark as unknown).
#define F110_ORDER_ITEMS_PER_THREAD 8
__device__ __forceinline__ void build_march_order(const f110_sim &s, unsigned first_block, unsigned items) {
    // Round 2 (the builder was most of k_dynamics' instructions at cfg3 -- 24 ballots
    // and up to 24 shared atomics per thread, a runtime division per item): a thread owns EIGHT CONSECUTIVE items, so
    //   * one division per thread (the items after the first step (agent, slice) incrementally),
    //   * the neighbours of an item are the thread's own registers (only the two ends are extra loads: 10 loads, not 24),
    //   * the per-class counts of a thread are packed into one word (3 x 10 bits) and ONE warp scan places all of them,
    //   * a warp touches the three shared counters once, the block the three global ones once,
    // and a class list is in item order within a block, i.e. consecutive entries are neighbouring slices of one agent.
    __shared__ unsigned s_cnt[3], s_base[3];
    const unsigned lane = threadIdx.x & 31u;
    const unsigned ipa = (unsigned)s.march_ipa;
    if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0u;
    const unsigned t = (blockIdx.x - first_block) * blockDim.x + threadIdx.x;
    const unsigned w0 = t * F110_ORDER_ITEMS_PER_THREAD;
    unsigned packed[F110_ORDER_ITEMS_PER_THREAD], c[F110_ORDER_ITEMS_PER_THREAD + 2];
    int cls[F110_ORDER_ITEMS_PER_THREAD];
    unsigned a = 0, j = 0;
    if (w0 < items) { a = w0 / ipa; j = w0 - a * ipa; }
    // c[0] = left neighbour of the first item, c[1..8] = the items, c[9] = right neighbour of the last one
    c[0] = (w0 < items && j > 0) ? s.march_cost[((a << 8) | j) - 1u] : F110_Q_UNKNOWN;
    unsigned aa = a, jj = j;
#pragma unroll
    for (int k = 0; k < F110_ORDER_ITEMS_PER_THREAD; k++) {
        const bool live = w0 + (unsigned)k < items;
        packed[k] = (aa << 8) | jj;
        c[k + 1] = live ? s.march_cost[packed[k]] : F110_Q_UNKNOWN;
        cls[k] = live ? 0 : -1;
        if (++jj == ipa) { jj = 0; aa++; }
    }
    {
        const unsigned wl = w0 + F110_ORDER_ITEMS_PER_THREAD;      // the item after this thread's last one
        c[F110_ORDER_ITEMS_PER_THREAD + 1] = (wl < items && jj > 0) ? s.march_cost[(aa << 8) | jj] : F110_Q_UNKNOWN;
    }
    unsigned mine = 0u;                                             // per-class counts, 10 bits each
#pragma unroll
    for (int k = 0; k < F110_ORDER_ITEMS_PER_THREAD; k++) {
        if (cls[k] == 0) {
            const unsigned sj = packed[k] & 255u;
            unsigned m = c[k + 1];
            if (m != F110_Q_UNKNOWN) {
                // neighbours only inside the same agent: slice 0 has no left one, slice ipa-1 no right one
                if (sj > 0 && c[k] != F110_Q_UNKNOWN) m = max(m, c[k]);
                if (sj + 1 < ipa && c[k + 2] != F110_Q_UNKNOWN) m = max(m, c[k + 2]);
            }
            cls[k] = (c[k + 1] == F110_Q_UNKNOWN || c[k + 1] >= F110_Q_VERY_HEAVY) ? 0 : (m >= F110_Q_HEAVY) ? 1 : 2;
            mine += 1u << (10 * cls[k]);
        }
    }
    // exclusive warp scan of the packed counts (a warp holds at most 256 items per class: 9 bits)
    unsigned incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)lane >= o) incl += v;
    }
    const unsigned excl = incl - mine;
    const unsigned wtot = __shfl_sync(0xffffffffu, incl, 31);
    __syncthreads();                                                // s_cnt zeroed
    unsigned wbase = 0u;                                            // lanes 0..2 fetch the warp's base of class `lane`
    if (lane < 3u) {
        const unsigned n = (wtot >> (10 * lane)) & 1023u;
        wbase = n ? atomicAdd(&s_cnt[lane], n) : 0u;
    }
    const unsigned b0 = __shfl_sync(0xffffffffu, wbase, 0), b1 = __shfl_sync(0xffffffffu, wbase, 1),
                   b2 = __shfl_sync(0xffffffffu, wbase, 2);
    __syncthreads();
    if (threadIdx.x < 3) s_base[threadIdx.x] = s_cnt[threadIdx.x] ? atomicAdd(s.march_count + threadIdx.x, s_cnt[threadIdx.x]) : 0u;
    __syncthreads();
    unsigned pos[3] = { s_base[0] + b0 + (excl & 1023u), s_base[1] + b1 + ((excl >> 10) & 1023u),
                        s_base[2] + b2 + ((excl >> 20) & 1023u) };
#pragma unroll
    for (int k = 0; k < F110_ORDER_ITEMS_PER_THREAD; k++) {
        if (cls[k] >= 0) {
            const unsigned at = (cls[k] == 0) ? pos[0]++ : (cls[k] == 1) ? pos[1]++ : pos[2]++;
            if (at < items) s.march_order[(size_t)cls[k] * items + at] = packed[k];
        }
    }
}

// Agent-level queue of the tile march kernel (march_tile.cuh): one thread per agent classifies it by the largest
// per-slice lookup maximum of the previous tick (unknown = very heavy), same three classes, lists in march_order[3][M].
__device__ __forceinline__ void build_agent_order(const f110_sim &s, unsigned first_block, unsigned agents) {
    __shared__ unsigned s_cnt[3], s_base[3];
    if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0u;
    __syncthreads();
    const unsigned a = (blockIdx.x - first_block) * blockDim.x + threadIdx.x;
    int cls = -1;
    unsigned slot = 0;
    if (a < agents) {
        unsigned m = 0;
        for (int j = 0; j < s.march_ipa; j++) m = max(m, s.march_cost[((size_t)a << 8) + (size_t)j]);     // unknown = 0xFFFFFFFF wins
        cls = (m >= F110_Q_VERY_HEAVY) ? 0 : (m >= F110_Q_HEAVY) ? 1 : 2;
        slot = atomicAdd(&s_cnt[cls], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 3) s_base[threadIdx.x] = s_cnt[threadIdx.x] ? atomicAdd(s.march_count + threadIdx.x, s_cnt[threadIdx.x]) : 0u;
    __syncthreads();
    if (cls >= 0) {
        const unsigned at = s_base[cls] + slot;
        if (at < agents) s.march_order[(size_t)cls * agents + at] = a;
    }
}

// ------------------------------------------------------------------------------------ k_dynamics
struct FirstLookup {
    const double *__restrict__ cells;    // dt / res (cell units) or dt (metres), or NULL: generic march kernel
    double ox, oy, inv_res;              // cell units
    double res, orig_x, orig_y, x_max, y_max;   // metres
    unsigned width, height, last;
    int metres;
    const int32_t *__restrict__ env_layer;   // multi-map batches: layer of each env, or NULL
    unsigned long long layer_stride;
    // per-agent record of the lean march kernel (march_lean.cuh); rec == NULL: not written
    double2 *__restrict__ rec;
    double side_max, ttc_margin;
    unsigned long long rec_layer_stride;     // elements between map layers of the table the lean kernel reads
    int agent_queue;                         // 1: the extra blocks build the agent-level queue of the tile march kernel
    const double *__restrict__ layer_geom;   // canvas stack (f110_map.layer_geom): [L][6] per-layer origin and extent, or NULL
    const double *__restrict__ layer_res;    // canvas stack of several resolutions (f110_map.layer_res): [L][2], or NULL
    const double *__restrict__ layer_rot;    // canvas stack with rotated origins (f110_map.layer_rot): [L][2], or NULL
    double orig_c, orig_s;                   // one metre map with a rotated origin (rotated = 1)
    int rotated;
};

__global__ void __launch_bounds__(128) k_dynamics(f110_sim s, const double *__restrict__ actions, double fov,
                                                  double theta_dis_f, int dyn_blocks, FirstLookup fl) {
    const int NA = s.num_envs * s.num_agents;
    pdl_launch_dependents();                 // the march kernel may start its launch / prologue now (it waits before reading)
    if ((int)blockIdx.x >= dyn_blocks) {     // extra blocks: build the march work queue (block-uniform branch)
        if (fl.agent_queue) build_agent_order(s, (unsigned)dyn_blocks, (unsigned)NA);
        else build_march_order(s, (unsigned)dyn_blocks, (unsigned)NA * (unsigned)s.march_ipa);
        return;
    }
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= NA) return;
    // the tick counter advances once per tick, here, before any kernel of the tick reads it (noise stream id,
    // auto-reset draw); nothing else in this kernel uses it
    if (a == 0 && s.tick_counter) *s.tick_counter += 1ull;
    const double *p = s.params + (size_t)(s.params_per_env ? a : a % s.num_agents) * F110_NPARAM;
    double st[7];
#pragma unroll
    for (int k = 0; k < 7; k++) st[k] = s.state[(size_t)k * NA + a];
    // steering delay FIFO (base_classes.py:270-278): depth 2, zeros until two commands are queued
    const double raw_steer = actions[2 * (size_t)a], speed = actions[2 * (size_t)a + 1];
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

// ------------------------------------------------------------------------------------ k_lidar_order (f110_lidar)
// The march queue of a tick with a lidar mask: build_march_order over the items of the agents whose slot has a lidar only.
// Item w of N * slots * ipa is slice w % ipa of the (w / ipa)-th such agent, envs in order and the slots of an env in ascending
// order; entries keep the (agent << 8 | slice) encoding, so the march kernels run unchanged.  A launch of its own after
// k_dynamics (which then has no queue-building blocks): an instance of k_dynamics with a mask-aware builder changes the code of
// the k_dynamics every tick without a mask runs.  The statements are build_march_order's except where an item's agent is found.
struct LidarOrder {
    uint32_t mask;           // bit i: slot i has a lidar (no bit at or above num_agents)
    unsigned slots;          // popcount of mask, >= 1
};
__device__ __forceinline__ unsigned lidar_agent(unsigned r, const LidarOrder &lo, unsigned A) {
    const unsigned e = r / lo.slots, k = r - e * lo.slots;
    unsigned m = lo.mask;
    for (unsigned i = 0; i < k; i++) m &= m - 1u;          // drop the k lowest set bits: the k-th lidar slot is the lowest left
    return e * A + (unsigned)(__ffs((int)m) - 1);
}
__global__ void __launch_bounds__(128) k_lidar_order(f110_sim s, LidarOrder lo) {
    __shared__ unsigned s_cnt[3], s_base[3];
    const unsigned items = (unsigned)s.num_envs * lo.slots * (unsigned)s.march_ipa;
    const unsigned A = (unsigned)s.num_agents;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned ipa = (unsigned)s.march_ipa;
    if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0u;
    const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned w0 = t * F110_ORDER_ITEMS_PER_THREAD;
    unsigned packed[F110_ORDER_ITEMS_PER_THREAD], c[F110_ORDER_ITEMS_PER_THREAD + 2];
    int cls[F110_ORDER_ITEMS_PER_THREAD];
    unsigned a = 0, j = 0, r = 0;
    if (w0 < items) { r = w0 / ipa; j = w0 - r * ipa; a = lidar_agent(r, lo, A); }
    c[0] = (w0 < items && j > 0) ? s.march_cost[((a << 8) | j) - 1u] : F110_Q_UNKNOWN;
    unsigned aa = a, jj = j;
#pragma unroll
    for (int k = 0; k < F110_ORDER_ITEMS_PER_THREAD; k++) {
        const bool live = w0 + (unsigned)k < items;
        packed[k] = (aa << 8) | jj;
        c[k + 1] = live ? s.march_cost[packed[k]] : F110_Q_UNKNOWN;
        cls[k] = live ? 0 : -1;
        if (++jj == ipa) { jj = 0; aa = lidar_agent(++r, lo, A); }
    }
    {
        const unsigned wl = w0 + F110_ORDER_ITEMS_PER_THREAD;
        c[F110_ORDER_ITEMS_PER_THREAD + 1] = (wl < items && jj > 0) ? s.march_cost[(aa << 8) | jj] : F110_Q_UNKNOWN;
    }
    unsigned mine = 0u;
#pragma unroll
    for (int k = 0; k < F110_ORDER_ITEMS_PER_THREAD; k++) {
        if (cls[k] == 0) {
            const unsigned sj = packed[k] & 255u;
            unsigned m = c[k + 1];
            if (m != F110_Q_UNKNOWN) {
                if (sj > 0 && c[k] != F110_Q_UNKNOWN) m = max(m, c[k]);
                if (sj + 1 < ipa && c[k + 2] != F110_Q_UNKNOWN) m = max(m, c[k + 2]);
            }
            cls[k] = (c[k + 1] == F110_Q_UNKNOWN || c[k + 1] >= F110_Q_VERY_HEAVY) ? 0 : (m >= F110_Q_HEAVY) ? 1 : 2;
            mine += 1u << (10 * cls[k]);
        }
    }
    unsigned incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)lane >= o) incl += v;
    }
    const unsigned excl = incl - mine;
    const unsigned wtot = __shfl_sync(0xffffffffu, incl, 31);
    __syncthreads();
    unsigned wbase = 0u;
    if (lane < 3u) {
        const unsigned n = (wtot >> (10 * lane)) & 1023u;
        wbase = n ? atomicAdd(&s_cnt[lane], n) : 0u;
    }
    const unsigned b0 = __shfl_sync(0xffffffffu, wbase, 0), b1 = __shfl_sync(0xffffffffu, wbase, 1),
                   b2 = __shfl_sync(0xffffffffu, wbase, 2);
    __syncthreads();
    if (threadIdx.x < 3) s_base[threadIdx.x] = s_cnt[threadIdx.x] ? atomicAdd(s.march_count + threadIdx.x, s_cnt[threadIdx.x]) : 0u;
    __syncthreads();
    unsigned pos[3] = { s_base[0] + b0 + (excl & 1023u), s_base[1] + b1 + ((excl >> 10) & 1023u),
                        s_base[2] + b2 + ((excl >> 20) & 1023u) };
#pragma unroll
    for (int k = 0; k < F110_ORDER_ITEMS_PER_THREAD; k++) {
        if (cls[k] >= 0) {
            const unsigned at = (cls[k] == 0) ? pos[0]++ : (cls[k] == 1) ? pos[1]++ : pos[2]++;
            if (at < items) s.march_order[(size_t)cls[k] * items + at] = packed[k];
        }
    }
}

// ------------------------------------------------------------------------------------ k_raymarch
// One thread per beam; a warp owns 32 consecutive beams of (mostly) one agent, so its lanes walk
// neighbouring cells of the DT grid.  The grid is read through the read-only path: per scan the
// ~7-8 k lookups touch only ~1.3 k distinct 32-byte sectors (measured, DESIGN.md), i.e. the working
// set of the agents resident on an SM lives in L1 and the whole 20 MB table in L2.
struct MarchArgs {
    const double *__restrict__ scan_pose;   // [M][4] (x, y, yaw, theta_index0)    (STANDALONE: [M][3])
    const double *__restrict__ vel;         // [M] longitudinal velocity for iTTC, or NULL
    float *__restrict__ out_f32;            // [M][B] or NULL
    double *__restrict__ out_f64;           // [M][B] or NULL
    int32_t *__restrict__ wall_flag;        // [M] or NULL
    unsigned long long *lookup_counter;     // [1] or NULL
    const unsigned long long *tick_counter; // [1] or NULL (noise stream id)
    double ttc_thresh, noise_std;
    unsigned long long noise_seed;
    long long total;                        // M * B
};

template <bool FAST, bool STANDALONE>
__global__ void __launch_bounds__(256) k_raymarch(MapView m, BeamView bv, MarchArgs g) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = gid < g.total;
    int nlook = 0;
    if (valid) {
        const int B = bv.num_beams;
        const int a = (int)(gid / B);
        const int i = (int)(gid - (long long)a * B);
        double px, py, ti0;
        if (STANDALONE) {
            px = g.scan_pose[3 * (size_t)a];
            py = g.scan_pose[3 * (size_t)a + 1];
            ti0 = theta_index0(g.scan_pose[3 * (size_t)a + 2], bv.fov, m.theta_dis_f);
        } else {
            const double2 *sp = reinterpret_cast<const double2 *>(g.scan_pose) + 2 * (size_t)a;
            const double2 xy = __ldg(sp), yt = __ldg(sp + 1);
            px = xy.x; py = xy.y; ti0 = yt.y;
        }
        const int ti = beam_theta_index(ti0, i, bv.theta_index_increment, m.theta_dis_f);
        const double s = __ldg(m.sines + ti), c = __ldg(m.cosines + ti);
        double range = trace_ray<FAST>(m, px, py, s, c, nlook);
        if (g.noise_std > 0.0) {
            unsigned long long tick = g.tick_counter ? *g.tick_counter : 0ull;
            range = range + g.noise_std * normal_sample(g.noise_seed, tick, (uint64_t)gid);
        }
        if (g.wall_flag) {
            const double v = __ldg(g.vel + a);
            if (ttc_hit(range, v, __ldg(bv.cosines + i), __ldg(bv.side_distances + i), g.ttc_thresh))
                atomicOr(g.wall_flag + a, 1);
        }
        if (g.out_f32) g.out_f32[gid] = (float)range;
        if (g.out_f64) g.out_f64[gid] = range;
    }
    if (g.lookup_counter) {
        unsigned n = (unsigned)nlook;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
        if ((threadIdx.x & 31) == 0 && n) atomicAdd(g.lookup_counter, (unsigned long long)n);
    }
}

// ------------------------------------------------------------------------------------ finalize
// an angle difference reduced to [-pi, pi] (up to rounding), for any finite input
__device__ __forceinline__ double wrap_2pi_diff(double d) { return d - (2 * M_PI) * rint(d * (1.0 / (2 * M_PI))); }

// One warp finalises one agent (base_classes.py:536-550 check_collision, :579-589 update_scan loop).
__device__ __forceinline__ void finalize_agent(const f110_sim &s, const BeamView &bv, int a, int lane,
                                               double max_scan_range) {
    const int NA = s.num_envs * s.num_agents;
    const int A = s.num_agents;
    const int env = a / A, slot = a - env * A;
    const int hit = s.wall_flag[a];
    const double *pa = s.agent_poses + 5 * (size_t)a;
    const double px = pa[0], py = pa[1];      // == state[0], state[1]
    // check_ttc zeroes state[3:] — including the yaw — before the opponent ray-cast reads it (:246-249, :225)
    const double yaw = hit ? 0.0 : pa[2];
    const double cyaw = hit ? 1.0 : pa[3], syaw = hit ? 0.0 : pa[4];
    if (hit && lane < 4) s.state[(size_t)(3 + lane) * NA + a] = 0.0;

    // GJK against the other agents of this env, lower index first (collision_multiple :184-212)
    int col = 0, cidx = -1;
    if (A > 1) {
        double vme[8];
        get_vertices_cs(pa[0], pa[1], pa[3], pa[4], s.sim_length, s.sim_width, vme);
        // two car bodies can only overlap if their centres are closer than one body diagonal; beyond that
        // (with a 0.1 % margin) the shapes are strictly separated and GJK returns False, so it is not run
        const double reach2 = (s.sim_length * s.sim_length + s.sim_width * s.sim_width) * 1.001;
        for (int j = lane; j < A; j += 32) {
            if (j == slot) continue;
            const double *pb = s.agent_poses + 5 * (size_t)(env * A + j);
            const double ddx = pb[0] - pa[0], ddy = pb[1] - pa[1];
            if (ddx * ddx + ddy * ddy > reach2) continue;
            double vo[8];
            get_vertices_cs(pb[0], pb[1], pb[3], pb[4], s.sim_length, s.sim_width, vo);
            bool c = (slot < j) ? gjk_collision(vme, vo) : gjk_collision(vo, vme);
            if (c) { col = 1; cidx = max(cidx, j); }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            col |= __shfl_xor_sync(0xffffffffu, col, o);
            cidx = max(cidx, __shfl_xor_sync(0xffffffffu, cidx, o));
        }
    }
    if (lane == 0) {
        s.collisions[a] = (col || hit) ? 1.0 : 0.0;
        s.collision_idx[a] = cidx;
    }

    // ray_cast_agents (:206-227): opponents in ascending index, each bounded to its blocked-view window
    if (A > 1) {
        const double *p = s.params + (size_t)(s.params_per_env ? a : slot) * F110_NPARAM;
        const double length = p[P_LENGTH], width = p[P_WIDTH];
        float *scan = s.scans + (size_t)a * bv.num_beams;
        // an opponent whose nearest point is farther than any range the scan can hold (max_range plus noise
        // head-room) cannot shorten a beam: ray_cast would leave the scan unchanged, so it is skipped
        const double half_diag = 0.5 * sqrt(length * length + width * width);
        for (int j = 0; j < A; j++) {
            if (j == slot) continue;
            const double *pb = s.agent_poses + 5 * (size_t)(env * A + j);
            {
                const double ddx = pb[0] - px, ddy = pb[1] - py;
                const double far = max_scan_range + half_diag;
                if (ddx * ddx + ddy * ddy > far * far) continue;
            }
            double v[8];
            get_vertices_cs(pb[0], pb[1], pb[3], pb[4], length, width, v);
            int lo, hi;
            double phi;
            blocked_view_indices_warp(px, py, cyaw, syaw, v, bv.scan_angles, bv.num_beams, bv.fov, bv.angle_increment,
                                      lane, pb[0], pb[1], lo, hi, phi);
            // When the opponent straddles the rear cut of the field of view the window is ALL beams
            // (laser_models.py:310-315 takes min/max of the four nearest-beam indices).  A ray can only meet an
            // edge if it points into the cone that contains the opponent's bounding circle, so beams outside
            // that cone (+0.05 rad of slack) would get four `inf` ranges and leave the scan unchanged: skip them.
            // The cone (an asin and a sqrt) is only worth computing for a WIDE window; a narrow window (opponent in front)
            // consists of beams that point at the opponent anyway, so it runs unfiltered (cone = 4 > pi).
            double cone = 4.0;      // > pi: no filtering (also when the ego is inside / next to the bounding circle)
            const bool wide = hi - lo >= 96;
            if (wide) {
                const double ddx = pb[0] - px, ddy = pb[1] - py;
                const double dist = sqrt(ddx * ddx + ddy * ddy);
                if (dist > 1.25 * half_diag) cone = asin(half_diag / dist) + 0.05;
            }
            // one beam of the window: cone test, then the four edges (only `min(scan, range)` is needed)
            auto cast_beams = [&](int i0, int i1) {
                for (int i = i0 + lane; i <= i1; i += 32) {
                    const float cur = scan[i];          // issued early: often an L2/DRAM miss (the march just wrote it)
                    double bt = yaw + bv.scan_angles[i];
                    double dl = bt - phi;
                    dl = dl - (2 * M_PI) * rint(dl * (1.0 / (2 * M_PI)));
                    // (the mirrored cone is kept too: get_range's collinear branch, laser_models.py:275-278, has no
                    // direction test, so a beam pointing exactly away along an edge line still reports that edge)
                    const double adl = fabs(dl);
                    if (adl > cone && (M_PI - adl) > cone) continue;
                    double v3x, v3y;
                    sincos(bt + M_PI / 2., &v3y, &v3x);
                    const double curd = (double)cur;
                    double r = INFINITY;
#pragma unroll
                    for (int e = 0; e < 4; e++) {
                        int e2 = (e + 1) & 3;
                        double d = get_range_below(px, py, v3x, v3y, v[2 * e], v[2 * e + 1], v[2 * e2], v[2 * e2 + 1], curd);
                        if (d < r) r = d;
                    }
                    float rf = (float)r;
                    if (rf < cur) scan[i] = rf;
                }
            };
            if (cone < 3.5 && wide) {
                // wide window (the opponent straddles the rear cut: ALL beams): only beams whose angle lies within `cone` of
                // the direction to the opponent, or of the opposite direction, can pass the test above.  Those are the
                // beams around the centres (phi - yaw) + m pi; visit just these index intervals, with two beams of slack
                // on both sides -- the exact per-beam test still decides.
                // (phi - yaw reduced modulo 2 pi: the state's yaw is wrapped once per step only, so an integration that blows
                // up -- e.g. the single-track model at a 0.05 s time step -- leaves it anywhere, and the clamped m range below
                // would then miss the centres)
                const double base = wrap_2pi_diff(phi - yaw), half = bv.fov / 2., inv_inc = 1.0 / bv.angle_increment;
                // centres base + m pi that can reach the beam range [-half, half] (+- cone and slack): usually 1-3 of them
                const int m0 = max(-3, (int)floor((-half - cone - 0.02 - base) * (1.0 / M_PI))),
                          m1 = min(5, (int)ceil((half + cone + 0.02 - base) * (1.0 / M_PI)));
                for (int m = m0; m <= m1; m++) {
                    const double c = base + (double)m * M_PI;
                    const double f0 = (c - cone + half) * inv_inc - 2.0, f1 = (c + cone + half) * inv_inc + 2.0;
                    if (f1 < (double)lo || f0 > (double)hi) continue;
                    const int i0 = max(lo, (int)floor(fmax(f0, (double)lo))), i1 = min(hi, (int)ceil(fmin(f1, (double)hi)));
                    cast_beams(i0, i1);
                }
            } else {
                cast_beams(lo, hi);
            }
            __syncwarp();
        }
    }
}

// the march work-queue counters are consumed once k_march has run; the next tick's k_dynamics refills them
__device__ __forceinline__ void end_of_tick_housekeeping(const f110_sim &s) {
    if (s.march_count) { s.march_count[0] = 0u; s.march_count[1] = 0u; s.march_count[2] = 0u; s.march_count[3] = 0u; }
}

// f110_step: warp per agent
__global__ void __launch_bounds__(128, 8) k_finalize(f110_sim s, BeamView bv, double max_scan_range) {
    pdl_wait();
    const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (a >= s.num_envs * s.num_agents) return;
    finalize_agent(s, bv, a, lane, max_scan_range);
    if (a == 0 && lane == 0) end_of_tick_housekeeping(s);
}

// ------------------------------------------------------------------------------------ reset kernels
// a reset agent has no lookup history: its march items are scheduled with the very-heavy class next tick
__device__ __forceinline__ void mark_march_cost_unknown(const f110_sim &s, size_t a) {
    if (s.march_cost)
        for (int j = 0; j < s.march_ipa; j++) s.march_cost[(a << 8) + (size_t)j] = F110_Q_UNKNOWN;
}

__global__ void k_reset(f110_sim s, const double *__restrict__ poses, const uint8_t *__restrict__ mask) {
    const int NA = s.num_envs * s.num_agents;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= NA) return;
    if (mask && !mask[a / s.num_agents]) return;
    // RaceCar.reset base_classes.py:183-204
#pragma unroll
    for (int k = 0; k < 7; k++) s.state[(size_t)k * NA + a] = 0.0;
    s.state[a] = poses[3 * (size_t)a];
    s.state[(size_t)NA + a] = poses[3 * (size_t)a + 1];
    s.state[(size_t)4 * NA + a] = poses[3 * (size_t)a + 2];
    s.steer_cnt[a] = 0;
    s.steer_buf[a] = 0.0;
    s.steer_buf[(size_t)NA + a] = 0.0;
    s.wall_flag[a] = 0;
    mark_march_cost_unknown(s, a);
}

// clear_done: f110_env_reset (a fresh episode requested by the caller) clears the done flag; the auto-reset does NOT --
// the tick that ended an episode must still report done = 1 for it (the next tick recomputes the flag)
__device__ __forceinline__ void env_counters_reset(const f110_sim &s, int env, const double *agent_pose3 /* [A][3] */,
                                                   bool clear_done = true) {
    const int A = s.num_agents;
    s.current_time[env] = 0.0;
    for (int i = 0; i < A; i++) {
        const size_t a = (size_t)env * A + i;
        s.near_starts[a] = 1;
        s.toggle_list[a] = 0.0;
        s.start_xs[a] = agent_pose3[3 * i];
        s.start_ys[a] = agent_pose3[3 * i + 1];
        s.start_thetas[a] = agent_pose3[3 * i + 2];
    }
    // f110_env.py:331 start_rot from the ego's start heading
    const double th = -agent_pose3[3 * s.ego_idx + 2];
    double *R = s.start_rot + 4 * (size_t)env;
    R[0] = cos(th); R[1] = -sin(th); R[2] = sin(th); R[3] = cos(th);
    if (s.done && clear_done) s.done[env] = 0;
}

__global__ void k_env_reset(f110_sim s, const double *__restrict__ poses, const uint8_t *__restrict__ mask) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= s.num_envs) return;
    if (mask && !mask[env]) return;
    env_counters_reset(s, env, poses + 3 * (size_t)env * s.num_agents);
}

// f110_env.py:294-302 + _check_done :204-246, one thread per env
__device__ __forceinline__ void env_post_step_one(const f110_sim &s, int env) {
    const int A = s.num_agents, NA = s.num_envs * s.num_agents;
    const double left_t = 2, right_t = 2;
    const double now = s.current_time[env] + s.timestep;
    s.current_time[env] = now;
    const double *R = s.start_rot + 4 * (size_t)env;
    bool all_done = true;
    for (int i = 0; i < A; i++) {
        const size_t a = (size_t)env * A + i;
        double px = s.state[a] - s.start_xs[a];
        double py = s.state[(size_t)NA + a] - s.start_ys[a];
        double dx = R[0] * px + R[1] * py;
        double ty = R[2] * px + R[3] * py;
        if (ty > left_t) ty -= left_t;
        else if (ty < -right_t) ty = -right_t - ty;
        else ty = 0;
        double dist2 = dx * dx + ty * ty;
        bool close = dist2 <= 0.1;
        int near = s.near_starts[a];
        double tog = s.toggle_list[a];
        if (close && !near) { near = 1; tog += 1; }
        else if (!close && near) { near = 0; tog += 1; }
        s.near_starts[a] = near;
        s.toggle_list[a] = tog;
        s.lap_counts[a] = floor(tog / 2);
        if (tog < 4) s.lap_times[a] = now;
        bool cp = tog >= 4;
        if (s.checkpoint_done) s.checkpoint_done[a] = cp ? 1 : 0;
        all_done = all_done && cp;
    }
    s.done[env] = ((s.collisions[(size_t)env * A + s.ego_idx] != 0.0) || all_done) ? 1 : 0;
}

__global__ void k_env_post_step(f110_sim s) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env < s.num_envs) env_post_step_one(s, env);
}

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

struct AutoResetArgs {
    const double *start_poses;   // [num_start][3] or NULL = off
    int num_start, pose_gap;
    uint64_t seed, tick_host;
    int num_tables;              // 0: one shared start table; L: per-layer tables (f110_sim.start_offsets), env_layer set
    int32_t start_off[F110_MAX_START_TABLES + 1];   // host copy of f110_sim.start_offsets, by value (CUDA graphs keep it)
};

// one thread per env: reset the env if its ego collided (benchmark / RL convenience, SURVEY.md 8d)
__device__ __forceinline__ void autoreset_one(const f110_sim &s, int env, const AutoResetArgs &ar) {
    const int A = s.num_agents, NA = s.num_envs * s.num_agents;
    if (s.collisions[(size_t)env * A + s.ego_idx] == 0.0) return;
    const double *__restrict__ start_poses = ar.start_poses;
    int num_start = ar.num_start;
    const int pose_gap = ar.pose_gap;
    if (ar.num_tables) {         // the start table of the env's own map: rows [start_off[l], start_off[l + 1])
        const int l = s.env_layer[env];
        start_poses += 3 * (size_t)ar.start_off[l];
        num_start = ar.start_off[l + 1] - ar.start_off[l];
    }
    const uint64_t seed = ar.seed;
    const uint64_t tick = s.tick_counter ? (uint64_t)*s.tick_counter : ar.tick_host;
    uint64_t h = mix64(seed + 0x9E3779B97F4A7C15ull * (tick + 1) + 0xD1B54A32D192ED03ull * (uint64_t)(env + 1));
    int k = (int)((double)(h >> 11) * (1.0 / 9007199254740992.0) * num_start);
    if (k >= num_start) k = num_start - 1;
    double pose3[3 * 32];
    for (int i = 0; i < A; i++) {
        int kk = ((k - pose_gap * i) % num_start + num_start) % num_start;
        const size_t a = (size_t)env * A + i;
        const double x = start_poses[3 * kk], y = start_poses[3 * kk + 1], th = start_poses[3 * kk + 2];
        if (i < 32) { pose3[3 * i] = x; pose3[3 * i + 1] = y; pose3[3 * i + 2] = th; }
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
    if (s.current_time && A <= 32) env_counters_reset(s, env, pose3, false);
}

__global__ void k_autoreset(f110_sim s, AutoResetArgs ar) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env < s.num_envs) autoreset_one(s, env, ar);
}

// f110_tick: warp per agent; the warp that finishes an env last (per-env arrival counter) also runs the F110Env
// lap logic and the auto-reset for that env: k_finalize + k_env_post_step + k_autoreset in one launch
// MAXT / MINB: blocks of up to 4 agent-warps (A <= 4) are compiled without the 64-register cap of a 1024-thread block
template <int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) k_tail(f110_sim s, BeamView bv, int env_level, AutoResetArgs ar,
                                                      double max_scan_range, int envs_per_block) {
    // a block owns whole envs (blockDim = 32 * A * envs_per_block, A <= 32): the env-level step only needs what the
    // warps of its own block wrote, so a block barrier orders it -- no device-scope fence, no arrival atomics.  (The
    // first version had every warp execute __threadfence() + atomicAdd on a per-env counter; the fence's L1
    // invalidation (CCTL.IVALL) kept evicting the beam tables and poses of the other warps on the SM: 19 % of the
    // kernel's stall samples sat on the fences and 8 % on the scan-angle loads behind them.)
    const int A = s.num_agents;
    const int lane = threadIdx.x & 31;
    pdl_wait();                              // the march kernel (scans, wall flags) must be complete
    const int env0 = blockIdx.x * envs_per_block;
    const int a = env0 * A + (int)(threadIdx.x >> 5);
    if (a < s.num_envs * A) finalize_agent(s, bv, a, lane, max_scan_range);
    __syncthreads();
    if ((int)threadIdx.x < envs_per_block) {
        const int env = env0 + (int)threadIdx.x;
        if (env < s.num_envs) {
            if (env_level) env_post_step_one(s, env);
            if (ar.start_poses) autoreset_one(s, env, ar);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) end_of_tick_housekeeping(s);
}

// ------------------------------------------------------------------------------------ k_tail2 (2 <= A <= 4)
// Same results as k_tail, reorganised (round 2).  ncu on k_tail at 16384 x 2: 1317 warp-instructions per agent, most of them the
// per-agent SCALAR prologue (opponent vertices, six atan2, asin, sqrt, nearest-beam searches) that all 32 lanes of the agent's
// warp execute redundantly.  Here a block owns EPB whole envs and works in three phases:
//   1. one THREAD per (ego, opponent) pair does the scalar prologue -- 32 pairs per warp instead of one -- and leaves a task
//      record in shared memory: the window and the beam intervals the cast visits; one thread per agent also does the wall-hit
//      zeroing, GJK and the collisions observation;
//   2. the beams of all tasks of one opponent rank form one flat list, and every thread of the block casts its share of it
//      (below); one pass per rank;
//   3. one thread per env: lap logic + auto-reset (as in k_tail).
// A task visits 33-56 beams on the benchmark's poses (tools/tail_cast_study.py), so a warp per ego -- the first version of
// phase 2 -- ran 2-3 loop iterations per opponent, each a serial chain of a scan load (mostly DRAM: the march's scans
// outgrow L2), an fp64 sincos and four edge tests, for ~10 egos one after the other per warp at cfg3.  The flat list spreads
// the same beams over every thread at once.
// The TailTask records of k_lidar_cast / k_episode_cast are separate: changing them would change those kernels.
#define F110_TAIL2_IVALS 4               // beam intervals per task (fov <= 2 pi, cone <= pi/2 + 0.05: at most 4)
struct Tail2Task {                       // 120 bytes, as the TailTask it replaced: the launch record's smem is unchanged
    double phi, cone;
    double v[8];
    int iv[2 * F110_TAIL2_IVALS];        // disjoint beam intervals [iv[2q], iv[2q + 1]], ascending
    int pad[2];
};
struct TailTask {                        // the records of k_lidar_cast / k_episode_cast (warp per ego)
    double px, py, yaw, phi, cone;
    double v[8];
    int lo, hi, active, pad;
};
#define F110_TAIL2_THREADS 256
#define F110_TAIL2_MAX_AGENTS 128        // agents per block: f110_debug_set_tail2 caps forced shapes here

// dynamic shared memory of k_tail2 for epb envs of A agents: the task records
static inline size_t tail2_smem_bytes(int epb, int A) { return (size_t)epb * A * (A - 1) * sizeof(Tail2Task); }

__global__ void __launch_bounds__(F110_TAIL2_THREADS, 3) k_tail2(f110_sim s, BeamView bv, int env_level, AutoResetArgs ar,
                                                                  double max_scan_range, int envs_per_block) {
    extern __shared__ __align__(16) unsigned char tail2_smem[];
    Tail2Task *tasks = reinterpret_cast<Tail2Task *>(tail2_smem);
    __shared__ double ego_pose[3][F110_TAIL2_MAX_AGENTS];      // px, py and the yaw the cast uses, per ego
    __shared__ int offs[3 * (F110_TAIL2_MAX_AGENTS + 1)];      // per opponent rank: beams per ego, then their exclusive scan
    const int A = s.num_agents, NA = s.num_envs * A;
    const int opp = A - 1;                                    // tasks per agent
    const int env0 = blockIdx.x * envs_per_block;
    const int envs_here = min(envs_per_block, s.num_envs - env0);
    const int agents_here = envs_here * A;
    const int ntasks = agents_here * opp;
    pdl_wait();                                                // the march kernel (scans, wall flags) must be complete

    // ---- phase 1: thread per (ego, opponent) pair
    for (int t = threadIdx.x; t < ntasks; t += blockDim.x) {
        const int la = t / opp, oj = t - la * opp;
        const int envl = la / A, slot = la - envl * A;
        const int env = env0 + envl, a = env * A + slot;
        const int j = oj < slot ? oj : oj + 1;                 // opponents in ascending index, skipping the ego itself
        const int hit = s.wall_flag[a];
        const double *pa = s.agent_poses + 5 * (size_t)a;
        const double px = pa[0], py = pa[1];
        // check_ttc zeroes state[3:] -- including the yaw -- before the opponent ray-cast reads it (:246-249, :225)
        const double yaw = hit ? 0.0 : pa[2];
        const double cyaw = hit ? 1.0 : pa[3], syaw = hit ? 0.0 : pa[4];
        const double *pb = s.agent_poses + 5 * (size_t)(env * A + j);
        if (oj == 0) {
            ego_pose[0][la] = px; ego_pose[1][la] = py; ego_pose[2][la] = yaw;
            // per-agent duties: wall-hit zeroing, GJK against the other agents (collision_multiple :184-212), collisions obs
            if (hit) {
#pragma unroll
                for (int q = 0; q < 4; q++) s.state[(size_t)(3 + q) * NA + a] = 0.0;
            }
            int col = 0, cidx = -1;
            const double reach2 = (s.sim_length * s.sim_length + s.sim_width * s.sim_width) * 1.001;
            for (int jj = 0; jj < A; jj++) {
                if (jj == slot) continue;
                const double *pc = s.agent_poses + 5 * (size_t)(env * A + jj);
                const double ddx = pc[0] - pa[0], ddy = pc[1] - pa[1];
                if (ddx * ddx + ddy * ddy > reach2) continue;
                double vme[8], vo[8];
                get_vertices_cs(pa[0], pa[1], pa[3], pa[4], s.sim_length, s.sim_width, vme);
                get_vertices_cs(pc[0], pc[1], pc[3], pc[4], s.sim_length, s.sim_width, vo);
                const bool c = (slot < jj) ? gjk_collision(vme, vo) : gjk_collision(vo, vme);
                if (c) { col = 1; cidx = max(cidx, jj); }
            }
            s.collisions[a] = (col || hit) ? 1.0 : 0.0;
            s.collision_idx[a] = cidx;
        }
        // ray_cast_agents (:206-227): the scalar part of one opponent
        Tail2Task &k = tasks[t];
        const double *p = s.params + (size_t)(s.params_per_env ? a : slot) * F110_NPARAM;
        const double length = p[P_LENGTH], width = p[P_WIDTH];
        const double half_diag = 0.5 * sqrt(length * length + width * width);
        const double ddx = pb[0] - px, ddy = pb[1] - py;
        const double far = max_scan_range + half_diag;
        int n = 0;
        if (ddx * ddx + ddy * ddy <= far * far) {              // else it cannot shorten any beam (see finalize_agent)
            double v[8];
            get_vertices_cs(pb[0], pb[1], pb[3], pb[4], length, width, v);
            int lo, hi;
            double phi;
            blocked_view_indices_cs(px, py, cyaw, syaw, v, bv.scan_angles, bv.num_beams, bv.fov, bv.angle_increment, pb[0], pb[1],
                                    lo, hi, phi);
            double cone = 4.0;
            if (hi - lo >= 96) {
                const double dist = sqrt(ddx * ddx + ddy * ddy);
                if (dist > 1.25 * half_diag) cone = asin(half_diag / dist) + 0.05;
            }
            k.phi = phi; k.cone = cone;
#pragma unroll
            for (int q = 0; q < 8; q++) k.v[q] = v[q];
            // the beams to visit: [lo, hi], or in a wide window the intervals around the centres (phi - yaw) + m pi (see
            // finalize_agent).  Clipping each interval to start after the previous one is exact: centres are pi apart and
            // cone < pi/2 here, so they do not overlap anyway, and a second visit of a beam by the same opponent stores nothing.
            int nq = 0;
            bool whole = true;
            if (cone < 3.5 && hi - lo >= 96) {
                whole = false;
                const double base = wrap_2pi_diff(phi - yaw), half = bv.fov / 2., inv_inc = 1.0 / bv.angle_increment;
                const int m0 = max(-3, (int)floor((-half - cone - 0.02 - base) * (1.0 / M_PI))),
                          m1 = min(5, (int)ceil((half + cone + 0.02 - base) * (1.0 / M_PI)));
                int next = lo;
                for (int m = m0; m <= m1; m++) {
                    const double c = base + (double)m * M_PI;
                    const double f0 = (c - cone + half) * inv_inc - 2.0, f1 = (c + cone + half) * inv_inc + 2.0;
                    if (f1 < (double)lo || f0 > (double)hi) continue;
                    const int i0 = max(next, (int)floor(fmax(f0, (double)lo))), i1 = min(hi, (int)ceil(fmin(f1, (double)hi)));
                    if (i0 > i1) continue;
                    // more intervals than the record holds (fov > 2 pi, or a cone the window rule cannot make): [lo, hi]
                    // instead, which is exact -- the per-beam cone test decides
                    if (nq == F110_TAIL2_IVALS) { whole = true; break; }
                    k.iv[2 * nq] = i0; k.iv[2 * nq + 1] = i1;
                    n += i1 - i0 + 1;
                    nq++;
                    next = i1 + 1;
                }
            }
            if (whole) { k.iv[0] = lo; k.iv[1] = hi; n = hi - lo + 1; nq = 1; }
        }
        offs[oj * (agents_here + 1) + la] = n;                  // beams the task visits (0: none)
    }
    __syncthreads();

    // ---- phase 2a: exclusive scan of the tasks' beam counts, one array per opponent rank (a warp per rank)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int oj = warp; oj < opp; oj += nwarps) {
        int *o = offs + oj * (agents_here + 1);
        int run = 0;
        for (int l0 = 0; l0 < agents_here; l0 += 32) {
            const int la = l0 + lane;
            const int n = la < agents_here ? o[la] : 0;
            int incl = n;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += u;
            }
            if (la < agents_here) o[la] = run + incl - n;
            run += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) o[agents_here] = run;
    }
    __syncthreads();

    // ---- phase 2b: flat beam list of each opponent rank over the whole block.  Flat index f of rank oj is beam f - o[la] of
    // ego la's intervals, o[la] <= f < o[la + 1]; thread tid takes f = tid, tid + blockDim, ...  Within a pass an (ego, beam)
    // pair occurs once, so no two threads touch one scan entry; the passes run in rank order, so a beam that two opponents
    // shorten sees them in k_tail's order.  Per beam the statements are finalize_agent's, except that the cone test comes
    // before the scan load (a rejected beam loads nothing).  Measured on the H100 at cfg3 (16384 x 2), k_tail2: 34 us with
    // one beam at a time per thread, 39.5 us when a thread first issued the loads of a batch of 4 beams, and no gain from an
    // L2 prefetch of the tasks' scan lines in phase 1 (39.4 us with, 39.3 without, at the batch of 4).
    const int B = bv.num_beams;
    float *scans0 = s.scans + (size_t)env0 * A * B;
    for (int oj = 0; oj < opp; oj++) {
        if (oj) __syncthreads();
        const int *o = offs + oj * (agents_here + 1);
        const int total = o[agents_here];
        int la = 0;
        if ((int)threadIdx.x < total) {                       // the task of the first index: largest la with o[la] <= tid
            int hi = agents_here;
            while (hi - la > 1) {
                const int mid = (la + hi) >> 1;
                if (o[mid] <= (int)threadIdx.x) la = mid;
                else hi = mid;
            }
        }
        for (int f = threadIdx.x; f < total; f += blockDim.x) {
            while (o[la + 1] <= f) la++;
            const Tail2Task &k = tasks[la * opp + oj];
            int r = f - o[la], q = 0;
            while (r > k.iv[2 * q + 1] - k.iv[2 * q]) { r -= k.iv[2 * q + 1] - k.iv[2 * q] + 1; q++; }
            const int i = k.iv[2 * q] + r;
            double bt = ego_pose[2][la] + bv.scan_angles[i];
            double dl = bt - k.phi;
            dl = dl - (2 * M_PI) * rint(dl * (1.0 / (2 * M_PI)));
            const double adl = fabs(dl);
            if (adl > k.cone && (M_PI - adl) > k.cone) continue;
            float *scan = scans0 + (size_t)la * B;
            const float cur = scan[i];
            const double px = ego_pose[0][la], py = ego_pose[1][la];
            double v[8];
#pragma unroll
            for (int e = 0; e < 8; e++) v[e] = k.v[e];
            double v3x, v3y;
            sincos(bt + M_PI / 2., &v3y, &v3x);
            const double curd = (double)cur;
            double rr = INFINITY;
#pragma unroll
            for (int e = 0; e < 4; e++) {
                int e2 = (e + 1) & 3;
                double d = get_range_below(px, py, v3x, v3y, v[2 * e], v[2 * e + 1], v[2 * e2], v[2 * e2 + 1], curd);
                if (d < rr) rr = d;
            }
            float rf = (float)rr;
            if (rf < cur) scan[i] = rf;
        }
    }
    __syncthreads();

    // ---- phase 3: env level (a loop: a forced shape of f110_debug_set_tail2 may have more envs than threads)
    for (int e = threadIdx.x; e < envs_here; e += blockDim.x) {
        const int env = env0 + e;
        if (env_level) env_post_step_one(s, env);
        if (ar.start_poses) autoreset_one(s, env, ar);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) end_of_tick_housekeeping(s);
}

// ------------------------------------------------------------------------------------ k_tail_noscan (f110_tick_repeat)
// The tail of a tick whose scans are withheld (march_ttc.cuh): k_tail2 without its task records and its phase 2, the opponent
// ray-cast, which is the only part of a tail that touches scans.  A block owns whole envs (A <= 32): one thread per agent does
// agent_duties, then one thread per env the lap logic, the done bookkeeping of the repeat call and the auto-reset.
// The per-agent duties of a tail that one thread can do: wall-hit zeroing, GJK against the other agents of the env
// (collision_multiple :184-212) and the collisions observation.  pa = the agent's pose snapshot.  The statements of k_tail2's
// phase 1, kept apart from it: calling this from k_tail2 changes that kernel's code.
__device__ __forceinline__ void agent_duties(const f110_sim &s, int env, int slot, int a, int hit, const double *pa) {
    const int A = s.num_agents, NA = s.num_envs * A;
    if (hit) {
#pragma unroll
        for (int q = 0; q < 4; q++) s.state[(size_t)(3 + q) * NA + a] = 0.0;
    }
    int col = 0, cidx = -1;
    const double reach2 = (s.sim_length * s.sim_length + s.sim_width * s.sim_width) * 1.001;
    for (int jj = 0; jj < A; jj++) {
        if (jj == slot) continue;
        const double *pc = s.agent_poses + 5 * (size_t)(env * A + jj);
        const double ddx = pc[0] - pa[0], ddy = pc[1] - pa[1];
        if (ddx * ddx + ddy * ddy > reach2) continue;
        double vme[8], vo[8];
        get_vertices_cs(pa[0], pa[1], pa[3], pa[4], s.sim_length, s.sim_width, vme);
        get_vertices_cs(pc[0], pc[1], pc[3], pc[4], s.sim_length, s.sim_width, vo);
        const bool c = (slot < jj) ? gjk_collision(vme, vo) : gjk_collision(vo, vme);
        if (c) { col = 1; cidx = max(cidx, jj); }
    }
    s.collisions[a] = (col || hit) ? 1.0 : 0.0;
    s.collision_idx[a] = cidx;
}

struct RepeatDone {
    uint8_t *done_any;       // [N] or NULL
    int32_t *done_tick;      // [N] or NULL
    int tick;                // index of this tick inside the call
};
// done_any / done_tick of f110_repeat from this tick's done flag: tick 0 overwrites what the previous call left
__device__ __forceinline__ void repeat_done_one(const f110_sim &s, int env, const RepeatDone &rd) {
    const int d = s.done[env] ? 1 : 0;
    if (rd.done_any) rd.done_any[env] = (uint8_t)((rd.tick == 0 ? 0 : rd.done_any[env]) | d);
    if (rd.done_tick) {
        const int first = rd.tick == 0 ? -1 : rd.done_tick[env];
        rd.done_tick[env] = (first < 0 && d) ? rd.tick : first;
    }
}
// after the ordinary tail of a tick of the call (its last one, or any tick of a call that takes the plain path)
__global__ void k_repeat_done(f110_sim s, RepeatDone rd) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env < s.num_envs) repeat_done_one(s, env, rd);
}

__global__ void __launch_bounds__(F110_TAIL_NOSCAN_THREADS) k_tail_noscan(f110_sim s, int env_level, AutoResetArgs ar,
                                                                          int envs_per_block, RepeatDone rd) {
    const int A = s.num_agents;
    const int env0 = blockIdx.x * envs_per_block;
    const int envs_here = min(envs_per_block, s.num_envs - env0);
    for (int la = threadIdx.x; la < envs_here * A; la += blockDim.x) {
        const int envl = la / A, slot = la - envl * A;
        const int a = env0 * A + la;
        agent_duties(s, env0 + envl, slot, a, s.wall_flag[a], s.agent_poses + 5 * (size_t)a);
    }
    __syncthreads();
    if ((int)threadIdx.x < envs_here) {
        const int env = env0 + (int)threadIdx.x;
        if (env_level) {
            env_post_step_one(s, env);
            repeat_done_one(s, env, rd);
        }
        if (ar.start_poses) autoreset_one(s, env, ar);
    }
}

// ------------------------------------------------------------------------------------ k_lidar_cast (f110_lidar)
// The opponent ray-cast of a tick with a lidar mask, for the egos whose slot has a lidar: a warp per such ego (LidarOrder's
// enumeration), any A <= 32.  Lane oj < A - 1 does k_tail2's scalar prologue for opponent oj into the warp's task records,
// then the warp walks its opponents in ascending order with k_tail2's beam loop -- the same statements, so the scans are
// bit-identical to the plain tick's (blocked_view_indices_cs equals the warp-cooperative version of k_tail / k_finalize).
// It must run before k_tail_noscan: that kernel's auto-reset clears wall_flag, which gives the yaw an iTTC hit zeroed.
// Thread 0 of block 0 consumes the march queue counters, as the tails' end_of_tick_housekeeping does.
#define F110_LIDAR_CAST_WARPS 4
__global__ void __launch_bounds__(32 * F110_LIDAR_CAST_WARPS) k_lidar_cast(f110_sim s, BeamView bv, LidarOrder lo,
                                                                            double max_scan_range) {
    __shared__ TailTask tasks_all[F110_LIDAR_CAST_WARPS][31];
    const int A = s.num_agents;
    const int opp = A - 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (blockIdx.x == 0 && threadIdx.x == 0) end_of_tick_housekeeping(s);
    const unsigned r = blockIdx.x * F110_LIDAR_CAST_WARPS + (unsigned)warp;
    if (opp < 1 || r >= (unsigned)s.num_envs * lo.slots) return;       // warp-uniform
    const int a = (int)lidar_agent(r, lo, (unsigned)A);
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

}  // namespace f110
#include "obstacles.cuh"     // k_obstacles, k_env_tail_obst: built on the tail's device functions above
#include "episodes.cuh"      // the restart of ended episodes: built on the same functions and on obstacles.cuh's
#include "episode_repeat.cuh"   // episodes under a held action: the end latch, reusing the restart kernels above
#include "param_draw.cuh"       // per-episode parameter draws, launched after the call that restarted the envs
#include "predict.cuh"          // predicted futures: k_dynamics' and k_march_ttc's per-agent statements in one rollout kernel
#include "mppi.cuh"             // the MPPI planner's sample and update steps around the scored rollout
namespace f110 {

// f110_track_progress_sum: the deltas of the ticks of one policy step, summed in tick order
__global__ void k_delta_sum(const double *__restrict__ delta, double *__restrict__ sum, int n, int restart) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a < n) sum[a] = restart ? delta[a] : sum[a] + delta[a];
}

// ------------------------------------------------------------------------------------ standalone kernels
__global__ void k_rhs(const double *__restrict__ x, const double *__restrict__ u, const double *__restrict__ p,
                      int M, double *__restrict__ f) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M) return;
    double xs[7], fs[7];
    for (int k = 0; k < 7; k++) xs[k] = x[7 * (size_t)i + k];
    vehicle_dynamics_st(xs, u[2 * (size_t)i], u[2 * (size_t)i + 1], p, fs);
    for (int k = 0; k < 7; k++) f[7 * (size_t)i + k] = fs[k];
}

__global__ void k_rhs_ks(const double *__restrict__ x, const double *__restrict__ u, const double *__restrict__ p,
                         int M, double *__restrict__ f) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M) return;
    double xs[5], fs[5];
    for (int k = 0; k < 5; k++) xs[k] = x[5 * (size_t)i + k];
    vehicle_dynamics_ks(xs, u[2 * (size_t)i], u[2 * (size_t)i + 1], p, fs);
    for (int k = 0; k < 5; k++) f[5 * (size_t)i + k] = fs[k];
}

__global__ void k_pid(const double *__restrict__ in, const double *__restrict__ p, int M, double *__restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M) return;
    double accl, sv;
    pid(in[4 * (size_t)i], in[4 * (size_t)i + 1], in[4 * (size_t)i + 2], in[4 * (size_t)i + 3], p[P_SVMAX],
        p[P_AMAX], p[P_VMAX], p[P_VMIN], accl, sv);
    out[2 * (size_t)i] = accl;
    out[2 * (size_t)i + 1] = sv;
}

__global__ void k_vertices(const double *__restrict__ poses, double length, double width, int M,
                           double *__restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M) return;
    double v[8];
    get_vertices(poses[3 * (size_t)i], poses[3 * (size_t)i + 1], poses[3 * (size_t)i + 2], length, width, v);
    for (int k = 0; k < 8; k++) out[8 * (size_t)i + k] = v[k];
}

__global__ void k_gjk(const double *__restrict__ va, const double *__restrict__ vb, int M, int32_t *__restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M) return;
    double a[8], b[8];
    for (int k = 0; k < 8; k++) { a[k] = va[8 * (size_t)i + k]; b[k] = vb[8 * (size_t)i + k]; }
    out[i] = gjk_collision(a, b) ? 1 : 0;
}

__global__ void k_gjk_multiple(const double *__restrict__ verts, int M, int n, double *__restrict__ collisions,
                               double *__restrict__ collision_idx) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= M) return;
    const double *V = verts + (size_t)e * n * 8;
    for (int i = 0; i < n; i++) { collisions[(size_t)e * n + i] = 0.; collision_idx[(size_t)e * n + i] = -1.; }
    for (int i = 0; i < n - 1; i++)
        for (int j = i + 1; j < n; j++) {
            double a[8], b[8];
            for (int k = 0; k < 8; k++) { a[k] = V[8 * i + k]; b[k] = V[8 * j + k]; }
            if (gjk_collision(a, b)) {
                collisions[(size_t)e * n + i] = 1.; collisions[(size_t)e * n + j] = 1.;
                collision_idx[(size_t)e * n + i] = j; collision_idx[(size_t)e * n + j] = i;
            }
        }
}

__global__ void k_check_ttc(BeamView bv, const double *__restrict__ scans, const double *__restrict__ vel,
                            double thresh, int M, int32_t *__restrict__ out) {
    const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (a >= M) return;
    int hit = 0;
    for (int i = lane; i < bv.num_beams; i += 32)
        hit |= ttc_hit(scans[(size_t)a * bv.num_beams + i], vel[a], bv.cosines[i], bv.side_distances[i], thresh) ? 1 : 0;
    hit = __any_sync(0xffffffffu, hit);
    if (lane == 0) out[a] = hit ? 1 : 0;
}

__global__ void k_ray_cast(BeamView bv, const double *__restrict__ poses, const double *__restrict__ opp, int M,
                           float *__restrict__ scans, int32_t *__restrict__ window) {
    const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (a >= M) return;
    const double px = poses[3 * (size_t)a], py = poses[3 * (size_t)a + 1], yaw = poses[3 * (size_t)a + 2];
    double v[8];
    for (int k = 0; k < 8; k++) v[k] = opp[8 * (size_t)a + k];
    int lo, hi;
    blocked_view_indices(px, py, yaw, v, bv.scan_angles, bv.num_beams, bv.fov, bv.angle_increment, lo, hi);
    if (window && lane == 0) { window[2 * a] = lo; window[2 * a + 1] = hi; }
    float *scan = scans + (size_t)a * bv.num_beams;
    for (int i = lo + lane; i <= hi; i += 32) {
        double bt = yaw + bv.scan_angles[i];
        double v3x = cos(bt + M_PI / 2.), v3y = sin(bt + M_PI / 2.);
        double r = INFINITY;
        for (int e = 0; e < 4; e++) {
            int e2 = (e + 1) & 3;
            double d = get_range(px, py, v3x, v3y, v[2 * e], v[2 * e + 1], v[2 * e2], v[2 * e2 + 1]);
            if (d < r) r = d;
        }
        float rf = (float)r;
        if (rf < scan[i]) scan[i] = rf;
    }
}

// four ranges -> three 32-bit words (12 bytes): 24-bit fixed point with 2^-19 m steps
__global__ void k_pack_u24(const float *__restrict__ scans, long long count, uint8_t *__restrict__ out) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i0 = g * 4;
    if (i0 >= count) return;
    unsigned q[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const float r = (i0 + k < count) ? scans[i0 + k] : 0.0f;
        const float v = fminf(fmaxf(r, 0.0f) * 524288.0f, 16777215.0f);      // 2^19; exact scaling, then round to nearest
        q[k] = (unsigned)__float2uint_rn(v);
    }
    if (i0 + 4 <= count && ((i0 * 3) & 3) == 0) {
        unsigned *o = reinterpret_cast<unsigned *>(out + i0 * 3);
        o[0] = q[0] | (q[1] << 24);
        o[1] = (q[1] >> 8) | (q[2] << 16);
        o[2] = (q[2] >> 16) | (q[3] << 8);
    } else {
        for (int k = 0; k < 4 && i0 + k < count; k++) {
            uint8_t *o = out + (i0 + k) * 3;
            o[0] = (uint8_t)q[k]; o[1] = (uint8_t)(q[k] >> 8); o[2] = (uint8_t)(q[k] >> 16);
        }
    }
}

__global__ void k_scan_noise(float *__restrict__ scans, long long count, double std_dev, uint64_t seed,
                             uint64_t offset) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    scans[i] = (float)((double)scans[i] + std_dev * normal_sample(seed, 0xFFFFFFFFull, offset + (uint64_t)i));
}

static int check_sim(const f110_sim *s) {
    if (!s) return F110_ERR_INVALID;
    if (s->num_envs <= 0 || s->num_agents <= 0) return F110_ERR_INVALID;
    if (s->integrator != 1 && s->integrator != 2) return F110_ERR_INTEGRATOR;
    if (!s->params || !s->state || !s->steer_buf || !s->steer_cnt || !s->scan_pose || !s->agent_poses ||
        !s->scans || !s->wall_flag || !s->collisions || !s->collision_idx)
        return F110_ERR_INVALID;
    return F110_OK;
}
static int check_map(const f110_map *m) {
    if (!m) return F110_ERR_INVALID;
    if (!m->dt || m->height <= 0 || m->width <= 0) return F110_ERR_NO_MAP;
    if (!m->sines || !m->cosines || m->theta_dis <= 0 || !(m->resolution > 0)) return F110_ERR_INVALID;
    return F110_OK;
}
static int check_beams(const f110_beams *b) {
    if (!b || b->num_beams <= 1 || !b->scan_angles || !b->cosines || !b->side_distances) return F110_ERR_INVALID;
    return F110_OK;
}

static unsigned long long *g_trace = nullptr;          // debug only: per-block timeline buffer (f110_debug_set_trace)
static unsigned long long *g_tile_counter = nullptr;   // debug only: lookups served from the shared-memory tile
// debug record of the kernels the last tick / f110_scan_layers of this thread launched (f110_debug_last_launch): host-side text only
static thread_local char g_launch_rec[768] = "";

static int num_sms() {
    static int n = 0;
    if (n <= 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            n = 132;                          // H100 SXM
    }
    return n;
}

// A/B switch for measurements (f110_debug_set_variant or F110_MARCH_VARIANT), interpreted by plan_march and nowhere else:
// 0 = default (k_march_lean, fp64 table, half of the queue dynamic); 66 / 60 / 61 = static dealing with 4 x 512 / 2 x 1024 /
// 8 x 256 threads per SM; 40 / 41 / 42 = dynamic with 4 x 512 / 3 x 512 / 2 x 1024; 43 / 45 = dynamic, 2 / 4 queue entries per
// ticket; 44 = static, 2 per ticket; 57 / 58 = dynamic, 3 x 512, 4 / 2 per ticket; 81-86 = ring hand-off through shared atomics
// (odd) or st.release / ld.acquire (even) with 4 / 2 entries per ticket / by run class; 20 / 22 = rank-coded table + shared LUT;
// 21 = 48 warps/SM; 30 / 31 = TMA tile 128 / 160 cells; 62-65 = thread-block clusters sharing a ticket counter; 1 / 6 = round-1
// persistent kernel (fp64 / coded); 7 / 9 = no queue (block per 64-beam tile); 13 = the literal k_raymarch; 90 = variant 0 on
// the padded row-major table even when a brick table is bound (f110_march_tables)
static int g_variant = -1, g_chunk = -1;
static bool g_no_brick = false;        // variant 90
// Dynamic second half of the queue (k_march_lean<DYN>): every block gets g_dyn_pct % of its fair share dealt statically and claims
// the rest in runs from one global counter, g_dyn_ahead runs ahead of their use.  50 % / 4 was the measured optimum at cfg3, cfg2x2
// and cfg2: the default of variant 0.
static int g_dyn_pct = 50, g_dyn_ahead = 4;
static int g_ipt[4] = {-1, -1, -1, 255};  // log2(entries per ticket): very heavy, heavy, light runs, dynamic tail (255 = by the class it starts in); -1 = by queue length
static int rm_variant() {
    if (g_variant < 0) {
        const char *e = getenv("F110_MARCH_VARIANT");
        g_variant = e ? atoi(e) : 0;
        if (g_variant == 90) { g_variant = 0; g_no_brick = true; }
    }
    return g_variant;
}
// log2 of the queue entries a block is dealt at a time (f110_debug_set_chunk or F110_MARCH_CHUNK)
static unsigned march_chunk() {
    if (g_chunk < 0) { const char *e = getenv("F110_MARCH_CHUNK"); g_chunk = e ? atoi(e) : 3; if (g_chunk < 0 || g_chunk > 6) g_chunk = 3; }
    return (unsigned)g_chunk;
}

// the brick table of a map (f110_map_brick, k_march_lean_brick): 4 x 4-cell bricks over the (height + 1) x (width + 1) padded
// table, bricks per row and elements (0 when the element index would not fit 32 bits)
#define F110_BRICK_MAX_BEAMS 1080
static unsigned long long brick_cols(const f110_map *map) { return ((unsigned long long)map->width + 4ull) / 4ull; }
static unsigned long long brick_elems(const f110_map *map) {
    const unsigned long long n = brick_cols(map) * 16ull * (((unsigned long long)map->height + 4ull) / 4ull);
    return n < (1ull << 32) ? n : 0ull;
}

// ------------------------------------------------------------------------------------ map geometry
// What the tick, f110_scan_layers and f110_render_views have to know about a map or map stack before they pick a kernel.
struct MapGeom {
    bool het;                  // canvas stack: layers of different sizes / origins (f110_map.layer_geom)
    bool mixres;               // ... of several resolutions (f110_map.layer_res)
    bool unrotated;            // the map's own origin has no yaw (a canvas stack carries its yaws in layer_rot)
    unsigned layers;           // at least 1
    double res_fine;           // the finest resolution of any layer
    double x_ext, y_ext;       // the extent at the coarsest resolution: bounds every layer's
    double orig_max, reach;    // largest origin coordinate of any layer; how far from the origin a ray can get
    bool reach_ok;             // origin, extent and ray reach stay well inside the absurd-coordinate bound (below)
    bool cells32, padded32;    // height x width, (height + 1) x (width + 1): the table's element index fits 32 bits
};
// F110_ERR_INVALID for per-layer tables on a map that cannot carry them: layer_rot needs a canvas stack with layer_res, layer_res
// a canvas stack and a sane resolution range, both metres only (no fast_path).
static int classify_map(const f110_map *map, MapGeom *g) {
    g->het = map->num_layers > 1 && map->layer_geom;
    const double res_min = map->layer_res_min, res_max = map->layer_res_max;
    if (map->layer_rot && (!g->het || !map->layer_res || map->fast_path)) return F110_ERR_INVALID;
    if (map->layer_res && (!g->het || map->fast_path || !(res_min > 0.0) || !(res_max >= res_min))) return F110_ERR_INVALID;
    g->mixres = g->het && map->layer_res;
    g->unrotated = map->orig_c == 1.0 && map->orig_s == 0.0;
    g->layers = map->num_layers > 1 ? (unsigned)map->num_layers : 1u;
    // The lean march kernels hand scan poses at absurd coordinates (|x| >= min(1e8 m, 1e9 cells)) to march_generic, which has no
    // row count: that is exact only while no ray from there can come back onto the map, i.e. the map, a ray's reach (max_range
    // plus one step of at most the map's diagonal) and the origin all stay below half of that bound.  Any other map takes the
    // literal arithmetic, which has the full row / column checks.
    // (a canvas stack: the largest origin of any layer and the canvas extent, which bounds every layer's)
    // (a rotated origin: the same bound keeps x_rot / res and y_rot / res below 2^31 for the scan poses k_dynamics passes to
    // the lean kernel, see `sane` there; march_generic_rot has the full row / column checks)
    // (a canvas stack of several resolutions: the extents at the coarsest layer resolution, the cell bound at the finest)
    g->res_fine = g->mixres ? res_min : map->resolution;
    g->x_ext = map->width * (g->mixres ? res_max : map->resolution);      // `width * resolution` (laser_models.py:79)
    g->y_ext = map->height * (g->mixres ? res_max : map->resolution);
    g->orig_max = fmax(fabs(map->orig_x), fabs(map->orig_y));
    if (g->het) g->orig_max = fmax(map->layer_orig_max, g->orig_max);
    g->reach = g->orig_max + 2.0 * (g->x_ext + g->y_ext) + map->max_range;
    g->reach_ok = g->reach < 0.5 * fmin(1e8, 1e9 * g->res_fine);
    g->cells32 = (unsigned long long)map->width * (unsigned long long)map->height < (1ull << 32);
    g->padded32 = (unsigned long long)(map->width + 1) * (unsigned long long)(map->height + 1) < (1ull << 32);
    return F110_OK;
}

// The beam LUT step of the lean kernels: theta_index_increment in Q16.48, and the replay guard.  The fixed-point index is within
// B * 2^-49 + 2^-48 of the real closed form, which is within B * 1.14e-13 of the reference's sequential sum (lidar.cuh): replay
// when the fraction (top 32 bits) is closer than that (x4) to an integer
static void lut_fixed_point(const f110_beams *beams, unsigned long long *inc_fx, unsigned *guard32) {
    *inc_fx = (unsigned long long)(beams->theta_index_increment * 281474976710656.0 + 0.5);
    const double guard = 4.0 * ((double)beams->num_beams * 1.2e-13 + 1e-12);
    *guard32 = (unsigned)(guard * 4294967296.0) + 2u;
}

// k_raymarch, thread per beam: the grid for `total` beams, 0 when it is not a legal one
#define F110_RAYMARCH_THREADS 256
static unsigned raymarch_blocks(long long total) {
    const long long blocks = (total + F110_RAYMARCH_THREADS - 1) / F110_RAYMARCH_THREADS;
    return (blocks <= 0 || blocks > 0x7fffffffll) ? 0u : (unsigned)blocks;
}

// ------------------------------------------------------------------------------------ the plan of a tick's ray march
// step_impl decides first and launches second: plan_march turns (sim, map, tables, beams, variant) into a MarchPlan by host
// arithmetic alone, the fillers below build the kernel parameter structs from it, launch_march_plan switches on the family, and
// the launch record is written from the plan.  Which configuration reaches which kernel:
//   LITERAL         k_raymarch, thread per beam: no cell march possible (map origin rotated without the lean tables, reach_ok
//                   false, sincos / cos_side missing) or variant 13
//   BLOCK_PER_TILE  k_march, block per 64-beam tile: cell march without the queue buffers (or variant 7 / 9)
//   PERSISTENT      k_march_persistent (round 1): queue, but not the lean kernel's tables / preconditions (or variant 1 / 6)
//   LEAN            k_march_lean: one map or a same-size stack, cell units or metres; block shape, ticket size and dynamic
//                   tail by queue length and variant
//   LEAN_BRICK      k_march_lean_brick: LEAN's single cell-unit map on the brick table, when one is bound (variant 0 only)
//   LEAN_HET        k_march_lean_het: canvas stack;   LEAN_HET_RES  k_march_lean_het_res: ... of several resolutions
//   LEAN_ROT        k_march_lean_rot: one metre map with a rotated origin, or a canvas stack with layer_rot
//   TILE            k_march_tile (variants 30 / 31): single cell-unit map with the padded code table
enum class MarchFamily { LITERAL, BLOCK_PER_TILE, PERSISTENT, LEAN, LEAN_BRICK, LEAN_HET, LEAN_HET_RES, LEAN_ROT, TILE };
struct MarchPlan {
    MarchFamily family;
    int variant;                 // (the record of a cluster launch names it)
    bool noise, count;           // NOISE / COUNT build of the kernel
    bool cell_units;             // march in cell units on the dt / res table (power-of-two resolution), else in metres
    bool layered;                // a map layer per env (f110_sim.env_layer on a stack)
    bool rot;                    // rotated origin(s): LEAN_ROT, or LITERAL when that kernel cannot run
    bool lean;                   // a lean family or TILE: k_dynamics writes the per-agent record, the tail may use PDL
    bool coded;                  // rank-coded table: variant 6 on the round-1 kernels, 20 / 22 on LEAN
    bool dyn;                    // LEAN / LEAN_BRICK: the second half of the queue is claimed dynamically
    int pt, minb;                // threads per block, blocks per SM (the launch bound of the kernel instance)
    dim3 grid;
    int ipt, ring;               // LEAN / LEAN_BRICK: queue entries per ticket (0 = by run class), ring hand-off flavour
    int cluster, cluster_pt;     // LEAN, variants 62-65: CTAs per cluster (0 = none) and its block size; pt / minb / grid hold
    unsigned cluster_grid;       // the shape to fall back to when the clusters do not fit the device
    int item_sub;                // 32-beam slices per queue item: 1, 2, or 0 = march_ipa matches neither
    int sub;                     // PERSISTENT: the kernel's SUB
    int tile_sz;                 // TILE
    int dyn_blocks, order_blocks, agent_queue;   // k_dynamics: agent blocks, queue-building blocks, 1 = the tile kernel's agent queue
    unsigned per_warp;           // queue entries per warp the ticket sizes were chosen for
    MarchQueue mq;
};

// queued_agents: the agents whose items the queue holds, -1 = all (a tick with a lidar mask queues the slots that have a lidar only)
static int plan_march(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                      const MapGeom &geom, int variant, MarchPlan *plan, long long queued_agents = -1) {
    MarchPlan p = {};
    const int NA = sim->num_envs * sim->num_agents;
    const long long QA = queued_agents < 0 ? (long long)NA : queued_agents;
    const unsigned sms = (unsigned)num_sms();
    p.variant = variant;
    p.noise = sim->noise_std > 0.0; p.count = sim->lookup_counter != nullptr;
    // work-item width: march_ipa = ceil(B/32) -> one 32-beam slice per item, ceil(B/64) -> two
    p.item_sub = (sim->march_ipa == (beams->num_beams + 31) / 32) ? 1 : (sim->march_ipa == (beams->num_beams + 63) / 64) ? 2 : 0;
    // the lean march kernel (march_lean.cuh): 32-beam queue items, `d > eps` == `d != 0` (every positive DT value exceeds
    // eps), fov < 2 pi (the doubled sin/cos LUT replaces the wrap), LUT indices that fit the Q16.48 fixed point
    const bool lean_tables = p.item_sub == 1 && sim->march_rec && map->sincos2 && map->eps >= 0.0 &&
                             (unsigned long long)NA * (unsigned long long)beams->num_beams < (1ull << 32) && geom.padded32 &&
                             map->dt_min_positive > map->eps && beams->fov > 0.0 && beams->fov < 6.283185307179586 &&
                             beams->theta_index_increment > 0.0 && map->theta_dis < 32768 && variant != 1 && variant != 6;
    const bool queue_tables = sim->march_cost && sim->march_order && sim->march_count && variant != 7 && p.item_sub != 0 &&
                              sim->march_ipa <= 256 && (unsigned long long)NA < (1ull << 22) && map->sincos && beams->cos_side &&
                              variant != 13;
    // rotated map origins run only on the lean kernel k_march_lean_rot (march_rot.cuh): one metre map that has every table
    // that kernel needs (any other takes k_raymarch), or a canvas stack with layer_rot
    const bool rot_single = !geom.unrotated && !(map->num_layers > 1) && !map->fast_path && queue_tables && lean_tables;
    p.rot = rot_single || (geom.het && map->layer_rot);
    const bool queued = queue_tables && (geom.unrotated || p.rot);
    // the march kernels that work on cell indices need an unrotated map origin (or k_march_lean_rot) and the interleaved tables;
    // cell units additionally a power-of-two resolution (fast_path) and the cell-unit table
    const bool cell_march = (geom.unrotated || p.rot) && map->sincos && beams->cos_side && geom.cells32 && geom.reach_ok &&
                            variant != 13;
    p.cell_units = cell_march && !p.rot && map->fast_path && map->dt_cells;
    p.layered = map->num_layers > 1 && sim->env_layer;
    if (map->num_layers > 1 && !cell_march) return F110_ERR_INVALID;     // stacked maps need the lean march kernels
    p.lean = queued && cell_march && lean_tables && (!p.cell_units || map->dt_cells_pad);
    // the TMA-tile kernel (march_tile.cuh; variants 30 / 31): single cell-unit map with the padded code table
    p.tile_sz = (variant == 31) ? 160 : 128;
    const bool tile = p.lean && (variant == 30 || variant == 31) && map->fast_path && map->dt_cells_pad && map->dt_codes_pad &&
                      map->dt_lut && !(map->num_layers > 1) && map->codes_pitch >= (unsigned)p.tile_sz && map->codes_pitch % 16 == 0 &&
                      map->height + 1 >= p.tile_sz && (unsigned long long)NA * (unsigned long long)sim->march_ipa < (1ull << 24);
    // a canvas stack runs only on the heterogeneous lean kernels (march_het.cuh, march_rot.cuh), one layer per env
    if (geom.het && (!p.lean || tile || !p.layered)) return F110_ERR_INVALID;
    p.dyn_blocks = (NA + 127) / 128;
    p.order_blocks = tile ? p.dyn_blocks
                   : queued ? (int)((QA * sim->march_ipa + 128 * F110_ORDER_ITEMS_PER_THREAD - 1) / (128 * F110_ORDER_ITEMS_PER_THREAD))
                   : 0;
    p.agent_queue = tile ? 1 : 0;

    if (!cell_march) {
        p.family = MarchFamily::LITERAL;
        p.pt = F110_RAYMARCH_THREADS;
        const unsigned blocks = raymarch_blocks((long long)NA * beams->num_beams);
        if (!blocks) return F110_ERR_INVALID;
        p.grid = dim3(blocks);
        *plan = p;
        return F110_OK;
    }
    const int bpa = (beams->num_beams + 63) / 64;
    if (bpa > 65000) return F110_ERR_INVALID;
    if (!queued) {
        p.family = MarchFamily::BLOCK_PER_TILE;
        p.coded = p.cell_units && !p.layered && map->dt_codes && map->dt_lut && variant == 6;   // measured: the fp64 table wins once issue-bound
        p.pt = 64; p.minb = (p.cell_units && variant == 9) ? 24 : 32;
        p.grid = dim3((unsigned)NA, (unsigned)bpa);
        *plan = p;
        return F110_OK;
    }

    MarchQueue &mq = p.mq;
    mq.cost = sim->march_cost; mq.order = sim->march_order; mq.count = sim->march_count;
    mq.ipa = (unsigned)sim->march_ipa; mq.items = (unsigned)QA * mq.ipa;
    mq.chunk_shift = march_chunk();
    mq.claim = sim->march_count + 3;
    // Dynamic tail of the queue (k_march_lean<DYN>): g_dyn_pct % of every block's share is dealt statically.  Whether the tail
    // runs depends on how many runs that leaves a block, so the queue is sized for the blocks per SM of the variant's dynamic
    // launch before the shape is final: the default (variants 0 / 40) runs 4 x 512 threads per SM, 41 / 57 / 58 3 x 512, 42 2 x 1024.
    // (Those four have their own shape on the single cell-unit map only; elsewhere they run 4 x 512 on a queue sized for it.)
    const int tail_minb = variant == 42 ? 2 : (variant == 41 || variant == 57 || variant == 58) ? 3 : 4;
    {
        const unsigned runs = (mq.items + (1u << mq.chunk_shift) - 1u) >> mq.chunk_shift;
        const unsigned blocks = sms * (unsigned)tail_minb;
        mq.dyn_ahead = (unsigned)g_dyn_ahead;
        mq.static_runs = (unsigned)((unsigned long long)runs * (unsigned)g_dyn_pct / 100ull / blocks);
        // entries per ticket by queue class (k_march_lean<IPT = 0>)
        unsigned sh[4];
        // (at least two tickets per run: with one, the 16 warps of a block could hold tickets of 16 runs at once and
        // the claim for run r + 16 could overwrite the ring slot of run r before it is read)
        const unsigned sh_max = mq.chunk_shift > 0u ? mq.chunk_shift - 1u : 0u;
        // queue entries per warp of the launch: one entry per ticket for the very heavy runs, four for the light ones, and
        // for the heavy runs two on a short queue, four on a longer one (measured at cfg2, cfg2x2 and n12288a1)
        p.per_warp = mq.items / (blocks * 16u);
        const int dflt[4] = {0, p.per_warp >= 27u ? 2 : 1, 2, 255};
        for (int z = 0; z < 4; z++) {
            const int want = g_ipt[z] < 0 ? dflt[z] : g_ipt[z];
            sh[z] = (z == 3 && want == 255) ? 255u : std::min((unsigned)want, sh_max);
        }
        mq.uniform_ipt4 = (g_ipt[0] >= 0 || g_ipt[1] >= 0 || g_ipt[2] >= 0 || mq.chunk_shift < 3u) ? 0u
                        : p.per_warp >= 72u ? 4u : p.per_warp >= 27u ? 2u : 0u;
        mq.ipt_shifts = sh[0] | (sh[1] << 8) | (sh[2] << 16) | (sh[3] << 24);
    }
    // Block shape at the same 64 warps/SM.  Two 1024-thread blocks per SM (32 warps share a ticket counter, the queue is dealt
    // to half as many blocks) beat four 512-thread blocks whenever a block gets enough items (cfg3, cfg5_2160, cfg2x2) and
    // lose when it does not (cfg2, 470 items per big block).
    const bool long_queue = (unsigned long long)mq.items >= 700ull * 2ull * (unsigned long long)sms;
    p.pt = 512; p.minb = 4; p.ipt = 1; p.ring = 0;

    if (!p.lean) {
        p.family = MarchFamily::PERSISTENT;
        p.coded = p.cell_units && !p.layered && map->dt_codes && map->dt_lut && variant == 6;
        p.sub = (p.cell_units && p.item_sub == 2) ? 2 : 1;
    } else if (tile) {
        p.family = MarchFamily::TILE;
    } else if (p.rot || geom.het) {
        // canvas stacks and rotated origins: static queue, one entry per ticket, the shape by the queue length alone
        p.family = p.rot ? MarchFamily::LEAN_ROT : geom.mixres ? MarchFamily::LEAN_HET_RES : MarchFamily::LEAN_HET;
        if (long_queue) { p.pt = 1024; p.minb = 2; }
    } else {
        p.coded = p.cell_units && !p.layered && map->dt_codes_pad && map->dt_lut && map->codes_pitch > (unsigned)map->width &&
                  (variant == 20 || variant == 22);
        // the brick table (f110_march_tables): a single fp64 cell-unit map on the default launch, up to 1080 beams per scan.
        // Measured (H100, bench.py, against the row-major table): 5-8 % off the march at 270-1080 beams, 4 % slower at 2160,
        // where a warp's rays are close enough together that the row-major gathers already touch few lines
        const bool brick = tables && tables->dt_cells_brick && p.cell_units && !p.layered && !(map->num_layers > 1) && !p.coded &&
                           variant == 0 && !g_no_brick && beams->num_beams <= F110_BRICK_MAX_BEAMS && brick_elems(map) != 0ull;
        p.family = brick ? MarchFamily::LEAN_BRICK : MarchFamily::LEAN;
        const bool dyn_variant = variant == 0 || (variant >= 40 && variant <= 43) || variant == 45 || variant == 57 || variant == 58 ||
                                 (variant >= 81 && variant <= 86);
        p.dyn = dyn_variant && !p.layered && mq.static_runs >= mq.dyn_ahead;
        const bool occ3 = variant == 21 || variant == 22 || variant == 41;          // 48 warps per SM (3 x 512 threads, 40 registers)
        // the single fp64 cell-unit map: the only launch with shapes of its own per variant
        const bool plain = p.cell_units && !p.layered && !p.coded;
        const unsigned cs = mq.chunk_shift;                                          // a ticket of 2^k entries needs runs of 2^(k+1)
        // variants 60 / 61 / 66 force 2 x 1024 / 8 x 256 / 4 x 512; the brick launch is always 4 x 512
        const bool big = !brick && (variant == 60 || (variant != 61 && variant != 66 && variant != 44 && variant != 21 && variant != 22 &&
                                                      !p.dyn && !p.coded && !occ3 && long_queue));
        if (big && !p.coded) { p.pt = 1024; p.minb = 2; }
        else if (plain && variant == 61) { p.pt = 256; p.minb = 8; }
        else if (plain && variant == 44 && cs >= 1) p.ipt = 2;
        else if (p.dyn && !p.cell_units) { p.ipt = 0; p.ring = 2; }
        else if (p.dyn) {                                                            // (dyn: neither layered nor coded, so `plain`)
            if (variant == 43 && cs >= 1) p.ipt = 2;
            else if (variant == 45 && cs >= 2) p.ipt = 4;
            else if (variant >= 81 && variant <= 86 && cs >= 3) { p.ipt = variant <= 82 ? 4 : variant <= 84 ? 2 : 0; p.ring = (variant & 1) ? 1 : 2; }
            else if (variant == 57 && cs >= 3) { p.minb = tail_minb; p.ipt = 4; }
            else if (variant == 58 && cs >= 2) { p.minb = tail_minb; p.ipt = 2; }
            else if (variant == 42) { p.pt = 1024; p.minb = tail_minb; }
            else if (occ3) p.minb = tail_minb;
            else if (variant != 40) {                                                // 40: one entry per ticket, compile-time
                // Long queues (>= 72 entries per warp: cfg3, the beam sweep): four entries per ticket throughout, fixed at compile
                // time -- faster at cfg3 than dealing the very heavy runs one or two entries at a time, and than one entry per
                // ticket everywhere.  Shorter queues: ticket size by the class of the run (dyn_queue_position_zoned), which is
                // what keeps four very heavy entries from landing on one warp (a uniform 4 is far slower at cfg2x2 and cfg2).
                // Medium queues (27..72 entries per warp: cfg2x2, n12288a1): two entries per ticket (slightly ahead of by class).
                // The ring words go through st.release / ld.acquire (RING = 2; the volatile formulation times the same, the one
                // in shared atomics that racecheck accepts is slower).
                p.ipt = variant == 0 ? (int)mq.uniform_ipt4 : 0; p.ring = 2;
            }
        } else if (p.cell_units && !p.layered && occ3) p.minb = 3;             // (fp64 or coded table)
        // thread-block clusters sharing one ticket counter (variants 62-65), plain noise-free marching only
        if (plain && !p.noise && !p.count && variant >= 62 && variant <= 65) {
            p.cluster = (variant == 63) ? 2 : (variant == 65) ? 8 : 4;
            p.cluster_pt = variant <= 63 ? 1024 : 512;
            p.cluster_grid = sms * (variant <= 63 ? 2u : 4u) / (unsigned)p.cluster * (unsigned)p.cluster;
        }
    }
    p.grid = dim3(sms * (unsigned)p.minb);
    *plan = p;
    return F110_OK;
}

// ------------------------------------------------------------------------------------ kernel parameters from the plan
static FirstLookup fill_first_lookup(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const MapGeom &geom,
                                     const MarchPlan &p) {
    FirstLookup fl;
    const bool cell_march = p.family != MarchFamily::LITERAL;
    fl.cells = cell_march ? (p.cell_units ? map->dt_cells : map->dt) : nullptr;
    fl.metres = p.cell_units ? 0 : 1;
    fl.res = map->resolution; fl.orig_x = map->orig_x; fl.orig_y = map->orig_y;
    fl.x_max = map->width * map->resolution; fl.y_max = map->height * map->resolution;
    fl.env_layer = p.layered ? sim->env_layer : nullptr;
    fl.layer_stride = (unsigned long long)map->width * (unsigned long long)map->height;
    fl.inv_res = 1.0 / geom.res_fine; fl.ox = map->orig_x * fl.inv_res; fl.oy = map->orig_y * fl.inv_res;
    fl.width = (unsigned)map->width; fl.height = (unsigned)map->height;
    fl.last = (unsigned)map->width * (unsigned)map->height - 1u;
    fl.agent_queue = p.agent_queue;
    fl.rec = p.lean ? reinterpret_cast<double2 *>(sim->march_rec) : nullptr;
    fl.side_max = beams->side_max > 0.0 ? beams->side_max : INFINITY;
    fl.ttc_margin = sim->ttc_thresh * 1.000001;
    fl.rec_layer_stride = p.cell_units ? (unsigned long long)(map->width + 1) * (unsigned long long)(map->height + 1) : fl.layer_stride;
    fl.layer_geom = geom.het ? map->layer_geom : nullptr;
    fl.layer_res = geom.mixres ? map->layer_res : nullptr;
    fl.layer_rot = geom.het ? map->layer_rot : nullptr;
    fl.rotated = p.rot && !geom.het ? 1 : 0;
    fl.orig_c = map->orig_c; fl.orig_s = map->orig_s;
    return fl;
}

// the round-1 kernels (BLOCK_PER_TILE, PERSISTENT)
static MarchK fill_march_k(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const MarchPlan &p) {
    MarchK k;
    k.codes = map->dt_codes; k.lut = map->dt_lut; k.cells = map->dt_cells;
    k.sincos = reinterpret_cast<const double2 *>(map->sincos);
    k.cos_side = reinterpret_cast<const double2 *>(beams->cos_side);
    k.scan_pose = reinterpret_cast<const double2 *>(sim->scan_pose);
    k.vel = sim->state + (size_t)3 * (sim->num_envs * sim->num_agents);
    k.out = sim->scans; k.wall_flag = sim->wall_flag;
    k.lookup_counter = sim->lookup_counter; k.tick_counter = sim->tick_counter;
    k.inv_res = 1.0 / map->resolution; k.res = map->resolution;
    k.ox = map->orig_x * k.inv_res; k.oy = map->orig_y * k.inv_res;
    k.eps = map->eps * k.inv_res; k.tmax = map->max_range * k.inv_res;
    k.inc = beams->theta_index_increment; k.theta_dis_f = (double)map->theta_dis;
    k.ti_guard = 4.0 * ((double)beams->num_beams * 1.14e-13 + 1e-12);
    k.ttc_thresh = sim->ttc_thresh; k.ttc_margin = sim->ttc_thresh * 1.000001;
    k.noise_std = sim->noise_std; k.noise_seed = sim->noise_seed;
    k.width = (unsigned)map->width; k.height = (unsigned)map->height;
    k.last = (unsigned)map->width * (unsigned)map->height - 1u;
    k.B = beams->num_beams;
    k.env_layer = p.layered ? sim->env_layer : nullptr;
    k.layer_stride = (unsigned long long)map->width * (unsigned long long)map->height;
    k.num_agents = (unsigned)sim->num_agents;
    k.trace = g_trace;
    k.dt = map->dt; k.orig_x = map->orig_x; k.orig_y = map->orig_y;
    k.x_max = map->width * map->resolution; k.y_max = map->height * map->resolution;
    k.dt_oob = map->dt_oob; k.eps_m = map->eps; k.max_range = map->max_range;
    return k;
}

// the lean families and the tile kernel
static LeanK fill_lean_k(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                         const MarchPlan &p) {
    LeanK q;
    const bool brick = p.family == MarchFamily::LEAN_BRICK;
    q.table = brick ? tables->dt_cells_brick : p.cell_units ? map->dt_cells_pad : map->dt;
    q.codes = map->dt_codes_pad; q.lut = map->dt_lut;
    q.sincos2 = reinterpret_cast<const double2 *>(map->sincos2);
    q.cos_side = reinterpret_cast<const double2 *>(beams->cos_side);
    q.rec = reinterpret_cast<const double2 *>(sim->march_rec);
    q.out = sim->scans; q.wall_flag = sim->wall_flag;
    q.lookup_counter = sim->lookup_counter; q.tick_counter = sim->tick_counter;
    q.res = map->resolution; q.inv_res = 1.0 / map->resolution;
    if (p.cell_units) { q.ox = map->orig_x * q.inv_res; q.oy = map->orig_y * q.inv_res; q.tmax = map->max_range * q.inv_res; }
    else { q.ox = map->orig_x; q.oy = map->orig_y; q.tmax = map->max_range; }
    q.x_max = map->width * map->resolution; q.y_max = map->height * map->resolution;
    q.ttc_thresh = sim->ttc_thresh; q.ttc_margin = sim->ttc_thresh * 1.000001;
    q.noise_std = sim->noise_std; q.noise_seed = sim->noise_seed;
    q.inc = beams->theta_index_increment; q.theta_dis_f = (double)map->theta_dis;
    lut_fixed_point(beams, &q.inc_fx, &q.guard32);
    q.width = (unsigned)map->width; q.height = (unsigned)map->height;
    q.last = (unsigned)map->width * (unsigned)map->height - 1u;
    q.B = beams->num_beams;
    q.layer_stride = (unsigned long long)map->width * (unsigned long long)map->height;
    q.layer_stride_lean = p.cell_units ? (unsigned long long)(map->width + 1) * (unsigned long long)(map->height + 1) : q.layer_stride;
    q.dt = map->dt; q.orig_x = map->orig_x; q.orig_y = map->orig_y;
    q.brick_cols1 = brick ? (unsigned)(brick_cols(map) - 1ull) : 0u; q.unused = 0u;
    q.eps_m = map->eps; q.max_range = map->max_range;
    q.codes_pitch = map->codes_pitch;
    return q;
}

// ------------------------------------------------------------------------------------ launches
// Launch with the programmatic-stream-serialization attribute (PDL) when enabled: the kernel may become resident before
// its predecessor in the stream has finished and synchronises itself with pdl_wait().
// measured: inside a CUDA graph PDL wins nothing, so it is off by default and kept as a switch (f110_debug_set_pdl); k_tail
// is fastest with the 64-register budget (occupancy beats spills against 96 / 128 registers)
static int g_pdl = 0;
static int g_tail_minb = 8;
static int g_tail2_threads = F110_TAIL2_THREADS, g_tail2_agents = 64;    // block shape of k_tail2 (f110_debug_set_tail2)
static int g_tail2_forced = 0;                                            // agents per block forced exactly (debug setter, agents > 64 or < 0)
static int g_tail2 = 1;          // 2 <= A <= 4: the two-phase k_tail2 (f110_debug_set_tail(-1) switches back to k_tail for the A/B)
template <typename... KArgs, typename... Args>
static void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = (pdl && g_pdl) ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, args...);
}
// launch in thread-block clusters of `cl` CTAs (grid must be a multiple of cl)
template <typename... KArgs, typename... Args>
static void launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, unsigned cl, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = 0; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kernel, args...);
}
// does a grid of `blocks` CTAs in clusters of CL fit on the device at once?  (a persistent kernel needs all of them resident)
template <typename K>
static bool clusters_fit(K kernel, unsigned blocks, unsigned threads, unsigned cl) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = 0;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) { cudaGetLastError(); return false; }
    return (unsigned)n * cl >= blocks;
}

// The NOISE / COUNT build of a kernel: f(noise, count) with the two run-time flags as std::true_type / std::false_type.
// Counting runs are noise-free (step_impl rejects the combination), so (true, true) is never instantiated.
template <typename F>
static void dispatch_noise_count(bool noise, bool count, F &&f) {
    if (count) f(std::false_type(), std::true_type());
    else if (noise) f(std::true_type(), std::false_type());
    else f(std::false_type(), std::false_type());
}
#define F110_NC(n, c) decltype(n)::value, decltype(c)::value

// The launch helpers below decide nothing: each *_t is one kernel instance the library holds, launches it when it is the one the
// plan names and says so; a plan that names none of them is an error (F110_ERR_INVALID), never another kernel.
static int launch_raymarch(const MapView &mv, const BeamView &bv, const MarchArgs &g, bool fast, bool standalone, unsigned blocks,
                           cudaStream_t st) {
    const dim3 grid(blocks), pt(F110_RAYMARCH_THREADS);
    if (fast) {
        if (standalone) k_raymarch<true, true><<<grid, pt, 0, st>>>(mv, bv, g);
        else k_raymarch<true, false><<<grid, pt, 0, st>>>(mv, bv, g);
    } else {
        if (standalone) k_raymarch<false, true><<<grid, pt, 0, st>>>(mv, bv, g);
        else k_raymarch<false, false><<<grid, pt, 0, st>>>(mv, bv, g);
    }
    LAUNCH_CHECK("k_raymarch");
    return F110_OK;
}

template <int MINB, bool CELLS>
static bool launch_block_per_tile_t(const MarchPlan &p, const MarchK &k, cudaStream_t st) {
    if (p.minb != MINB || p.cell_units != CELLS) return false;
    dispatch_noise_count(p.noise, p.count, [&](auto n, auto c) {
        if (p.coded && CELLS) k_march<CELLS, F110_NC(n, c), MINB, CELLS><<<p.grid, p.pt, 0, st>>>(k);
        else k_march<false, F110_NC(n, c), MINB, CELLS><<<p.grid, p.pt, 0, st>>>(k);
    });
    return true;
}

template <int PT, int SUB, bool CELLS>
static bool launch_persistent_t(const MarchPlan &p, const MarchK &k, cudaStream_t st) {
    if (p.pt != PT || p.sub != SUB || p.cell_units != CELLS) return false;
    if (k.trace) {
        if (p.coded && CELLS) k_march_persistent<CELLS, false, false, true, PT, SUB, CELLS><<<p.grid, PT, 0, st>>>(k, p.mq);
        else k_march_persistent<false, false, false, true, PT, SUB, CELLS><<<p.grid, PT, 0, st>>>(k, p.mq);
    } else dispatch_noise_count(p.noise, p.count, [&](auto n, auto c) {
        if (p.coded && CELLS) k_march_persistent<CELLS, F110_NC(n, c), false, PT, SUB, CELLS><<<p.grid, PT, 0, st>>>(k, p.mq);
        else k_march_persistent<false, F110_NC(n, c), false, PT, SUB, CELLS><<<p.grid, PT, 0, st>>>(k, p.mq);
    });
    return true;
}

template <int TABLE, bool CELLS, bool LAYERED, int MINB, bool DYN = false, int PT = 512, int IPT = 1, int RING = 0>
static bool launch_lean_t(const MarchPlan &p, const LeanK &q, bool pdl, cudaStream_t st) {
    if (p.coded != (TABLE == 1) || p.cell_units != CELLS || p.layered != LAYERED || p.minb != MINB || p.dyn != DYN || p.pt != PT ||
        p.ipt != IPT || p.ring != RING)
        return false;
    dispatch_noise_count(p.noise, p.count, [&](auto n, auto c) {
        launch_k(k_march_lean<TABLE, F110_NC(n, c), CELLS, LAYERED, PT, MINB, DYN, 1, IPT, RING>, p.grid, dim3(PT), 0, st, pdl, q, p.mq);
    });
    return true;
}
static bool launch_lean(const MarchPlan &p, const LeanK &q, bool pdl, cudaStream_t st) {
    // <TABLE, CELLS, LAYERED, MINB, DYN, PT, IPT, RING>: static dealing in the three block shapes; the dynamic tail with its
    // ticket sizes and ring flavours, single cell-unit map; the dynamic tail in metres
    return launch_lean_t<0, false, true, 2, false, 1024>(p, q, pdl, st) || launch_lean_t<0, false, false, 2, false, 1024>(p, q, pdl, st) ||
           launch_lean_t<0, true, true, 2, false, 1024>(p, q, pdl, st) || launch_lean_t<0, true, false, 2, false, 1024>(p, q, pdl, st) ||
           launch_lean_t<0, false, true, 4>(p, q, pdl, st) || launch_lean_t<0, false, false, 4>(p, q, pdl, st) ||
           launch_lean_t<0, true, true, 4>(p, q, pdl, st) || launch_lean_t<0, true, false, 4>(p, q, pdl, st) ||
           launch_lean_t<0, true, false, 3>(p, q, pdl, st) || launch_lean_t<1, true, false, 4>(p, q, pdl, st) ||
           launch_lean_t<1, true, false, 3>(p, q, pdl, st) || launch_lean_t<0, true, false, 8, false, 256>(p, q, pdl, st) ||
           launch_lean_t<0, true, false, 4, false, 512, 2>(p, q, pdl, st) ||
           launch_lean_t<0, true, false, 4, true, 512, 4, 2>(p, q, pdl, st) || launch_lean_t<0, true, false, 4, true, 512, 2, 2>(p, q, pdl, st) ||
           launch_lean_t<0, true, false, 4, true, 512, 0, 2>(p, q, pdl, st) || launch_lean_t<0, true, false, 4, true, 512, 4, 1>(p, q, pdl, st) ||
           launch_lean_t<0, true, false, 4, true, 512, 2, 1>(p, q, pdl, st) || launch_lean_t<0, true, false, 4, true, 512, 0, 1>(p, q, pdl, st) ||
           launch_lean_t<0, true, false, 4, true>(p, q, pdl, st) || launch_lean_t<0, true, false, 4, true, 512, 2>(p, q, pdl, st) ||
           launch_lean_t<0, true, false, 4, true, 512, 4>(p, q, pdl, st) || launch_lean_t<0, true, false, 3, true>(p, q, pdl, st) ||
           launch_lean_t<0, true, false, 3, true, 512, 4>(p, q, pdl, st) || launch_lean_t<0, true, false, 3, true, 512, 2>(p, q, pdl, st) ||
           launch_lean_t<0, true, false, 2, true, 1024>(p, q, pdl, st) ||
           launch_lean_t<0, false, false, 4, true, 512, 0, 2>(p, q, pdl, st);
}
// thread-block clusters (variants 62-65); false when the plan names another shape or the clusters do not fit the device
template <int PT, int MINB, int CL>
static bool launch_lean_cluster_t(const MarchPlan &p, const LeanK &q, cudaStream_t st) {
    auto k = k_march_lean<0, false, false, true, false, PT, MINB, false, CL>;
    if (p.cluster_pt != PT || p.cluster != CL || !clusters_fit(k, p.cluster_grid, PT, CL)) return false;
    launch_cluster(k, dim3(p.cluster_grid), dim3(PT), CL, st, q, p.mq);
    return true;
}
// k_march_lean_brick: the shapes of LEAN's single cell-unit map at variant 0
template <bool DYN, int IPT, int RING>
static bool launch_brick_t(const MarchPlan &p, const LeanK &q, bool pdl, cudaStream_t st) {
    if (p.pt != 512 || p.minb != 4 || p.dyn != DYN || p.ipt != IPT || p.ring != RING) return false;
    dispatch_noise_count(p.noise, p.count, [&](auto n, auto c) {
        launch_k(k_march_lean_brick<F110_NC(n, c), 512, 4, DYN, IPT, RING>, p.grid, dim3(512), 0, st, pdl, q, p.mq);
    });
    return true;
}
// canvas stacks (march_het.cuh): 2 x 1024 threads per SM for long queues, else 4 x 512
template <bool CELLS, int PT, int MINB>
static bool launch_het_t(const MarchPlan &p, const LeanK &q, const LayerGeomK &g, bool pdl, cudaStream_t st) {
    if (p.cell_units != CELLS || p.pt != PT || p.minb != MINB) return false;
    dispatch_noise_count(p.noise, p.count, [&](auto n, auto c) {
        launch_k(k_march_lean_het<F110_NC(n, c), CELLS, PT, MINB>, p.grid, dim3(PT), 0, st, pdl, q, g, p.mq);
    });
    return true;
}
// canvas stacks of several resolutions (f110_map.layer_res): metres only
template <int PT, int MINB>
static bool launch_het_res_t(const MarchPlan &p, const LeanK &q, const LayerGeomK &g, const double *layer_res, bool pdl, cudaStream_t st) {
    if (p.pt != PT || p.minb != MINB) return false;
    dispatch_noise_count(p.noise, p.count, [&](auto n, auto c) {
        launch_k(k_march_lean_het_res<F110_NC(n, c), PT, MINB>, p.grid, dim3(PT), 0, st, pdl, q, g, layer_res, p.mq);
    });
    return true;
}
// rotated map origins (march_rot.cuh): one map, or a canvas stack with f110_map.layer_rot; metres
template <int PT, int MINB>
static bool launch_rot_t(const MarchPlan &p, const LeanK &q, const RotGeomK &g, bool pdl, cudaStream_t st) {
    if (p.pt != PT || p.minb != MINB) return false;
    dispatch_noise_count(p.noise, p.count, [&](auto n, auto c) {
        launch_k(k_march_lean_rot<F110_NC(n, c), PT, MINB>, p.grid, dim3(PT), 0, st, pdl, q, g, p.mq);
    });
    return true;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link against libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// the TMA descriptor of the padded code table in boxes of tile x tile cells
static int encode_code_tiles(const f110_map *map, int tile, CUtensorMap *tm) {
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) return cuda_fail(cudaErrorNotSupported, "cuTensorMapEncodeTiled entry point");
    const cuuint64_t dims[2] = { (cuuint64_t)map->codes_pitch, (cuuint64_t)(map->height + 1) };
    const cuuint64_t strides[1] = { (cuuint64_t)map->codes_pitch };
    const cuuint32_t box[2] = { (cuuint32_t)tile, (cuuint32_t)tile };
    const cuuint32_t estr[2] = { 1u, 1u };
    const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void *)map->dt_codes_pad, dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? F110_OK : cuda_fail(cudaErrorInvalidValue, "cuTensorMapEncodeTiled");
}
// k_march_tile: 4 x 512 threads per SM
template <int TILE, int NSLOT>
static bool launch_tile_t(const MarchPlan &p, const TileK &t, const CUtensorMap &tm, cudaStream_t st, cudaError_t *e) {
    if (p.tile_sz != TILE) return false;
    const size_t smem = sizeof(TileSmem<TILE, NSLOT>);
    dispatch_noise_count(p.noise, p.count, [&](auto n, auto c) {
        auto k = k_march_tile<F110_NC(n, c), TILE, NSLOT, 512, 4>;
        *e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (*e == cudaSuccess) k<<<p.grid, 512, smem, st>>>(t, tm);
    });
    return true;
}

// Enqueue the march the plan names.  (A cluster launch that does not fit the device falls back to the plan's ordinary shape and
// clears plan.cluster, so that the launch record says what ran.)
static int launch_march_plan(MarchPlan &p, const f110_sim *sim, const f110_map *map, const f110_march_tables *tables,
                             const f110_beams *beams, const MapGeom &geom, bool pdl, cudaStream_t st) {
    bool ok = false;
    switch (p.family) {
    case MarchFamily::LITERAL: {
        MarchArgs g;
        g.scan_pose = sim->scan_pose;
        g.vel = sim->state + (size_t)3 * (sim->num_envs * sim->num_agents);
        g.out_f32 = sim->scans;
        g.out_f64 = nullptr;
        g.wall_flag = sim->wall_flag;
        g.lookup_counter = sim->lookup_counter;
        g.tick_counter = sim->tick_counter;
        g.ttc_thresh = sim->ttc_thresh;
        g.noise_std = sim->noise_std;
        g.noise_seed = sim->noise_seed;
        g.total = (long long)(sim->num_envs * sim->num_agents) * beams->num_beams;
        return launch_raymarch(make_view(map), make_view(beams), g, map->fast_path != 0, false, p.grid.x, st);
    }
    case MarchFamily::BLOCK_PER_TILE: {
        const MarchK k = fill_march_k(sim, map, beams, p);
        ok = launch_block_per_tile_t<32, false>(p, k, st) || launch_block_per_tile_t<24, true>(p, k, st) ||
             launch_block_per_tile_t<32, true>(p, k, st);
        break;
    }
    case MarchFamily::PERSISTENT: {
        const MarchK k = fill_march_k(sim, map, beams, p);
        ok = launch_persistent_t<512, 1, false>(p, k, st) || launch_persistent_t<512, 2, true>(p, k, st) ||
             launch_persistent_t<512, 1, true>(p, k, st);
        break;
    }
    case MarchFamily::LEAN: {
        const LeanK q = fill_lean_k(sim, map, tables, beams, p);
        if (p.cluster && !(launch_lean_cluster_t<1024, 2, 4>(p, q, st) || launch_lean_cluster_t<1024, 2, 2>(p, q, st) ||
                           launch_lean_cluster_t<512, 4, 4>(p, q, st) || launch_lean_cluster_t<512, 4, 8>(p, q, st))) {
            if (getenv("F110_DEBUG")) fprintf(stderr, "f110: cluster variant %d does not fit, using the default launch\n", p.variant);
            p.cluster = 0;
        }
        ok = p.cluster || launch_lean(p, q, pdl, st);
        break;
    }
    case MarchFamily::LEAN_BRICK: {
        const LeanK q = fill_lean_k(sim, map, tables, beams, p);
        ok = launch_brick_t<false, 1, 0>(p, q, pdl, st) || launch_brick_t<true, 4, 2>(p, q, pdl, st) ||
             launch_brick_t<true, 2, 2>(p, q, pdl, st) || launch_brick_t<true, 0, 2>(p, q, pdl, st);
        break;
    }
    case MarchFamily::LEAN_HET:
    case MarchFamily::LEAN_HET_RES: {
        const LeanK q = fill_lean_k(sim, map, tables, beams, p);
        LayerGeomK g;
        g.layer_geom = map->layer_geom; g.env_layer = sim->env_layer; g.num_agents = (unsigned)sim->num_agents;
        if (p.family == MarchFamily::LEAN_HET_RES)
            ok = launch_het_res_t<1024, 2>(p, q, g, map->layer_res, pdl, st) || launch_het_res_t<512, 4>(p, q, g, map->layer_res, pdl, st);
        else
            ok = launch_het_t<true, 1024, 2>(p, q, g, pdl, st) || launch_het_t<false, 1024, 2>(p, q, g, pdl, st) ||
                 launch_het_t<true, 512, 4>(p, q, g, pdl, st) || launch_het_t<false, 512, 4>(p, q, g, pdl, st);
        break;
    }
    case MarchFamily::LEAN_ROT: {
        const LeanK q = fill_lean_k(sim, map, tables, beams, p);
        const bool het = geom.het;
        RotGeomK g;
        g.layer_geom = het ? map->layer_geom : nullptr; g.layer_res = het ? map->layer_res : nullptr;
        g.layer_rot = het ? map->layer_rot : nullptr; g.env_layer = het ? sim->env_layer : nullptr;
        g.num_agents = (unsigned)sim->num_agents;
        g.orig = make_double2(map->orig_x, map->orig_y); g.ext = make_double2(map->width * map->resolution, map->height * map->resolution);
        g.res = make_double2(map->resolution, 1.0 / map->resolution); g.rot = make_double2(map->orig_c, map->orig_s);
        ok = launch_rot_t<1024, 2>(p, q, g, pdl, st) || launch_rot_t<512, 4>(p, q, g, pdl, st);
        break;
    }
    case MarchFamily::TILE: {
        TileK t;
        t.l = fill_lean_k(sim, map, tables, beams, p);
        t.order = sim->march_order; t.count = sim->march_count; t.claim = sim->march_count + 3;
        t.cost = sim->march_cost; t.agents = (unsigned)(sim->num_envs * sim->num_agents); t.ipa = (unsigned)sim->march_ipa;
        t.ipa_magic = (unsigned)(4294967296ull / (unsigned long long)sim->march_ipa) + 1u;
        t.codes_pitch = map->codes_pitch;
        t.c_max = (int)map->codes_pitch - p.tile_sz; t.r_max = map->height + 1 - p.tile_sz;
        t.tile_counter = g_tile_counter;
        CUtensorMap tm;
        int rc;
        if ((rc = encode_code_tiles(map, p.tile_sz, &tm))) return rc;
        cudaError_t e = cudaSuccess;
        ok = launch_tile_t<160, 2>(p, t, tm, st, &e) || launch_tile_t<128, 3>(p, t, tm, st, &e);
        if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(k_march_tile)");
        break;
    }
    }
    if (!ok) return F110_ERR_INVALID;
    LAUNCH_CHECK("k_march");
    return F110_OK;
}

// ------------------------------------------------------------------------------------ the tail of a tick
struct TailOpts {
    bool fused;              // k_tail instead of k_finalize
    int env_level;
    AutoResetArgs ar;
};
// what launch_tail launched, for the launch record
struct TailShape {
    enum { TAIL2, TAIL, FINALIZE, NOSCAN } kernel;
    int epb, threads, grid;          // envs per block, block size, blocks
    int cast_grid;                   // NOSCAN (a tick with a lidar mask): blocks of k_lidar_cast before k_tail_noscan
    size_t smem;                     // TAIL2
    int lb_threads, lb_minb;         // TAIL: the launch bounds of the instance
    bool separate;                   // FINALIZE standing in for the fused tail (more than 32 agents per env)
};

// largest value a scan entry can hold: the max_range clamp plus 8 sigma of the optional noise
static double max_scan_range(const f110_sim *sim, const f110_map *map) {
    return map->max_range + 8.0 * (sim->noise_std > 0.0 ? sim->noise_std : 0.0) + 1e-3;
}

static int launch_tail(const f110_sim *sim, const f110_map *map, const BeamView &bv, const TailOpts *tail, bool pdl, cudaStream_t st,
                       TailShape *shape) {
    const int NA = sim->num_envs * sim->num_agents;
    const bool fused = tail && tail->fused;
    TailShape &ts = *shape;
    const double max_scan = max_scan_range(sim, map);
    // k_tail2 (2 <= A <= 4): faster than k_tail at cfg3 and, once its blocks are small enough to fill the GPU, at cfg2x2
    if (sim->num_agents >= 2 && sim->num_agents <= 4 && g_tail2) {
        // two-phase tail: ~64 agents per block (thread per (ego, opponent) pair for the scalar work, warp per ego for the beams);
        // f110_step (no lap logic, no auto-reset) runs the same kernel with the env-level phase switched off
        // up to 64 agents per block, fewer when that would leave SMs without a block (cfg2x2: 4096 envs / 32 = 128 blocks lost
        // against 8 envs per block)
        int epb = g_tail2_forced ? max(1, g_tail2_agents / sim->num_agents) : max(1, min(g_tail2_agents / sim->num_agents, sim->num_envs / (4 * num_sms())));
        AutoResetArgs no_ar;
        no_ar.start_poses = nullptr; no_ar.num_start = 0; no_ar.pose_gap = 0; no_ar.seed = 0; no_ar.tick_host = 0;
        no_ar.num_tables = 0;
        // big blocks (>= 48 agents) run 256 threads, small ones 128 (measured: 256:64 best at cfg3, 128:12 at cfg2x2)
        int t2 = (g_tail2_threads != F110_TAIL2_THREADS) ? g_tail2_threads : (epb * sim->num_agents >= 48 ? 256 : 128);
        if (!g_tail2_forced && g_tail2_threads == F110_TAIL2_THREADS) {
            // Whole waves.  With 80 registers an SM holds six 128-thread blocks (three of 256 threads); a grid of about 1.4 waves
            // leaves the GPU two-thirds empty for the second half of the kernel, and grids of whole waves measured about a quarter
            // faster.  So: 128-thread blocks of up to 47 agents, and as many envs per block as fill a whole number of waves
            // (the wave size comes from the occupancy query and the SM count, not from a fixed device).
            // Re-swept with the flat phase 2 (every thread casts), k_tail2 in us on an H100 80GB HBM3 at 700 W, threads:agents:
            //   cfg3 (16384 x 2):  this rule (128:42, one wave) 32.8, 256:42 33.3, 256:96 35.8, 128:24 40.8, 256:16 46.6, 128:12 54.2
            //   cfg2x2 (4096 x 2): this rule (128:12) 19.8 (forced to the same shape 20.1), 256:16 21.4, 128:24 23.8, 256:42 28.1
            // so the rule stands.
            static int per_sm = 0;                          // resident 128-thread blocks per SM
            if (per_sm == 0) {
                const size_t sm0 = tail2_smem_bytes(47 / sim->num_agents, sim->num_agents);
                if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_tail2, 128, sm0) != cudaSuccess || per_sm < 1) { per_sm = -1; cudaGetLastError(); }
            }
            if (per_sm > 0) {
                const long long cap = (long long)per_sm * num_sms();
                const long long emax = max(1, 47 / sim->num_agents);
                const long long waves = (sim->num_envs + cap * emax - 1) / (cap * emax);
                epb = (int)((sim->num_envs + waves * cap - 1) / (waves * cap));
                t2 = 128;
            }
        }
        ts.kernel = TailShape::TAIL2; ts.epb = epb; ts.threads = t2; ts.grid = (sim->num_envs + epb - 1) / epb;
        ts.smem = tail2_smem_bytes(epb, sim->num_agents);
        if (ts.smem > 40 * 1024)   // with the ~4.6 KB of static arrays past the 48 KB default: forced shapes of A = 4 only
            cudaFuncSetAttribute(k_tail2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ts.smem);
        launch_k(k_tail2, dim3(ts.grid), dim3(t2), ts.smem, st, pdl, *sim, bv, fused ? (int)tail->env_level : 0,
                 fused ? tail->ar : no_ar, max_scan, epb);
        LAUNCH_CHECK("k_tail2");
    } else if (fused && sim->num_agents <= 32) {
        // whole envs per block, ~4 warps per block: A = 1 -> 4 envs, A = 2 -> 2 envs, A >= 4 -> 1 env
        const int epb = sim->num_agents >= 4 ? 1 : 4 / sim->num_agents;
        const int threads = 32 * sim->num_agents * epb;
        const dim3 tgrid((sim->num_envs + epb - 1) / epb);
        // register budget of the 128-thread flavour (A <= 4): 4 blocks/SM = 128 registers (no spills), 5 = 96, 8 = 64
        ts.kernel = TailShape::TAIL; ts.epb = epb; ts.threads = threads; ts.grid = (int)tgrid.x;
        ts.lb_threads = threads <= 128 ? 128 : 1024;
        ts.lb_minb = threads > 128 ? 1 : (g_tail_minb == 4 || g_tail_minb == 5) ? g_tail_minb : 8;
        if (ts.lb_threads == 128 && ts.lb_minb == 4)
            launch_k(k_tail<128, 4>, tgrid, dim3(threads), 0, st, pdl, *sim, bv, (int)tail->env_level, tail->ar, max_scan, epb);
        else if (ts.lb_threads == 128 && ts.lb_minb == 5)
            launch_k(k_tail<128, 5>, tgrid, dim3(threads), 0, st, pdl, *sim, bv, (int)tail->env_level, tail->ar, max_scan, epb);
        else if (ts.lb_threads == 128)
            launch_k(k_tail<128, 8>, tgrid, dim3(threads), 0, st, pdl, *sim, bv, (int)tail->env_level, tail->ar, max_scan, epb);
        else
            launch_k(k_tail<1024, 1>, tgrid, dim3(threads), 0, st, pdl, *sim, bv, (int)tail->env_level, tail->ar, max_scan, epb);
        LAUNCH_CHECK("k_tail");
    } else {
        ts.kernel = TailShape::FINALIZE; ts.epb = 0; ts.threads = 128; ts.grid = (NA * 32 + 127) / 128; ts.separate = fused;
        launch_k(k_finalize, dim3(ts.grid), dim3(128), 0, st, pdl, *sim, bv, max_scan);
        LAUNCH_CHECK("k_finalize");
        if (fused) {     // more than 32 agents per env: same semantics with separate launches
            if (tail->env_level) { k_env_post_step<<<(sim->num_envs + 127) / 128, 128, 0, st>>>(*sim); LAUNCH_CHECK("k_env_post_step"); }
            if (tail->ar.start_poses) { k_autoreset<<<(sim->num_envs + 127) / 128, 128, 0, st>>>(*sim, tail->ar); LAUNCH_CHECK("k_autoreset"); }
        }
    }
    return F110_OK;
}

// f110_debug_last_launch: `key=value` text of what the tick launched, from the plan and the tail's shape.  Tests match on it.
static void write_launch_record(const MarchPlan &p, const MapGeom &geom, const f110_map *map, const TailShape &ts) {
    char march[192] = "", tail[96] = "";
    const int N = p.noise ? 1 : 0, C = p.count ? 1 : 0, CELLS = p.cell_units ? 1 : 0;
    switch (p.family) {
    case MarchFamily::LITERAL:
        snprintf(march, sizeof(march), "march=literal FAST=%d NOISE=%d COUNT=%d PT=%d grid=%u", map->fast_path ? 1 : 0, N, C, p.pt, p.grid.x);
        break;
    case MarchFamily::BLOCK_PER_TILE:
        snprintf(march, sizeof(march), "march=block-per-tile CELLS=%d CODED=%d NOISE=%d COUNT=%d MINB=%d grid=%ux%u", CELLS,
                 p.coded ? 1 : 0, N, C, p.minb, p.grid.x, p.grid.y);
        break;
    case MarchFamily::PERSISTENT:
        snprintf(march, sizeof(march), "march=persistent CELLS=%d CODED=%d NOISE=%d COUNT=%d SUB=%d PT=%d grid=%u", CELLS,
                 p.coded ? 1 : 0, N, C, p.sub, p.pt, p.grid.x);
        break;
    case MarchFamily::LEAN:
    case MarchFamily::LEAN_BRICK:
        if (p.cluster) { snprintf(march, sizeof(march), "march=lean-cluster variant=%d", p.variant); break; }
        snprintf(march, sizeof(march),
                 "march=lean TABLE=%d CELLS=%d LAYERED=%d DYN=%d IPT=%d RING=%d PT=%d MINB=%d NOISE=%d COUNT=%d grid=%u%s", p.coded ? 1 : 0,
                 CELLS, p.layered ? 1 : 0, p.dyn ? 1 : 0, p.ipt, p.ring, p.pt, p.minb, N, C, p.grid.x,
                 p.family == MarchFamily::LEAN_BRICK ? " layout=brick4x4" : "");
        break;
    case MarchFamily::LEAN_HET:
    case MarchFamily::LEAN_HET_RES:
        snprintf(march, sizeof(march), "march=lean-het HET=1 layers=%d%s CELLS=%d DYN=0 IPT=1 PT=%d MINB=%d NOISE=%d COUNT=%d grid=%u",
                 map->num_layers, p.family == MarchFamily::LEAN_HET_RES ? " RES=1" : "", CELLS, p.pt, p.minb, N, C, p.grid.x);
        break;
    case MarchFamily::LEAN_ROT:
        snprintf(march, sizeof(march), "march=lean-rot ROT=1 layers=%d%s CELLS=0 DYN=0 IPT=1 PT=%d MINB=%d NOISE=%d COUNT=%d grid=%u",
                 map->num_layers, geom.het ? " HET=1 RES=1" : "", p.pt, p.minb, N, C, p.grid.x);
        break;
    case MarchFamily::TILE:
        snprintf(march, sizeof(march), "march=tile TILE=%d NSLOT=%d NOISE=%d COUNT=%d PT=%d MINB=%d grid=%u", p.tile_sz,
                 p.tile_sz == 160 ? 2 : 3, N, C, p.pt, p.minb, p.grid.x);
        break;
    }
    switch (ts.kernel) {
    case TailShape::TAIL2:
        snprintf(tail, sizeof(tail), "tail=k_tail2 epb=%d threads=%d tail_grid=%d smem=%zu", ts.epb, ts.threads, ts.grid, ts.smem);
        break;
    case TailShape::TAIL:
        snprintf(tail, sizeof(tail), "tail=k_tail<%d,%d> epb=%d threads=%d tail_grid=%d", ts.lb_threads, ts.lb_minb, ts.epb, ts.threads, ts.grid);
        break;
    case TailShape::FINALIZE:
        snprintf(tail, sizeof(tail), "tail=k_finalize%s epb=0 threads=128 tail_grid=%d", ts.separate ? "+separate" : "", ts.grid);
        break;
    case TailShape::NOSCAN:
        snprintf(tail, sizeof(tail), "tail=k_lidar_cast+k_tail_noscan cast_grid=%d epb=%d threads=%d tail_grid=%d", ts.cast_grid,
                 ts.epb, ts.threads, ts.grid);
        break;
    }
    snprintf(g_launch_rec, sizeof(g_launch_rec), "%s%s%s static_runs=%u per_warp=%u %s", march, geom.het ? "" : " HET=0",
             p.rot && p.lean ? "" : " ROT=0", p.mq.static_runs, p.per_warp, tail);
}

// ------------------------------------------------------------------------------------ obstacles (csrc/obstacles.cuh)
struct ObstPlan {
    ObstK k;
    ObstDraw d;
};
// f110_obstacles -> the kernels' views, every rule of the header checked before anything is enqueued.  num_layers: the map's
// layer count that per-layer candidate tables must match, or -1 when the call has no map.
static int plan_obstacles(const f110_sim *sim, const f110_obstacles *o, int num_layers, ObstPlan *p) {
    if (o->per_env < 1 || o->per_env > F110_MAX_OBSTACLES || !o->boxes || !o->active) return F110_ERR_INVALID;
    if (o->count_min < 0 || o->count_min > o->count_max || o->count_max > o->per_env) return F110_ERR_INVALID;
    if (!(o->clearance >= 0.0) || !isfinite(o->clearance)) return F110_ERR_INVALID;
    p->k.boxes = o->boxes; p->k.active = o->active; p->k.hit = o->hit; p->k.K = o->per_env; p->k.lidar = F110_LIDAR_ALL;
    ObstDraw &d = p->d;
    memset(&d, 0, sizeof(d));
    d.boxes = o->boxes; d.active = o->active; d.cand = o->candidates; d.K = o->per_env;
    d.num_cand = o->num_candidates; d.num_tables = 0;
    d.count_min = o->count_min; d.count_max = o->count_max; d.clearance = o->clearance; d.seed = o->seed;
    if (!o->candidates) return F110_OK;
    if (o->num_candidates < 1) return F110_ERR_INVALID;
    if (!o->cand_offsets) return F110_OK;
    const int L = o->num_cand_tables;
    if (L < 1 || L > F110_MAX_START_TABLES || !sim->env_layer || o->cand_offsets[0] != 0 || o->cand_offsets[L] != o->num_candidates)
        return F110_ERR_INVALID;
    if (num_layers >= 0 && L != std::max(num_layers, 1)) return F110_ERR_INVALID;
    for (int l = 0; l <= L; l++) {
        if (l < L && o->cand_offsets[l + 1] <= o->cand_offsets[l]) return F110_ERR_INVALID;
        d.off[l] = o->cand_offsets[l];
    }
    d.num_tables = L;
    return F110_OK;
}
// measurement aid (f110_debug_set_obst_events): events recorded before k_obstacles, after it, and after k_env_tail_obst
static cudaEvent_t g_obst_ev[3] = {nullptr, nullptr, nullptr};
// after the tail of a tick that ran without its env-level part: k_obstacles, then (a tick with lap logic or auto-reset)
// k_env_tail_obst.  tail NULL: f110_step.  rd: the repeat bookkeeping of an intermediate tick of f110_tick_repeat, or NULL.
// lidar: the mask of a tick with a lidar mask on its short path (only those slots' scans are clipped), else F110_LIDAR_ALL
static int launch_obst_tail(const f110_sim *sim, const BeamView &bv, const ObstPlan &ob, const TailOpts *tail, bool scan,
                            const RepeatDone *rd, double max_scan, cudaStream_t st, uint32_t lidar = F110_LIDAR_ALL) {
    const int NA = sim->num_envs * sim->num_agents;
    const unsigned grid = (unsigned)(((long long)NA * 32 + 127) / 128);
    if (g_obst_ev[0]) CUDA_TRY(cudaEventRecord(g_obst_ev[0], st));
    if (scan && lidar != F110_LIDAR_ALL) {
        ObstK k = ob.k;
        k.lidar = lidar;
        k_obstacles<true, true><<<grid, 128, 0, st>>>(*sim, bv, k, max_scan);
    } else if (scan) k_obstacles<true><<<grid, 128, 0, st>>>(*sim, bv, ob.k, max_scan);
    else k_obstacles<false><<<grid, 128, 0, st>>>(*sim, bv, ob.k, max_scan);
    LAUNCH_CHECK("k_obstacles");
    if (g_obst_ev[1]) CUDA_TRY(cudaEventRecord(g_obst_ev[1], st));
    if (tail && (tail->env_level || tail->ar.start_poses)) {
        RepeatDone r;
        r.done_any = rd ? rd->done_any : nullptr; r.done_tick = rd ? rd->done_tick : nullptr; r.tick = rd ? rd->tick : 0;
        k_env_tail_obst<<<(sim->num_envs + 127) / 128, 128, 0, st>>>(*sim, (int)tail->env_level, tail->ar, r, ob.d);
        LAUNCH_CHECK("k_env_tail_obst");
    }
    if (g_obst_ev[2]) CUDA_TRY(cudaEventRecord(g_obst_ev[2], st));
    return F110_OK;
}

// ------------------------------------------------------------------------------------ the plan and the launches of a tick
// ---- ticks whose scans nobody reads, in whole (the intermediate ticks of f110_tick_repeat) or in part (the sensorless agents of
// a tick with a lidar mask): march_ttc.cuh.  Decided here from what the host can observe, never by an option.  The short path
// needs: no scan noise (the bound does not hold for a Gaussian, and the Philox stream must stay the plain run's); a lean march
// family, which brings the per-agent record, the doubled LUT and `dt_min_positive > eps`; a known max side distance below
// max_range (otherwise every moving agent is listed); and at most 32 agents per env (the block-owns-envs tail).
// The map and beam part of those conditions is also what f110_predict needs: the per-agent record's arithmetic and k_march_ttc's.
static bool ttc_tables_ok(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const MarchPlan &m) {
    const bool lean_family = m.family == MarchFamily::LEAN || m.family == MarchFamily::LEAN_BRICK || m.family == MarchFamily::LEAN_HET ||
                             m.family == MarchFamily::LEAN_HET_RES || m.family == MarchFamily::LEAN_ROT;
    return m.lean && lean_family && sim->march_rec && map->sincos2 && map->dt_min_positive > map->eps && beams->side_max > 0.0 &&
           beams->side_max < map->max_range;
}
static bool ttc_path_ok(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const MarchPlan &m) {
    return sim->noise_std == 0.0 && ttc_tables_ok(sim, map, beams, m) && sim->num_agents <= 32;
}
// The units (F110_SCAN_UNITS_*) k_march_ttc and k_restart_march run in for a march plan.  They follow the family, never the
// queue length, so a tick's plan and its lidar-mask plan agree.
static int scan_units(const MarchPlan &m) {
    return m.rot ? F110_SCAN_UNITS_ROT : m.cell_units ? F110_SCAN_UNITS_CELLS : F110_SCAN_UNITS_METRES;
}
// The UNITS build of a kernel: f(units) with the run-time F110_SCAN_UNITS_* value as a std::integral_constant.
template <typename F>
static void dispatch_units(int units, F &&f) {
    if (units == F110_SCAN_UNITS_ROT) f(std::integral_constant<int, F110_SCAN_UNITS_ROT>());
    else if (units == F110_SCAN_UNITS_CELLS) f(std::integral_constant<int, F110_SCAN_UNITS_CELLS>());
    else f(std::integral_constant<int, F110_SCAN_UNITS_METRES>());
}
static void launch_march_ttc(const TtcK &q, int units, bool count, unsigned grid, cudaStream_t st) {
    dispatch_units(units, [&](auto u) {
        if (count) k_march_ttc<decltype(u)::value, true><<<grid, F110_TTC_THREADS, 0, st>>>(q);
        else k_march_ttc<decltype(u)::value, false><<<grid, F110_TTC_THREADS, 0, st>>>(q);
    });
}
static void launch_restart_march(const TtcK &q, const RestartK &r, int units, bool count, unsigned grid, cudaStream_t st) {
    dispatch_units(units, [&](auto u) {
        if (count) k_restart_march<decltype(u)::value, true><<<grid, F110_TTC_THREADS, 0, st>>>(q, r);
        else k_restart_march<decltype(u)::value, false><<<grid, F110_TTC_THREADS, 0, st>>>(q, r);
    });
}
// The fixed grid of a grid-stride kernel of F110_TTC_THREADS threads: resident blocks per SM x SMs, the occupancy of each
// kernel instance queried once.
template <auto KERNEL>
static int resident_grid(unsigned *grid) {
    static int per_sm = 0;
    if (per_sm <= 0) {
        CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, KERNEL, F110_TTC_THREADS, 0));
        if (per_sm <= 0) return F110_ERR_INVALID;
    }
    *grid = (unsigned)per_sm * (unsigned)num_sms();
    return F110_OK;
}
// the grid of k_march_ttc, or with restart of k_restart_march
static int ttc_grid(bool restart, int units, bool count, unsigned *grid) {
    int rc = F110_OK;
    dispatch_units(units, [&](auto u) {
        constexpr int U = decltype(u)::value;
        if (restart) rc = count ? resident_grid<k_restart_march<U, true>>(grid) : resident_grid<k_restart_march<U, false>>(grid);
        else rc = count ? resident_grid<k_march_ttc<U, true>>(grid) : resident_grid<k_march_ttc<U, false>>(grid);
    });
    return rc;
}
// k_march_ttc's units for the tick's march, and its grid
static int plan_ttc(const MarchPlan &m, int *units, unsigned *grid) {
    *units = scan_units(m);
    return ttc_grid(false, *units, m.count, grid);
}

struct TickPlan {
    MapGeom geom;
    MarchPlan march;
    const ObstPlan *obst;    // NULL: no obstacles (the tail runs as before)
    // a lidar mask (f110_lidar): on the short path `lidar` is set, the march plan queues the `lidar_slots` slots that have a
    // lidar, and k_march_ttc runs with ttc_units / ttc_grid; lidar_full: a mask was given and is ignored (the full path)
    const f110_lidar *lidar;
    bool lidar_full;
    unsigned lidar_slots;
    int ttc_units;
    unsigned ttc_grid;
};
// a lidar mask the call may take (before anything is enqueued, on either path); sim already checked
static int check_lidar(const f110_sim *sim, const f110_lidar *lidar) {
    if (!lidar || lidar->mask == F110_LIDAR_ALL) return F110_OK;
    if (sim->num_agents > 32) return F110_ERR_INVALID;
    if (sim->num_agents < 32 && (lidar->mask >> sim->num_agents) != 0u) return F110_ERR_INVALID;
    if (!lidar->list || !lidar->list_count) return F110_ERR_INVALID;
    return F110_OK;
}
static int plan_tick(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                     const double *actions, TickPlan *tp, const f110_lidar *lidar = nullptr) {
    int rc;
    tp->obst = nullptr;
    tp->lidar = nullptr; tp->lidar_full = false; tp->lidar_slots = 0u; tp->ttc_units = 0; tp->ttc_grid = 0u;
    if ((rc = check_sim(sim)) || (rc = check_lidar(sim, lidar)) || (rc = check_map(map)) || (rc = check_beams(beams))) return rc;
    if (!actions) return F110_ERR_INVALID;
    if (sim->lookup_counter && sim->noise_std > 0.0) return F110_ERR_INVALID;   // counting runs are noise-free by construction
    if ((long long)sim->num_envs * sim->num_agents > 0x7fffffffll) return F110_ERR_INVALID;
    if ((rc = classify_map(map, &tp->geom))) return rc;
    if ((rc = plan_march(sim, map, tables, beams, tp->geom, rm_variant(), &tp->march))) return rc;
    if (!lidar || lidar->mask == F110_LIDAR_ALL) return F110_OK;
    if (!ttc_path_ok(sim, map, beams, tp->march)) { tp->lidar_full = true; return F110_OK; }
    tp->lidar = lidar;
    tp->lidar_slots = (unsigned)__builtin_popcount(lidar->mask);
    // the same family and kernel shape rules on the shorter queue (the family never depends on the queue length)
    if ((rc = plan_march(sim, map, tables, beams, tp->geom, rm_variant(), &tp->march, (long long)sim->num_envs * tp->lidar_slots)))
        return rc;
    return plan_ttc(tp->march, &tp->ttc_units, &tp->ttc_grid);
}
static int launch_lidar_tick(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                             const double *actions, TickPlan &tp, cudaStream_t st, const TailOpts *tail);
static void append_launch_record(const char *fmt, ...) {
    const size_t n = strlen(g_launch_rec);
    va_list va;
    va_start(va, fmt);
    vsnprintf(g_launch_rec + n, sizeof(g_launch_rec) - n, fmt, va);
    va_end(va);
}
static int launch_tick(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                       const double *actions, TickPlan &tp, cudaStream_t st, cudaEvent_t *ev /* NULL or [4] */, const TailOpts *tail) {
    int rc;
    MarchPlan &plan = tp.march;
    const bool pdl = (ev == nullptr);         // PDL only when no events are recorded between the kernels
    if (tp.lidar) return launch_lidar_tick(sim, map, tables, beams, actions, tp, st, tail);

    if (ev) CUDA_TRY(cudaEventRecord(ev[0], st));
    k_dynamics<<<plan.dyn_blocks + plan.order_blocks, 128, 0, st>>>(*sim, actions, beams->fov, (double)map->theta_dis, plan.dyn_blocks,
                                                                    fill_first_lookup(sim, map, beams, tp.geom, plan));
    LAUNCH_CHECK("k_dynamics");
    if (ev) CUDA_TRY(cudaEventRecord(ev[1], st));
    if ((rc = launch_march_plan(plan, sim, map, tables, beams, tp.geom, pdl, st))) return rc;
    if (ev) CUDA_TRY(cudaEventRecord(ev[2], st));
    TailShape ts = {};
    const BeamView bv = make_view(beams);
    // with obstacles the tail runs without its env-level part: contact with a box must be known before `done` and the auto-reset
    if ((rc = launch_tail(sim, map, bv, tp.obst ? nullptr : tail, pdl && plan.lean, st, &ts))) return rc;
    if (tp.obst && (rc = launch_obst_tail(sim, bv, *tp.obst, tail, true, nullptr, max_scan_range(sim, map), st))) return rc;
    write_launch_record(plan, tp.geom, map, ts);
    if (tp.obst) append_launch_record(" obst=%d", tp.obst->k.K);
    if (tp.lidar_full) append_launch_record(" lidar=full");
    if (ev) CUDA_TRY(cudaEventRecord(ev[3], st));
    return F110_OK;
}
// ---- f110_tick_repeat: `repeat` ticks under one action; the ticks whose scans nobody reads march only for the iTTC flag
// The plan of the call: the plain tick's plan, and whether ticks 0 .. repeat - 2 take the short path (ttc_path_ok).
// Everything else runs `repeat` plain ticks.
struct RepeatPlan {
    TickPlan tick;
    bool ttc;                // ticks 0 .. repeat - 2: k_dynamics, k_ttc_select, k_march_ttc, k_tail_noscan
    int units;               // F110_SCAN_UNITS_* of k_march_ttc
    unsigned grid;           // its fixed grid: resident blocks per SM x SMs
};
static int plan_repeat(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                       const double *actions, int32_t repeat, RepeatPlan *rp) {
    int rc;
    if ((rc = plan_tick(sim, map, tables, beams, actions, &rp->tick))) return rc;
    const MarchPlan &m = rp->tick.march;
    rp->ttc = repeat > 1 && ttc_path_ok(sim, map, beams, m);
    rp->units = scan_units(m);
    rp->grid = 0u;
    if (!rp->ttc) return F110_OK;
    return plan_ttc(m, &rp->units, &rp->grid);
}
// the tail options and plans of a held-action call (f110_tick_repeat_ticks_lidar, f110_tick_repeat_episodes_ticks)
struct RepeatCall {
    TailOpts t;
    RepeatPlan rp;
    TickPlan last;           // with a lidar mask: the last tick of the call, the plain tick's plan with the mask
    ObstPlan ob;
    bool masked;
    TickPlan &last_tick() { return masked ? last : rp.tick; }
};

// list / count: the agents k_ttc_select listed
static TtcK fill_ttc_k(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const TickPlan &tp, const uint32_t *list,
                       const uint32_t *count) {
    const MarchPlan &m = tp.march;
    const bool het = tp.geom.het;
    TtcK q;
    q.table = m.cell_units ? map->dt_cells_pad : map->dt;
    q.dt = map->dt;
    q.sincos2 = reinterpret_cast<const double2 *>(map->sincos2);
    q.cos_side = reinterpret_cast<const double2 *>(beams->cos_side);
    q.rec = reinterpret_cast<const double2 *>(sim->march_rec);
    q.list = list; q.count = count;
    q.wall_flag = sim->wall_flag; q.lookup_counter = sim->lookup_counter;
    q.layer_geom = het ? map->layer_geom : nullptr; q.layer_res = het ? map->layer_res : nullptr;
    q.layer_rot = het ? map->layer_rot : nullptr; q.env_layer = het ? sim->env_layer : nullptr;
    q.orig = make_double2(map->orig_x, map->orig_y);
    q.ext = make_double2(map->width * map->resolution, map->height * map->resolution);
    q.res = make_double2(map->resolution, 1.0 / map->resolution);
    q.rot = make_double2(map->orig_c, map->orig_s);
    q.tmax = m.cell_units ? map->max_range * (1.0 / map->resolution) : map->max_range;
    q.max_range = map->max_range; q.eps = map->eps;
    q.ttc_thresh = sim->ttc_thresh; q.ttc_margin = sim->ttc_thresh * 1.000001;
    q.inc = beams->theta_index_increment; q.theta_dis_f = (double)map->theta_dis;
    lut_fixed_point(beams, &q.inc_fx, &q.guard32);
    q.layer_stride = (unsigned long long)map->width * (unsigned long long)map->height;
    q.layer_stride_lean = m.cell_units ? (unsigned long long)(map->width + 1) * (unsigned long long)(map->height + 1) : q.layer_stride;
    q.width = (unsigned)map->width; q.height = (unsigned)map->height;
    q.last = (unsigned)map->width * (unsigned)map->height - 1u;
    q.ipa = (unsigned)((beams->num_beams + 31) / 32);
    q.num_agents = (unsigned)sim->num_agents;
    q.B = beams->num_beams;
    return q;
}

// k_ttc_select: the agents a wall could stop into list / count, except those of the slots in `skip`
static int launch_ttc_select(const f110_sim *sim, const f110_map *map, const MarchPlan &m, uint32_t *list, uint32_t *count,
                             unsigned long long *marched, uint32_t skip, cudaStream_t st) {
    const int NA = sim->num_envs * sim->num_agents;
    TtcSelectK sel;
    sel.rec = reinterpret_cast<const double2 *>(sim->march_rec); sel.list = list; sel.count = count;
    sel.marched = marched; sel.d0_scale = m.cell_units ? map->resolution : 1.0; sel.max_range = map->max_range;
    sel.agents = (unsigned)NA; sel.skip = skip; sel.num_agents = (unsigned)sim->num_agents;
    k_ttc_select<<<(NA + F110_TTC_SELECT_THREADS - 1) / F110_TTC_SELECT_THREADS, F110_TTC_SELECT_THREADS, 0, st>>>(sel);
    LAUNCH_CHECK("k_ttc_select");
    return F110_OK;
}

// one intermediate tick of the short path
static int launch_ttc_tick(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const double *actions,
                           const RepeatPlan &rp, const f110_repeat *rep, int tick, const TailOpts &tail, cudaStream_t st) {
    int rc;
    const MarchPlan &m = rp.tick.march;
    // k_dynamics without its queue-building blocks: the queue is built once, by the last tick of the call
    k_dynamics<<<m.dyn_blocks, 128, 0, st>>>(*sim, actions, beams->fov, (double)map->theta_dis, m.dyn_blocks,
                                             fill_first_lookup(sim, map, beams, rp.tick.geom, m));
    LAUNCH_CHECK("k_dynamics");
    if ((rc = launch_ttc_select(sim, map, m, rep->list, rep->list_count + tick, rep->marched_agents, 0u, st))) return rc;
    launch_march_ttc(fill_ttc_k(sim, map, beams, rp.tick, rep->list, rep->list_count + tick), rp.units, m.count, rp.grid, st);
    LAUNCH_CHECK("k_march_ttc");
    const int epb = std::max(1, F110_TAIL_NOSCAN_THREADS / sim->num_agents);
    RepeatDone rd;
    rd.done_any = rep->done_any; rd.done_tick = rep->done_tick; rd.tick = tick;
    if (rp.tick.obst) {       // the agent part here, then box contact, then the env level with the respawn
        AutoResetArgs no_ar = tail.ar;
        no_ar.start_poses = nullptr;
        k_tail_noscan<<<(sim->num_envs + epb - 1) / epb, F110_TAIL_NOSCAN_THREADS, 0, st>>>(*sim, 0, no_ar, epb, rd);
        LAUNCH_CHECK("k_tail_noscan");
        return launch_obst_tail(sim, make_view(beams), *rp.tick.obst, &tail, false, &rd, max_scan_range(sim, map), st);
    }
    k_tail_noscan<<<(sim->num_envs + epb - 1) / epb, F110_TAIL_NOSCAN_THREADS, 0, st>>>(*sim, (int)tail.env_level, tail.ar, epb, rd);
    LAUNCH_CHECK("k_tail_noscan");
    return F110_OK;
}

// A tick with a lidar mask on its short path (TickPlan.lidar): S = lidar_slots slots have a lidar.
//   k_dynamics         the dynamics of every agent, without its queue-building blocks
//   k_lidar_order      the march queue of the S slots only (skipped when S = 0)
//   the planned march  unchanged kernels on that queue: scans and iTTC flags of the agents that have a lidar (skipped when S = 0)
//   k_ttc_select       the sensorless agents a wall could stop, into f110_lidar.list
//   k_march_ttc        those agents, for the iTTC flag alone
//   k_lidar_cast       the opponent ray-cast of the egos that have a lidar, and the queue counters (skipped when S = 0)
//   k_tail_noscan      agent duties, env level and auto-reset -- after the ray-cast, whose yaw comes from wall_flag
// With obstacles, k_tail_noscan runs without its env level, then k_obstacles<true, true> (contact for every agent, the scan
// clip for the agents that have a lidar) and k_env_tail_obst.
static int launch_lidar_tick(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                             const double *actions, TickPlan &tp, cudaStream_t st, const TailOpts *tail) {
    int rc;
    MarchPlan &plan = tp.march;
    const f110_lidar &ld = *tp.lidar;
    const unsigned S = tp.lidar_slots;
    const LidarOrder lo = {ld.mask, S};
    k_dynamics<<<plan.dyn_blocks, 128, 0, st>>>(*sim, actions, beams->fov, (double)map->theta_dis, plan.dyn_blocks,
                                                fill_first_lookup(sim, map, beams, tp.geom, plan));
    LAUNCH_CHECK("k_dynamics");
    if (S) {
        k_lidar_order<<<plan.order_blocks, 128, 0, st>>>(*sim, lo);
        LAUNCH_CHECK("k_lidar_order");
    }
    if (S && (rc = launch_march_plan(plan, sim, map, tables, beams, tp.geom, false, st))) return rc;
    CUDA_TRY(cudaMemsetAsync(ld.list_count, 0, sizeof(uint32_t), st));
    if ((rc = launch_ttc_select(sim, map, plan, ld.list, ld.list_count, ld.listed, ld.mask, st))) return rc;
    launch_march_ttc(fill_ttc_k(sim, map, beams, tp, ld.list, ld.list_count), tp.ttc_units, plan.count, tp.ttc_grid, st);
    LAUNCH_CHECK("k_march_ttc");
    const BeamView bv = make_view(beams);
    const double max_scan = max_scan_range(sim, map);
    unsigned cast_grid = 0u;
    if (S) {
        cast_grid = (unsigned)(((unsigned long long)sim->num_envs * S + F110_LIDAR_CAST_WARPS - 1) / F110_LIDAR_CAST_WARPS);
        k_lidar_cast<<<cast_grid, 32 * F110_LIDAR_CAST_WARPS, 0, st>>>(*sim, bv, lo, max_scan);
        LAUNCH_CHECK("k_lidar_cast");
    }
    const int epb = std::max(1, F110_TAIL_NOSCAN_THREADS / sim->num_agents);
    const unsigned tgrid = (unsigned)((sim->num_envs + epb - 1) / epb);
    RepeatDone rd;
    rd.done_any = nullptr; rd.done_tick = nullptr; rd.tick = 0;
    AutoResetArgs ar;
    memset(&ar, 0, sizeof(ar));
    if (tail) ar = tail->ar;
    const int env_level = tail ? (int)tail->env_level : 0;
    if (tp.obst) {
        AutoResetArgs no_ar = ar;
        no_ar.start_poses = nullptr;
        k_tail_noscan<<<tgrid, F110_TAIL_NOSCAN_THREADS, 0, st>>>(*sim, 0, no_ar, epb, rd);
        LAUNCH_CHECK("k_tail_noscan");
        if ((rc = launch_obst_tail(sim, bv, *tp.obst, tail, true, nullptr, max_scan, st, ld.mask))) return rc;
    } else {
        k_tail_noscan<<<tgrid, F110_TAIL_NOSCAN_THREADS, 0, st>>>(*sim, env_level, ar, epb, rd);
        LAUNCH_CHECK("k_tail_noscan");
    }
    // the record: the march (when one ran), then the tail kernels
    g_launch_rec[0] = '\0';
    if (S) {
        TailShape ts = {};
        ts.kernel = TailShape::NOSCAN; ts.epb = epb; ts.threads = F110_TAIL_NOSCAN_THREADS; ts.grid = (int)tgrid;
        ts.cast_grid = (int)cast_grid;
        write_launch_record(plan, tp.geom, map, ts);
    } else {
        snprintf(g_launch_rec, sizeof(g_launch_rec), "march=none tail=k_tail_noscan epb=%d threads=%d tail_grid=%d", epb,
                 F110_TAIL_NOSCAN_THREADS, (int)tgrid);
    }
    append_launch_record(" ttc=%s grid=%u", tp.ttc_units == F110_SCAN_UNITS_ROT ? "rot" : tp.ttc_units == F110_SCAN_UNITS_CELLS ?
                         "cells" : "metres", tp.ttc_grid);
    if (tp.obst) append_launch_record(" obst=%d", tp.obst->k.K);
    append_launch_record(" lidar=%u/%d", S, sim->num_agents);
    return F110_OK;
}

// ---- episodes (csrc/episodes.cuh): the plain tick, then the end decision and the restart of the ended envs
// The restart march reuses k_march_ttc's beam arithmetic, which covers the lean march families only.
static bool episode_march_ok(const MarchPlan &m) {
    return m.lean && (m.family == MarchFamily::LEAN || m.family == MarchFamily::LEAN_BRICK || m.family == MarchFamily::LEAN_HET ||
                      m.family == MarchFamily::LEAN_HET_RES || m.family == MarchFamily::LEAN_ROT);
}
// The scans of the envs on r.list / r.count for the slots in r.lidar, from the plan tp, on `grid` blocks of k_restart_march.
// restart, the kernel that listed the ended envs (k_episode_end / k_episode_restart): their restart on view = *sim --
//   k_episode_dyn, k_restart_march, k_episode_cast, k_episode_tail, k_episode_obstacles -- and the `episodes restart=` record.
// restart NULL: the final-scan pass on a snapshot `view` whose march records are `rec` -- k_restart_march without the lookup
//   count, k_episode_cast, and k_episode_obstacles without box contact (ObstK.hit NULL); the caller writes its record.
static int launch_restart(const char *restart, const f110_sim &view, const double *rec, const f110_map *map,
                          const f110_beams *beams, const TickPlan &tp, const RestartK &r, unsigned grid, cudaStream_t st) {
    const int N = view.num_envs, A = view.num_agents, NA = N * A;
    if (restart) {
        k_episode_dyn<<<(NA + 127) / 128, 128, 0, st>>>(view, beams->fov, (double)map->theta_dis,
                                                        fill_first_lookup(&view, map, beams, tp.geom, tp.march), r.list, r.count);
        LAUNCH_CHECK("k_episode_dyn");
    }
    TtcK q = fill_ttc_k(&view, map, beams, tp, r.list, r.count);
    q.rec = reinterpret_cast<const double2 *>(rec);
    launch_restart_march(q, r, scan_units(tp.march), restart && tp.march.count, grid, st);
    LAUNCH_CHECK("k_restart_march");
    const BeamView bv = make_view(beams);
    const double max_scan = max_scan_range(&view, map);
    const unsigned slots = (unsigned)__builtin_popcount(r.lidar);
    if (A > 1 && slots) {
        const LidarOrder lo = {r.lidar, slots};
        k_episode_cast<<<(unsigned)(((unsigned long long)N * slots + F110_LIDAR_CAST_WARPS - 1) / F110_LIDAR_CAST_WARPS),
                         32 * F110_LIDAR_CAST_WARPS, 0, st>>>(view, bv, lo, r.list, r.count, max_scan);
        LAUNCH_CHECK("k_episode_cast");
    }
    if (restart) {
        k_episode_tail<<<(N + 127) / 128, 128, 0, st>>>(view, r.list, r.count);
        LAUNCH_CHECK("k_episode_tail");
    }
    if (tp.obst) {
        ObstK o = tp.obst->k;
        o.lidar = r.lidar;
        if (!restart) o.hit = nullptr;
        k_episode_obstacles<<<(unsigned)(((long long)NA * 32 + 127) / 128), 128, 0, st>>>(view, bv, o, max_scan, r.list, r.count);
        LAUNCH_CHECK("k_episode_obstacles");
    }
    if (restart)
        append_launch_record(" episodes restart=%s+k_episode_dyn+k_restart_march%s+k_episode_tail%s restart_grid=%u", restart,
                             (A > 1 && slots) ? "+k_episode_cast" : "", tp.obst ? "+k_episode_obstacles" : "", grid);
    return F110_OK;
}
static EpisodeK episode_k(const f110_episodes *ep) {
    EpisodeK k;
    k.ticks = ep->ticks; k.length = ep->length; k.terminated = ep->terminated; k.truncated = ep->truncated;
    k.final_state = ep->final_state; k.final_collisions = ep->final_collisions; k.final_lap_times = ep->final_lap_times;
    k.final_lap_counts = ep->final_lap_counts; k.final_collision_idx = ep->final_collision_idx;
    k.list = ep->list; k.count = ep->list_count; k.track_seg = ep->track_seg; k.max_ticks = ep->max_ticks;
    return k;
}
static int check_episodes(const f110_sim *sim, const f110_episodes *ep, const double *start_poses) {
    if (!ep || !start_poses) return F110_ERR_INVALID;
    if (!ep->ticks || !ep->terminated || !ep->truncated || !ep->length || !ep->final_state || !ep->final_scans ||
        !ep->final_collisions || !ep->final_collision_idx || !ep->final_lap_times || !ep->final_lap_counts || !ep->list ||
        !ep->list_count)
        return F110_ERR_INVALID;
    if (ep->max_ticks < 0 || sim->num_agents > 32) return F110_ERR_INVALID;
    return F110_OK;
}

}  // namespace f110

using namespace f110;

// ================================================================================== C ABI
extern "C" {

int f110_abi_version(void) { return F110_ABI_VERSION; }

/* debug aid (not in the public header): device buffer [blocks][4] u64 that the march kernels fill with
 * (smid, start ns, end ns, max steps of warp 0) per block; NULL switches it off. */
void f110_debug_set_trace(unsigned long long *buf) { g_trace = buf; }
/* measurement aid (not in the public header): select the march kernel variant at run time (tools/ab_march.py) */
void f110_debug_set_variant(int variant) {
    g_no_brick = variant == 90;
    g_variant = (variant < 0 || variant == 90) ? 0 : variant;
}
void f110_debug_set_dyn(int static_pct, int ahead) {
    g_dyn_pct = static_pct < 0 ? 0 : (static_pct > 100 ? 100 : static_pct);
    g_dyn_ahead = ahead < 1 ? 1 : (ahead > 8 ? 8 : ahead);
}
/* log2(queue entries per ticket) for runs of very heavy / heavy / light entries and for the dynamic tail of the default launch
 * (dyn_tail < 0: by the class the tail starts in) */
void f110_debug_set_ipt(int very_heavy, int heavy, int light, int dyn_tail) {
    const int v[4] = {very_heavy, heavy, light, dyn_tail};
    for (int z = 0; z < 4; z++) g_ipt[z] = (v[z] < 0 || v[z] > 3) ? (z == 3 ? 255 : -1) : v[z];
}
void f110_debug_set_pdl(int on) { g_pdl = on ? 1 : 0; }
void f110_debug_set_tail2(int threads, int agents) {
    g_tail2_threads = (threads >= 32 && threads <= F110_TAIL2_THREADS) ? (threads / 32) * 32 : F110_TAIL2_THREADS;
    g_tail2_forced = (agents > 64 || agents < 0) ? 1 : 0;
    if (agents < 0) agents = -agents;
    g_tail2_agents = (agents >= 4 && agents <= 128) ? agents : 64;
}
void f110_debug_set_tail(int minb) {      // -1: k_tail always; -2 or a register budget: k_tail2 for 2 <= A <= 4 (the default)
    if (minb == -1) { g_tail2 = 0; g_tail_minb = 8; }
    else if (minb == -2) { g_tail2 = 1; g_tail_minb = 8; }
    else { g_tail2 = 1; g_tail_minb = minb; }
}
void f110_debug_set_tile_counter(unsigned long long *buf) { g_tile_counter = buf; }
/* measurement aid: three cudaEvent_t (or NULL) recorded around k_obstacles and k_env_tail_obst of every obstacle tick (not
 * for graph capture: tools/bench_obstacles.py times plain ticks with them) */
void f110_debug_set_obst_events(void *before, void *between, void *after) {
    g_obst_ev[0] = (cudaEvent_t)before; g_obst_ev[1] = (cudaEvent_t)between; g_obst_ev[2] = (cudaEvent_t)after;
}
void f110_debug_set_chunk(int chunk_shift) { g_chunk = (chunk_shift < 0 || chunk_shift > 6) ? 3 : chunk_shift; }
/* test aid (not in the public header): `key=value` record of the kernels the last step / tick of the calling thread launched
 * (march kernel family and template choices, queue figures, tail kernel and shape); empty before the first one */
const char *f110_debug_last_launch(void) { return g_launch_rec; }

const char *f110_status_string(int status) {
    switch (status) {
        case F110_OK: return "ok";
        case F110_ERR_INVALID: return "invalid argument";
        case F110_ERR_NO_MAP: return "Map is not set for scan simulator.";
        case F110_ERR_CUDA: return "CUDA runtime error";
        case F110_ERR_INTEGRATOR: return "Invalid Integrator Specified. Please choose RK4 or Euler";
        case F110_ERR_POSE_COUNT: return "Number of poses for reset does not match number of agents.";
        case F110_ERR_AGENT_INDEX: return "Index given is out of bounds for list of agents.";
        default: return "unknown status";
    }
}

const char *f110_last_cuda_error(void) { return g_cuda_err; }

// One tick: validate, classify the map, plan the march (all before anything is enqueued: a tick either runs completely or not
// at all), then k_dynamics, the planned march and the tail, with an event between them when the caller profiles.
static int step_impl(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                     const double *actions, cudaStream_t st, cudaEvent_t *ev /* NULL or [4] */, const TailOpts *tail = nullptr,
                     const f110_obstacles *obst = nullptr, const f110_lidar *lidar = nullptr) {
    int rc;
    g_launch_rec[0] = '\0';
    TickPlan tp;
    ObstPlan ob;
    if ((rc = plan_tick(sim, map, tables, beams, actions, &tp, lidar))) return rc;
    if (obst) {
        if ((rc = plan_obstacles(sim, obst, map->num_layers, &ob))) return rc;
        tp.obst = &ob;
    }
    return launch_tick(sim, map, tables, beams, actions, tp, st, ev, tail);
}

int f110_step(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const double *actions,
              void *stream) {
    return f110_step_ex(sim, map, nullptr, beams, actions, stream);
}
int f110_step_ex(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                 const double *actions, void *stream) {
    return f110_step_obst(sim, map, tables, beams, actions, nullptr, stream);
}
int f110_step_obst(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                   const double *actions, const f110_obstacles *obst, void *stream) {
    return f110_step_lidar(sim, map, tables, beams, actions, obst, nullptr, stream);
}
int f110_step_lidar(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                    const double *actions, const f110_obstacles *obst, const f110_lidar *lidar, void *stream) {
    return step_impl(sim, map, tables, beams, actions, (cudaStream_t)stream, nullptr, nullptr, obst, lidar);
}

int f110_step_profile(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const double *actions,
                      float *kernel_ms /* host [3] */, void *stream) {
    return f110_step_profile_ex(sim, map, nullptr, beams, actions, kernel_ms, stream);
}
int f110_step_profile_ex(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                         const double *actions, float *kernel_ms /* host [3] */, void *stream) {
    if (!kernel_ms) return F110_ERR_INVALID;
    cudaEvent_t ev[4];
    for (int i = 0; i < 4; i++) CUDA_TRY(cudaEventCreate(&ev[i]));
    int rc = step_impl(sim, map, tables, beams, actions, (cudaStream_t)stream, ev);
    if (rc == F110_OK) {
        cudaError_t e = cudaEventSynchronize(ev[3]);
        if (e != cudaSuccess) rc = cuda_fail(e, "cudaEventSynchronize");
        for (int i = 0; i < 3 && rc == F110_OK; i++) {
            e = cudaEventElapsedTime(&kernel_ms[i], ev[i], ev[i + 1]);
            if (e != cudaSuccess) rc = cuda_fail(e, "cudaEventElapsedTime");
        }
    }
    for (int i = 0; i < 4; i++) cudaEventDestroy(ev[i]);
    return rc;
}

int f110_reset(const f110_sim *sim, const double *poses, const uint8_t *env_mask, void *stream) {
    int rc;
    if ((rc = check_sim(sim))) return rc;
    if (!poses) return F110_ERR_INVALID;
    const int NA = sim->num_envs * sim->num_agents;
    k_reset<<<(NA + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*sim, poses, env_mask);
    LAUNCH_CHECK("k_reset");
    return F110_OK;
}

static int check_env_arrays(const f110_sim *s) {
    if (!s->current_time || !s->lap_times || !s->lap_counts || !s->toggle_list || !s->near_starts ||
        !s->start_xs || !s->start_ys || !s->start_thetas || !s->start_rot || !s->done)
        return F110_ERR_INVALID;
    if (s->ego_idx < 0 || s->ego_idx >= s->num_agents) return F110_ERR_AGENT_INDEX;
    return F110_OK;
}

int f110_env_reset(const f110_sim *sim, const double *poses, const uint8_t *env_mask, void *stream) {
    int rc;
    if ((rc = check_sim(sim)) || (rc = check_env_arrays(sim))) return rc;
    if (!poses) return F110_ERR_INVALID;
    k_env_reset<<<(sim->num_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*sim, poses, env_mask);
    LAUNCH_CHECK("k_env_reset");
    return F110_OK;
}

int f110_env_post_step(const f110_sim *sim, void *stream) {
    int rc;
    if ((rc = check_sim(sim)) || (rc = check_env_arrays(sim))) return rc;
    k_env_post_step<<<(sim->num_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*sim);
    LAUNCH_CHECK("k_env_post_step");
    return F110_OK;
}

// per-layer start tables (f110_sim.start_offsets, host memory) -> ar.num_tables / ar.start_off; no tables without env_layer
static int start_tables(const f110_sim *sim, int32_t num_start, AutoResetArgs &ar) {
    ar.num_tables = 0;
    if (!sim->start_offsets || !sim->env_layer) return F110_OK;
    const int L = sim->num_start_tables;
    if (L < 1 || L > F110_MAX_START_TABLES || sim->start_offsets[0] != 0 || sim->start_offsets[L] != num_start)
        return F110_ERR_INVALID;
    for (int l = 0; l <= L; l++) {
        if (l < L && sim->start_offsets[l + 1] <= sim->start_offsets[l]) return F110_ERR_INVALID;
        ar.start_off[l] = sim->start_offsets[l];
    }
    ar.num_tables = L;
    return F110_OK;
}

int f110_autoreset(const f110_sim *sim, const double *start_poses, int32_t num_start, int32_t pose_gap,
                   uint64_t seed, uint64_t tick, void *stream) {
    return f110_autoreset_obst(sim, start_poses, num_start, pose_gap, seed, tick, nullptr, stream);
}
int f110_autoreset_obst(const f110_sim *sim, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
                        uint64_t tick, const f110_obstacles *obst, void *stream) {
    int rc;
    if ((rc = check_sim(sim))) return rc;
    if (!start_poses || num_start <= 0) return F110_ERR_INVALID;
    if (sim->ego_idx < 0 || sim->ego_idx >= sim->num_agents) return F110_ERR_AGENT_INDEX;
    if (sim->num_agents > 32) return F110_ERR_INVALID;      // the device-side auto-reset stages at most 32 start poses per env
    AutoResetArgs ar;
    ar.start_poses = start_poses; ar.num_start = num_start; ar.pose_gap = pose_gap; ar.seed = seed; ar.tick_host = tick;
    if ((rc = start_tables(sim, num_start, ar))) return rc;
    if (obst) {
        ObstPlan ob;
        if ((rc = plan_obstacles(sim, obst, -1, &ob))) return rc;
        RepeatDone rd;
        rd.done_any = nullptr; rd.done_tick = nullptr; rd.tick = 0;
        k_env_tail_obst<<<(sim->num_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*sim, 0, ar, rd, ob.d);
        LAUNCH_CHECK("k_env_tail_obst");
        return F110_OK;
    }
    k_autoreset<<<(sim->num_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*sim, ar);
    LAUNCH_CHECK("k_autoreset");
    return F110_OK;
}

int f110_obstacles_respawn(const f110_sim *sim, const f110_obstacles *obst, const uint8_t *env_mask, uint64_t tick, void *stream) {
    int rc;
    if ((rc = check_sim(sim))) return rc;
    if (!obst || !obst->candidates || sim->num_agents > 32) return F110_ERR_INVALID;
    ObstPlan ob;
    if ((rc = plan_obstacles(sim, obst, -1, &ob))) return rc;
    k_obst_respawn<<<(sim->num_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*sim, ob.d, env_mask, tick);
    LAUNCH_CHECK("k_obst_respawn");
    return F110_OK;
}

int f110_tick(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const double *actions,
              int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
              void *stream) {
    return f110_tick_ex(sim, map, nullptr, beams, actions, env_level, start_poses, num_start, pose_gap, seed, stream);
}
// the checks and the tail options of a whole tick (f110_tick_ex, f110_tick_repeat)
static int tick_tail_opts(const f110_sim *sim, const f110_map *map, int32_t env_level, const double *start_poses, int32_t num_start,
                          int32_t pose_gap, uint64_t seed, TailOpts *t) {
    int rc;
    if ((rc = check_sim(sim))) return rc;
    if (env_level && (rc = check_env_arrays(sim))) return rc;
    if (start_poses && (num_start <= 0 || sim->ego_idx < 0 || sim->ego_idx >= sim->num_agents || sim->num_agents > 32))
        return F110_ERR_INVALID;
    t->fused = true; t->env_level = env_level;
    t->ar.start_poses = start_poses; t->ar.num_start = num_start; t->ar.pose_gap = pose_gap; t->ar.seed = seed; t->ar.tick_host = 0;
    t->ar.num_tables = 0;
    if (start_poses && (rc = start_tables(sim, num_start, t->ar))) return rc;
    if (t->ar.num_tables && (!map || t->ar.num_tables != map->num_layers)) return F110_ERR_INVALID;
    return F110_OK;
}

int f110_tick_ex(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                 const double *actions, int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap,
                 uint64_t seed, void *stream) {
    return f110_tick_obst(sim, map, tables, beams, actions, env_level, start_poses, num_start, pose_gap, seed, nullptr, stream);
}
int f110_tick_obst(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                   const double *actions, int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap,
                   uint64_t seed, const f110_obstacles *obst, void *stream) {
    return f110_tick_lidar(sim, map, tables, beams, actions, env_level, start_poses, num_start, pose_gap, seed, obst, nullptr, stream);
}
int f110_tick_lidar(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                    const double *actions, int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap,
                    uint64_t seed, const f110_obstacles *obst, const f110_lidar *lidar, void *stream) {
    int rc;
    TailOpts t;
    if ((rc = tick_tail_opts(sim, map, env_level, start_poses, num_start, pose_gap, seed, &t))) return rc;
    return step_impl(sim, map, tables, beams, actions, (cudaStream_t)stream, nullptr, &t, obst, lidar);
}

int f110_tick_episodes(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                       const double *actions, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
                       const f110_obstacles *obst, const f110_lidar *lidar, const f110_episodes *ep, void *stream) {
    int rc;
    TailOpts t;
    TickPlan tp;
    ObstPlan ob;
    cudaStream_t st = (cudaStream_t)stream;
    if ((rc = tick_tail_opts(sim, map, 1, start_poses, num_start, pose_gap, seed, &t))) return rc;
    if ((rc = check_episodes(sim, ep, start_poses))) return rc;
    const AutoResetArgs ar = t.ar;
    t.ar.start_poses = nullptr;          // the plain tick runs without the auto-reset; k_episode_end restarts the ended envs
    g_launch_rec[0] = '\0';
    if ((rc = plan_tick(sim, map, tables, beams, actions, &tp, lidar))) return rc;
    if (!episode_march_ok(tp.march)) return F110_ERR_INVALID;
    if (obst) {
        if ((rc = plan_obstacles(sim, obst, map->num_layers, &ob))) return rc;
        tp.obst = &ob;
    }
    unsigned grid = 0u;
    if ((rc = ttc_grid(true, scan_units(tp.march), tp.march.count, &grid))) return rc;

    if ((rc = launch_tick(sim, map, tables, beams, actions, tp, st, nullptr, &t))) return rc;
    const int N = sim->num_envs, A = sim->num_agents;
    const uint32_t all = A == 32 ? 0xFFFFFFFFu : (1u << A) - 1u;
    // the slots whose scans exist: the mask on the short path, every slot when the tick ignores it (or has none)
    const uint32_t scan_slots = tp.lidar ? tp.lidar->mask : all;
    const uint32_t final_slots = (lidar && lidar->mask != F110_LIDAR_ALL) ? (lidar->mask & all) : all;
    ObstDraw no_draw;
    memset(&no_draw, 0, sizeof(no_draw));
    CUDA_TRY(cudaMemsetAsync(ep->list_count, 0, sizeof(uint32_t), st));
    k_episode_end<<<(N + 127) / 128, 128, 0, st>>>(*sim, ar, episode_k(ep), obst ? ob.d : no_draw);
    LAUNCH_CHECK("k_episode_end");
    RestartK r;
    r.list = ep->list; r.count = ep->list_count; r.scans = sim->scans; r.final_scans = ep->final_scans;
    r.tick_counter = sim->tick_counter; r.noise_std = sim->noise_std; r.noise_seed = sim->noise_seed;
    r.lidar = scan_slots; r.final_slots = final_slots;
    return launch_restart("k_episode_end", *sim, sim->march_rec, map, beams, tp, r, grid, st);
}

// ---- a held-action call (f110_tick_repeat_ticks_lidar, f110_tick_repeat_episodes_ticks): its checks, before anything is planned
static int check_repeat(const f110_sim *sim, const f110_map *map, int32_t repeat, int32_t first_tick, int32_t num_ticks,
                        const f110_repeat *rep, int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap,
                        uint64_t seed, const f110_lidar *lidar, TailOpts *t) {
    int rc;
    if ((rc = tick_tail_opts(sim, map, env_level, start_poses, num_start, pose_gap, seed, t))) return rc;
    if ((rc = check_lidar(sim, lidar))) return rc;
    if (repeat < 1 || repeat > F110_MAX_REPEAT || first_tick < 0 || num_ticks < 1 || first_tick > repeat - num_ticks) return F110_ERR_INVALID;
    if (!rep || !rep->list || !rep->list_count) return F110_ERR_INVALID;
    if ((rep->done_any || rep->done_tick) && !env_level) return F110_ERR_INVALID;     // done is computed by the env-level part
    return F110_OK;
}
// its plans: the ticks', the last tick's with a lidar mask, the obstacles'
static int plan_repeat_call(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                            const double *actions, int32_t repeat, const f110_obstacles *obst, const f110_lidar *lidar,
                            RepeatCall *c) {
    int rc;
    g_launch_rec[0] = '\0';
    if ((rc = plan_repeat(sim, map, tables, beams, actions, repeat, &c->rp))) return rc;
    c->masked = lidar && lidar->mask != F110_LIDAR_ALL;
    if (c->masked && (rc = plan_tick(sim, map, tables, beams, actions, &c->last, lidar))) return rc;
    if (obst) {
        if ((rc = plan_obstacles(sim, obst, map->num_layers, &c->ob))) return rc;
        c->rp.tick.obst = &c->ob;
        c->last.obst = &c->ob;
    }
    return F110_OK;
}
// its ticks first_tick .. first_tick + num_ticks - 1, each followed by k_repeat_done (a plain tick, when rep has the done
// outputs) and k_episode_latch (when latch is given; its tick and scans_exist are the last tick's on return), then the record
static int launch_repeat_ticks(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                               const double *actions, int32_t repeat, int32_t first_tick, int32_t num_ticks, const f110_repeat *rep,
                               RepeatCall &c, LatchK *latch, cudaStream_t st) {
    int rc;
    const RepeatPlan &rp = c.rp;
    const bool track_done = rep->done_any || rep->done_tick;
    for (int tick = first_tick; tick < first_tick + num_ticks; tick++) {
        const bool short_tick = rp.ttc && tick < repeat - 1;
        if (short_tick) {
            if ((rc = launch_ttc_tick(sim, map, beams, actions, rp, rep, tick, c.t, st))) return rc;
        } else {
            if ((rc = launch_tick(sim, map, tables, beams, actions, tick == repeat - 1 ? c.last_tick() : c.rp.tick, st, nullptr, &c.t)))
                return rc;
            if (track_done) {
                RepeatDone rd;
                rd.done_any = rep->done_any; rd.done_tick = rep->done_tick; rd.tick = tick;
                k_repeat_done<<<(sim->num_envs + 127) / 128, 128, 0, st>>>(*sim, rd);
                LAUNCH_CHECK("k_repeat_done");
            }
        }
        if (latch) {
            latch->tick = tick;
            latch->scans_exist = short_tick ? 0 : 1;
            k_episode_latch<<<(unsigned)(((long long)sim->num_envs * 32 + 127) / 128), 128, 0, st>>>(*sim, *latch);
            LAUNCH_CHECK("k_episode_latch");
        }
    }
    // the record of the call: the last plain tick's record (when the range holds one) and the repeat part
    static const char *units[3] = {"cells", "metres", "rot"};
    append_launch_record("%srepeat=%d sub=%s UNITS=%s grid=%u", g_launch_rec[0] ? " " : "", (int)repeat, rp.ttc ? "ttc" : "full",
                         units[rp.units], rp.grid);
    return F110_OK;
}

int f110_tick_repeat_ticks(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                           const double *actions, int32_t repeat, int32_t first_tick, int32_t num_ticks, const f110_repeat *rep,
                           int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
                           void *stream) {
    return f110_tick_repeat_ticks_obst(sim, map, tables, beams, actions, repeat, first_tick, num_ticks, rep, env_level, start_poses,
                                       num_start, pose_gap, seed, nullptr, stream);
}
int f110_tick_repeat_ticks_obst(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                                const double *actions, int32_t repeat, int32_t first_tick, int32_t num_ticks, const f110_repeat *rep,
                                int32_t env_level, const double *start_poses, int32_t num_start, int32_t pose_gap, uint64_t seed,
                                const f110_obstacles *obst, void *stream) {
    return f110_tick_repeat_ticks_lidar(sim, map, tables, beams, actions, repeat, first_tick, num_ticks, rep, env_level, start_poses,
                                        num_start, pose_gap, seed, obst, nullptr, stream);
}
int f110_tick_repeat_ticks_lidar(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables,
                                 const f110_beams *beams, const double *actions, int32_t repeat, int32_t first_tick,
                                 int32_t num_ticks, const f110_repeat *rep, int32_t env_level, const double *start_poses,
                                 int32_t num_start, int32_t pose_gap, uint64_t seed, const f110_obstacles *obst,
                                 const f110_lidar *lidar, void *stream) {
    int rc;
    RepeatCall c;
    cudaStream_t st = (cudaStream_t)stream;
    if ((rc = check_repeat(sim, map, repeat, first_tick, num_ticks, rep, env_level, start_poses, num_start, pose_gap, seed, lidar,
                           &c.t)))
        return rc;
    if ((rc = plan_repeat_call(sim, map, tables, beams, actions, repeat, obst, lidar, &c))) return rc;
    if (first_tick == 0) CUDA_TRY(cudaMemsetAsync(rep->list_count, 0, sizeof(uint32_t) * (size_t)repeat, st));
    return launch_repeat_ticks(sim, map, tables, beams, actions, repeat, first_tick, num_ticks, rep, c, nullptr, st);
}

int f110_tick_repeat(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                     const double *actions, int32_t repeat, const f110_repeat *rep, int32_t env_level, const double *start_poses,
                     int32_t num_start, int32_t pose_gap, uint64_t seed, void *stream) {
    return f110_tick_repeat_ticks(sim, map, tables, beams, actions, repeat, 0, repeat, rep, env_level, start_poses, num_start,
                                  pose_gap, seed, stream);
}

// ---- episodes under a held action (csrc/episode_repeat.cuh): the ticks of f110_tick_repeat, k_episode_latch after each, then
// the final scans of the envs that ended on a short-path tick and the restart of every env that ended in the call
int f110_tick_repeat_episodes_ticks(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables,
                                    const f110_beams *beams, const double *actions, int32_t repeat, int32_t first_tick,
                                    int32_t num_ticks, const f110_repeat *rep, const double *start_poses, int32_t num_start,
                                    int32_t pose_gap, uint64_t seed, const f110_obstacles *obst, const f110_lidar *lidar,
                                    const f110_episodes *ep, const f110_episode_repeat *er, void *stream) {
    int rc;
    RepeatCall c;
    cudaStream_t st = (cudaStream_t)stream;
    if ((rc = check_repeat(sim, map, repeat, first_tick, num_ticks, rep, 1, start_poses, num_start, pose_gap, seed, lidar, &c.t)))
        return rc;
    if ((rc = check_episodes(sim, ep, start_poses))) return rc;
    if (!er || !er->end_tick || !er->snap_rec || !er->snap_poses || !er->snap_wall_flag || !er->scan_list || !er->scan_count)
        return F110_ERR_INVALID;
    const AutoResetArgs ar = c.t.ar;
    c.t.ar.start_poses = nullptr;        // the ticks run without the auto-reset; k_episode_restart restarts the ended envs
    if ((rc = plan_repeat_call(sim, map, tables, beams, actions, repeat, obst, lidar, &c))) return rc;
    const RepeatPlan &rp = c.rp;
    const TickPlan &lp = c.last_tick();
    // the plans the final-scan pass and the last tick and the restart march run with
    if (!episode_march_ok(rp.tick.march) || !episode_march_ok(lp.march)) return F110_ERR_INVALID;
    const int units = scan_units(lp.march);
    unsigned grid = 0u, fs_grid = 0u;
    if ((rc = ttc_grid(true, units, lp.march.count, &grid))) return rc;
    if (rp.ttc && (rc = ttc_grid(true, units, false, &fs_grid))) return rc;

    const int N = sim->num_envs, A = sim->num_agents;
    const uint32_t all = A == 32 ? 0xFFFFFFFFu : (1u << A) - 1u;
    // the slots whose scans the last tick computes, and the slots that have a lidar (their scans go to final_scans)
    const uint32_t scan_slots = lp.lidar ? lp.lidar->mask : all;
    const uint32_t final_slots = c.masked ? (lidar->mask & all) : all;
    f110_repeat rn = *rep;               // the ticks' own done bookkeeping is off: k_episode_latch keeps it to the running episode
    rn.done_any = nullptr; rn.done_tick = nullptr;
    LatchK k;
    k.ep = episode_k(ep);
    k.end_tick = er->end_tick; k.done_any = rep->done_any; k.done_tick = rep->done_tick;
    k.scans = sim->scans; k.final_scans = ep->final_scans;
    k.snap_rec = reinterpret_cast<double2 *>(er->snap_rec); k.snap_poses = er->snap_poses; k.snap_flag = er->snap_wall_flag;
    k.scan_list = er->scan_list; k.scan_count = er->scan_count;
    k.num_beams = beams->num_beams; k.final_slots = final_slots;

    if (first_tick == 0) {
        CUDA_TRY(cudaMemsetAsync(rep->list_count, 0, sizeof(uint32_t) * (size_t)repeat, st));
        CUDA_TRY(cudaMemsetAsync(er->scan_count, 0, sizeof(uint32_t), st));
    }
    if ((rc = launch_repeat_ticks(sim, map, tables, beams, actions, repeat, first_tick, num_ticks, &rn, c, &k, st))) return rc;
    if (first_tick + num_ticks < repeat) return F110_OK;

    // the final scans of the envs that ended on a short-path tick, from the snapshot of their end tick
    const bool final_pass = rp.ttc && repeat > 1 && final_slots != 0u;
    if (final_pass) {
        f110_sim fs = *sim;
        fs.agent_poses = er->snap_poses; fs.scans = ep->final_scans;
        fs.wall_flag = er->snap_wall_flag;          // never written: the snapshot's iTTC threshold is -inf
        fs.collisions = ep->final_collisions; fs.collision_idx = ep->final_collision_idx;
        RestartK r;
        r.list = er->scan_list; r.count = er->scan_count; r.scans = ep->final_scans; r.final_scans = ep->final_scans;
        r.tick_counter = sim->tick_counter; r.noise_std = 0.0; r.noise_seed = 0ull;
        r.lidar = final_slots; r.final_slots = 0u;
        if ((rc = launch_restart(nullptr, fs, er->snap_rec, map, beams, rp.tick, r, fs_grid, st))) return rc;
    }

    // the restart of every env that ended in the call, at the counter of its last tick
    ObstDraw no_draw;
    memset(&no_draw, 0, sizeof(no_draw));
    CUDA_TRY(cudaMemsetAsync(ep->list_count, 0, sizeof(uint32_t), st));
    k_episode_restart<<<(N + 127) / 128, 128, 0, st>>>(*sim, ar, k, obst ? c.ob.d : no_draw, ep->track_seg, er->track_delta_sum,
                                                      ep->list, ep->list_count);
    LAUNCH_CHECK("k_episode_restart");
    RestartK r;
    r.list = ep->list; r.count = ep->list_count; r.scans = sim->scans; r.final_scans = ep->final_scans;
    r.tick_counter = sim->tick_counter; r.noise_std = sim->noise_std; r.noise_seed = sim->noise_seed;
    r.lidar = scan_slots; r.final_slots = 0u;    // the crash scans are in final_scans already (k_episode_latch)
    if ((rc = launch_restart("k_episode_restart", *sim, sim->march_rec, map, beams, lp, r, grid, st))) return rc;
    if (final_pass)
        append_launch_record(" final_scan=k_restart_march%s%s", A > 1 ? "+k_episode_cast" : "", obst ? "+k_episode_obstacles" : "");
    else
        append_launch_record(" final_scan=none");
    return F110_OK;
}
int f110_tick_repeat_episodes(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                              const double *actions, int32_t repeat, const f110_repeat *rep, const double *start_poses,
                              int32_t num_start, int32_t pose_gap, uint64_t seed, const f110_obstacles *obst,
                              const f110_lidar *lidar, const f110_episodes *ep, const f110_episode_repeat *er, void *stream) {
    return f110_tick_repeat_episodes_ticks(sim, map, tables, beams, actions, repeat, 0, repeat, rep, start_poses, num_start,
                                           pose_gap, seed, obst, lidar, ep, er, stream);
}

// ---- per-episode parameter draws (csrc/param_draw.cuh): one k_param_draw launch, after the call that restarted the envs
static int param_draw_launch(const f110_sim *sim, const f110_param_draw *draw, int rule, const uint8_t *mask,
                             const f110_episodes *ep, void *stream) {
    if (!sim || !draw || !draw->lo || !draw->hi) return F110_ERR_INVALID;
    if (sim->num_envs <= 0 || sim->num_agents <= 0 || sim->num_agents > 32 || !sim->params || !sim->params_per_env ||
        !sim->tick_counter)
        return F110_ERR_INVALID;
    if (rule == PARAM_DRAW_AUTORESET && (!sim->collisions || sim->ego_idx < 0 || sim->ego_idx >= sim->num_agents))
        return F110_ERR_INVALID;
    if (rule == PARAM_DRAW_EPISODES && (!ep || !ep->terminated || !ep->truncated)) return F110_ERR_INVALID;
    const int A = sim->num_agents;
    for (int i = 0; i < A; i++)
        if (draw->keys[i] >> F110_PARAM_DRAW_KEYS) return F110_ERR_INVALID;
    for (int q = 0; q < F110_NPARAM; q++)
        if (draw->group[q] < 0 || draw->group[q] >= F110_NPARAM) return F110_ERR_INVALID;
    ParamDrawK k;
    k.lo = draw->lo; k.hi = draw->hi;
    k.params = const_cast<double *>(sim->params);
    k.final_params = rule == PARAM_DRAW_EPISODES ? draw->final_params : nullptr;
    k.tick_counter = sim->tick_counter;
    k.mask = mask; k.collisions = sim->collisions;
    k.terminated = ep ? ep->terminated : nullptr; k.truncated = ep ? ep->truncated : nullptr;
    k.seed = draw->seed;
    k.num_envs = sim->num_envs; k.num_agents = A; k.ego = sim->ego_idx; k.rule = rule; k.per_env = draw->per_env ? 1 : 0;
    memcpy(k.keys, draw->keys, sizeof(k.keys));
    memcpy(k.group, draw->group, sizeof(k.group));
    const long long NA = (long long)sim->num_envs * A;
    k_param_draw<<<(unsigned)((NA + 127) / 128), 128, 0, (cudaStream_t)stream>>>(k);
    LAUNCH_CHECK("k_param_draw");
    return F110_OK;
}
// ---- f110_predict (include/f110_predict.h, csrc/predict.cuh)
// The tick's own plan decides the map kind: the record arithmetic (fill_first_lookup) and the per-beam march (fill_ttc_k) of
// k_march_ttc on it, with the units of the tick's short path.  Validation ends before the one launch.
struct PredictCall {
    PredictK p;
    FirstLookup fl;
    TtcK q;
    int units;
    unsigned grid;
};
static int plan_predict(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                        const f110_predict_args *args, PredictCall *pc) {
    int rc;
    if (!sim || !args || !args->agent_ids || !args->actions || !args->final_state || !args->wall_step) return F110_ERR_INVALID;
    if (args->M < 1 || args->K < 1 || args->H < 1 || args->H > F110_PREDICT_MAX_H) return F110_ERR_INVALID;
    const long long samples = (long long)args->M * (long long)args->K;
    if (samples > 0x7fffffffll) return F110_ERR_INVALID;
    if ((rc = check_sim(sim)) || (rc = check_map(map)) || (rc = check_beams(beams))) return rc;
    if ((long long)sim->num_envs * sim->num_agents > 0x7fffffffll) return F110_ERR_INVALID;
    TickPlan tp = {};
    if ((rc = classify_map(map, &tp.geom))) return rc;
    if ((rc = plan_march(sim, map, tables, beams, tp.geom, rm_variant(), &tp.march))) return rc;
    if (!ttc_tables_ok(sim, map, beams, tp.march)) return F110_ERR_INVALID;
    const MarchPlan &m = tp.march;
    PredictK &p = pc->p;
    p.agent_ids = args->agent_ids;
    p.actions = reinterpret_cast<const double2 *>(args->actions);
    p.final_state = args->final_state; p.wall_step = args->wall_step;
    p.states = args->states; p.clearance = args->clearance;
    p.samples = (unsigned long long)samples; p.K = (unsigned)args->K; p.H = args->H;
    p.d0_scale = m.cell_units ? map->resolution : 1.0;
    p.fov = beams->fov; p.theta_dis_f = (double)map->theta_dis;
    pc->fl = fill_first_lookup(sim, map, beams, tp.geom, m);
    pc->q = fill_ttc_k(sim, map, beams, tp, nullptr, nullptr);
    pc->units = scan_units(m);
    pc->grid = (unsigned)((samples + F110_PREDICT_THREADS - 1) / F110_PREDICT_THREADS);
    return F110_OK;
}
int f110_predict(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                 const f110_predict_args *args, void *stream) {
    int rc;
    PredictCall c;
    if ((rc = plan_predict(sim, map, tables, beams, args, &c))) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    dispatch_units(c.units, [&](auto u) {
        k_predict<decltype(u)::value><<<c.grid, F110_PREDICT_THREADS, 0, st>>>(*sim, c.fl, c.q, c.p);
    });
    LAUNCH_CHECK("k_predict");
    return F110_OK;
}

// ---- f110_predict_scored (include/f110_mppi.h, csrc/predict.cuh): k_scored_acquire, then k_scored_rollout
static bool track_ok(const f110_track *track);
int f110_predict_scored(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables, const f110_beams *beams,
                        const f110_track *track, const f110_predict_args *args, const f110_cost *cost, void *stream) {
    int rc;
    if (!map || !track_ok(track) || !cost || !cost->cost || !cost->seg0 || !cost->s0) return F110_ERR_INVALID;
    if (track->num_tables != (map->num_layers > 1 ? map->num_layers : 1)) return F110_ERR_INVALID;
    if (cost->back < 0 || cost->fwd < 0 || (long long)cost->back + cost->fwd + 1 > F110_TRACK_MAX_WINDOW) return F110_ERR_INVALID;
    if (!isfinite(cost->reacquire_dist) || !(cost->reacquire_dist > 0.0)) return F110_ERR_INVALID;
    const double w[7] = {cost->w_lat, cost->w_head, cost->w_clear, cost->w_dsteer, cost->w_dspeed, cost->w_prog, cost->w_wall};
    for (double v : w)
        if (!isfinite(v) || !(v >= 0.0)) return F110_ERR_INVALID;
    if (!isfinite(cost->clear_min)) return F110_ERR_INVALID;
    PredictCall pc;
    if ((rc = plan_predict(sim, map, tables, beams, args, &pc))) return rc;
    CostK c;
    c.segments = track->segments; c.table_start = track->table_start; c.num_tables = track->num_tables;
    c.back = cost->back; c.window = cost->back + cost->fwd + 1; c.reacquire_dist = cost->reacquire_dist;
    c.seg0 = cost->seg0; c.s0 = cost->s0;
    c.prev_action = reinterpret_cast<const double2 *>(cost->prev_action);
    c.cost = cost->cost;
    c.w_lat = cost->w_lat; c.w_head = cost->w_head; c.w_clear = cost->w_clear; c.w_dsteer = cost->w_dsteer;
    c.w_dspeed = cost->w_dspeed; c.w_prog = cost->w_prog; c.w_wall = cost->w_wall; c.clear_min = cost->clear_min;
    const cudaStream_t st = (cudaStream_t)stream;
    const int M = args->M;
    k_scored_acquire<<<(unsigned)(((long long)M * 32 + 127) / 128), 128, 0, st>>>(*sim, args->agent_ids, M, c);
    LAUNCH_CHECK("k_scored_acquire");
    dispatch_units(pc.units, [&](auto u) {
        k_scored_rollout<decltype(u)::value><<<pc.grid, F110_PREDICT_THREADS, 0, st>>>(*sim, pc.fl, pc.q, pc.p, c);
    });
    LAUNCH_CHECK("k_scored_rollout");
    return F110_OK;
}

// ---- f110_mppi_sample / f110_mppi_update (include/f110_mppi.h, csrc/mppi.cuh)
static bool mppi_ok(const f110_mppi *g, MppiK *k) {
    if (!g || !g->agent_ids || !g->nominal || !g->iteration || !g->no_finite) return false;
    if (g->M < 1 || g->K < 2 || g->K > F110_MPPI_MAX_K || g->H < 1 || g->H > F110_MPPI_MAX_H) return false;
    if ((long long)g->M * g->K * g->H > 0x7fffffffll) return false;
    const double v[8] = {g->sigma_steer, g->sigma_speed, g->steer_lo, g->steer_hi, g->speed_lo, g->speed_hi, g->lambda, 0.0};
    for (double x : v)
        if (!isfinite(x)) return false;
    if (!(g->sigma_steer >= 0.0) || !(g->sigma_speed >= 0.0) || !(g->lambda > 0.0)) return false;
    if (!(g->steer_lo <= g->steer_hi) || !(g->speed_lo <= g->speed_hi)) return false;
    k->agent_ids = g->agent_ids;
    k->nominal = reinterpret_cast<double2 *>(g->nominal);
    k->iteration = g->iteration; k->no_finite = g->no_finite;
    k->sigma = make_double2(g->sigma_steer, g->sigma_speed);
    k->lo = make_double2(g->steer_lo, g->speed_lo); k->hi = make_double2(g->steer_hi, g->speed_hi);
    k->lambda = g->lambda; k->seed = g->seed;
    k->M = g->M; k->K = g->K; k->H = g->H;
    return true;
}

int f110_mppi_sample(const f110_sim *sim, const f110_mppi *mppi, const f110_episodes *ep, double *actions, void *stream) {
    MppiK k;
    if (!mppi_ok(mppi, &k) || !sim || !sim->steer_cnt || !actions) return F110_ERR_INVALID;
    if (sim->num_envs <= 0 || sim->num_agents <= 0 || (long long)sim->num_envs * sim->num_agents > 0x7fffffffll)
        return F110_ERR_INVALID;
    if (ep && (!ep->terminated || !ep->truncated)) return F110_ERR_INVALID;
    const long long n = (long long)k.M * k.K * k.H;
    k_mppi_sample<<<(unsigned)((n + F110_MPPI_SAMPLE_THREADS - 1) / F110_MPPI_SAMPLE_THREADS), F110_MPPI_SAMPLE_THREADS, 0,
                    (cudaStream_t)stream>>>(k, sim->steer_cnt, ep ? ep->terminated : nullptr, ep ? ep->truncated : nullptr,
                                            sim->num_envs * sim->num_agents, sim->num_agents,
                                            reinterpret_cast<double2 *>(actions));
    LAUNCH_CHECK("k_mppi_sample");
    return F110_OK;
}

int f110_mppi_update(const f110_mppi *mppi, const double *actions, const double *cost, double *action_out, int32_t num_rows,
                     double *weights, int32_t *argmin, void *stream) {
    MppiK k;
    if (!mppi_ok(mppi, &k) || !actions || !cost || !action_out || num_rows < 1) return F110_ERR_INVALID;
    const size_t smem = ((size_t)k.K + 2 * (size_t)k.H) * sizeof(double);     // with the static part <= 48 KiB (mppi.cuh)
    k_mppi_update<<<(unsigned)k.M, F110_MPPI_UPDATE_THREADS, smem, (cudaStream_t)stream>>>(
        k, reinterpret_cast<const double2 *>(actions), cost, reinterpret_cast<double2 *>(action_out), num_rows, weights, argmin);
    LAUNCH_CHECK("k_mppi_update");
    return F110_OK;
}

int f110_params_draw(const f110_sim *sim, const f110_param_draw *draw, const uint8_t *env_mask, void *stream) {
    return param_draw_launch(sim, draw, PARAM_DRAW_MASK, env_mask, nullptr, stream);
}
int f110_params_draw_autoreset(const f110_sim *sim, const f110_param_draw *draw, void *stream) {
    return param_draw_launch(sim, draw, PARAM_DRAW_AUTORESET, nullptr, nullptr, stream);
}
int f110_params_draw_episodes(const f110_sim *sim, const f110_param_draw *draw, const f110_episodes *ep, void *stream) {
    return param_draw_launch(sim, draw, PARAM_DRAW_EPISODES, nullptr, ep, stream);
}

// the tail of a host-buffer step: the fused tail, with the env level when the sim has its arrays, and no auto-reset
static TailOpts host_step_tail(bool env_level) {
    TailOpts t;
    t.fused = true; t.env_level = env_level ? 1 : 0;
    t.ar.start_poses = nullptr; t.ar.num_start = 0; t.ar.pose_gap = 0; t.ar.seed = 0; t.ar.tick_host = 0;
    return t;
}
int f110_step_host(const f110_sim *sim, const f110_map *map, const f110_beams *beams, const double *actions_host,
                   double *actions_dev_scratch, const f110_host_obs *out, void *stream) {
    int rc;
    if ((rc = check_sim(sim))) return rc;
    if (!actions_host || !actions_dev_scratch || !out) return F110_ERR_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t NA = (size_t)sim->num_envs * sim->num_agents;
    CUDA_TRY(cudaMemcpyAsync(actions_dev_scratch, actions_host, NA * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
    const bool env_level = sim->current_time && sim->done;
    if (env_level && (rc = check_env_arrays(sim))) return rc;
    const TailOpts t = host_step_tail(env_level);
    if ((rc = step_impl(sim, map, nullptr, beams, actions_dev_scratch, st, nullptr, &t))) return rc;
    if (out->scans)
        CUDA_TRY(cudaMemcpyAsync(out->scans, sim->scans, NA * beams->num_beams * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (out->state)
        CUDA_TRY(cudaMemcpyAsync(out->state, sim->state, NA * 7 * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (out->collisions)
        CUDA_TRY(cudaMemcpyAsync(out->collisions, sim->collisions, NA * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (env_level) {
        if (out->done)
            CUDA_TRY(cudaMemcpyAsync(out->done, sim->done, (size_t)sim->num_envs, cudaMemcpyDeviceToHost, st));
        if (out->lap_times)
            CUDA_TRY(cudaMemcpyAsync(out->lap_times, sim->lap_times, NA * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (out->lap_counts)
            CUDA_TRY(cudaMemcpyAsync(out->lap_counts, sim->lap_counts, NA * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    return F110_OK;
}

int f110_step_host_async(const f110_sim *sim, const f110_map *map, const f110_beams *beams,
                         const double *actions_host, double *actions_dev_scratch, const f110_host_obs *stage,
                         const f110_host_obs *out, void *compute_stream, void *copy_stream, void *ev_tick_done,
                         void *ev_copy_done) {
    return f110_step_host_async_ex(sim, map, nullptr, beams, actions_host, actions_dev_scratch, stage, out, compute_stream,
                                   copy_stream, ev_tick_done, ev_copy_done);
}
int f110_step_host_async_ex(const f110_sim *sim, const f110_map *map, const f110_march_tables *tables,
                            const f110_beams *beams, const double *actions_host, double *actions_dev_scratch,
                            const f110_host_obs *stage, const f110_host_obs *out, void *compute_stream, void *copy_stream,
                            void *ev_tick_done, void *ev_copy_done) {
    int rc;
    if ((rc = check_sim(sim))) return rc;
    if (!actions_host || !actions_dev_scratch || !stage || !out || !ev_tick_done || !ev_copy_done) return F110_ERR_INVALID;
    cudaStream_t cs = (cudaStream_t)compute_stream, ps = (cudaStream_t)copy_stream;
    cudaEvent_t e_tick = (cudaEvent_t)ev_tick_done, e_copy = (cudaEvent_t)ev_copy_done;
    const size_t NA = (size_t)sim->num_envs * sim->num_agents;
    const bool env_level = sim->current_time && sim->done;
    if (env_level && (rc = check_env_arrays(sim))) return rc;
    CUDA_TRY(cudaMemcpyAsync(actions_dev_scratch, actions_host, NA * 2 * sizeof(double), cudaMemcpyHostToDevice, cs));
    const TailOpts t = host_step_tail(env_level);
    if ((rc = step_impl(sim, map, tables, beams, actions_dev_scratch, cs, nullptr, &t))) return rc;
    // the staging buffers may still be draining to the host from their previous use
    CUDA_TRY(cudaStreamWaitEvent(cs, e_copy, 0));
    struct Part { void *dst_dev, *dst_host; const void *src; size_t bytes; };
    const Part parts[6] = {
        { stage->scans, out->scans, sim->scans, NA * beams->num_beams * sizeof(float) },
        { stage->state, out->state, sim->state, NA * 7 * sizeof(double) },
        { stage->collisions, out->collisions, sim->collisions, NA * sizeof(double) },
        { stage->done, out->done, env_level ? sim->done : nullptr, (size_t)sim->num_envs },
        { stage->lap_times, out->lap_times, env_level ? sim->lap_times : nullptr, NA * sizeof(double) },
        { stage->lap_counts, out->lap_counts, env_level ? sim->lap_counts : nullptr, NA * sizeof(double) },
    };
    for (int i = 0; i < 6; i++)
        if (parts[i].dst_dev && parts[i].dst_host && parts[i].src)
            CUDA_TRY(cudaMemcpyAsync(parts[i].dst_dev, parts[i].src, parts[i].bytes, cudaMemcpyDeviceToDevice, cs));
    // narrow scan block: the snapshot IS the packing (3 bytes per beam cross PCIe instead of 4)
    const bool packed = !stage->scans && !out->scans && stage->scans_u24 && out->scans_u24;
    if (packed && (rc = f110_pack_scans_u24(sim->scans, (int64_t)(NA * beams->num_beams), stage->scans_u24, cs))) return rc;
    CUDA_TRY(cudaEventRecord(e_tick, cs));
    CUDA_TRY(cudaStreamWaitEvent(ps, e_tick, 0));
    for (int i = 0; i < 6; i++)
        if (parts[i].dst_dev && parts[i].dst_host && parts[i].src)
            CUDA_TRY(cudaMemcpyAsync(parts[i].dst_host, parts[i].dst_dev, parts[i].bytes, cudaMemcpyDeviceToHost, ps));
    if (packed)
        CUDA_TRY(cudaMemcpyAsync(out->scans_u24, stage->scans_u24, NA * beams->num_beams * 3, cudaMemcpyDeviceToHost, ps));
    CUDA_TRY(cudaEventRecord(e_copy, ps));
    return F110_OK;
}

int64_t f110_map_brick_elems(const f110_map *map) {
    if (!map || !map->dt_cells_pad || !map->fast_path || map->num_layers > 1 || map->layer_geom || map->height < 1 ||
        map->width < 1)
        return 0;
    return (int64_t)brick_elems(map);
}

int f110_map_brick(const f110_map *map, double *out, void *stream) {
    const int64_t n = f110_map_brick_elems(map);
    if (n <= 0 || !out) return F110_ERR_INVALID;
    k_map_brick<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(map->dt_cells_pad, (unsigned)map->height,
                                                                                 (unsigned)map->width, (unsigned)brick_cols(map),
                                                                                 out, (unsigned)n);
    LAUNCH_CHECK("k_map_brick");
    return F110_OK;
}

int f110_scan(const f110_map *map, const f110_beams *beams, const double *poses, int32_t M, float *out_f32,
              double *out_f64, unsigned long long *lookup_counter, void *stream) {
    int rc;
    if ((rc = check_map(map)) || (rc = check_beams(beams))) return rc;
    if (!poses || M <= 0 || (!out_f32 && !out_f64)) return F110_ERR_INVALID;
    if ((map->num_layers > 1 && map->layer_geom) || map->layer_res || map->layer_rot) return F110_ERR_INVALID;     // canvas stacks: the tick only
    MarchArgs g;
    memset(&g, 0, sizeof(g));
    g.scan_pose = poses;
    g.out_f32 = out_f32;
    g.out_f64 = out_f64;
    g.lookup_counter = lookup_counter;
    g.total = (long long)M * beams->num_beams;
    const unsigned blocks = raymarch_blocks(g.total);
    if (!blocks) return F110_ERR_INVALID;
    return launch_raymarch(make_view(map), make_view(beams), g, map->fast_path != 0, true, blocks, (cudaStream_t)stream);
}

int f110_scan_layers(const f110_map *map, const f110_beams *beams, const double *poses, const int32_t *layer_ids, int32_t M,
                     float *out_f32, double *out_f64, unsigned long long *lookup_counter, void *stream) {
    int rc;
    if ((rc = check_map(map)) || (rc = check_beams(beams))) return rc;
    if (!poses || M <= 0 || (!out_f32 && !out_f64)) return F110_ERR_INVALID;
    MapGeom geom;
    if ((rc = classify_map(map, &geom))) return rc;
    const bool het = geom.het, unrotated = geom.unrotated;
    const unsigned layers = geom.layers;
    if (!unrotated && layers > 1 && !map->layer_rot) return F110_ERR_INVALID;     // a rotated stack carries its yaws in layer_rot
    if (!layer_ids && layers > 1) return F110_ERR_INVALID;
    // the lean march's preconditions: `d > eps` == `d != 0`, the doubled LUT instead of the wrap, a Q16.48 LUT index
    if (!map->sincos2 || !(map->eps >= 0.0) || !(map->dt_min_positive > map->eps) || !(beams->fov > 0.0) ||
        !(beams->fov < 6.283185307179586) || !(beams->theta_index_increment > 0.0) || map->theta_dis >= 32768)
        return F110_ERR_INVALID;
    if ((unsigned long long)M * (unsigned long long)beams->num_beams >= (1ull << 32)) return F110_ERR_INVALID;
    const int units = (!unrotated || map->layer_rot) ? F110_SCAN_UNITS_ROT
                    : (map->fast_path && map->dt_cells_pad) ? F110_SCAN_UNITS_CELLS : F110_SCAN_UNITS_METRES;
    const bool cells = units == F110_SCAN_UNITS_CELLS;
    const MapView mv = make_view(map);
    ScanLeanK p;
    memset(&p, 0, sizeof(p));
    p.table = cells ? map->dt_cells_pad : map->dt;
    p.dt = map->dt;
    p.sincos2 = reinterpret_cast<const double2 *>(map->sincos2);
    p.poses = poses;
    p.layer_ids = layers > 1 ? layer_ids : nullptr;
    p.out_f32 = out_f32; p.out_f64 = out_f64; p.lookup_counter = lookup_counter;
    p.layer_geom = het ? map->layer_geom : nullptr;
    p.layer_res = het ? map->layer_res : nullptr;
    p.layer_rot = het ? map->layer_rot : nullptr;
    p.orig = make_double2(map->orig_x, map->orig_y); p.ext = make_double2(mv.x_max, mv.y_max);
    p.res = make_double2(map->resolution, 1.0 / map->resolution); p.rot = make_double2(map->orig_c, map->orig_s);
    p.tmax = cells ? map->max_range * p.res.y : map->max_range;
    p.max_range = map->max_range; p.eps = map->eps; p.fov = beams->fov; p.theta_dis_f = (double)map->theta_dis;
    p.inc = beams->theta_index_increment;
    lut_fixed_point(beams, &p.inc_fx, &p.guard32);
    const unsigned long long cells_hw = (unsigned long long)map->width * (unsigned long long)map->height;
    p.table_stride = cells ? (unsigned long long)(map->width + 1) * (unsigned long long)(map->height + 1) : cells_hw;
    p.dt_stride = cells_hw;
    p.width = (unsigned)map->width; p.height = (unsigned)map->height; p.last = (unsigned)(cells_hw - 1ull);
    p.B = beams->num_beams;
    p.ipa = (unsigned)((beams->num_beams + 31) / 32);
    p.items = (unsigned long long)M * p.ipa;
    p.num_layers = layers;
    // a map that breaks the half-bound rule on origin, extent and ray reach (MapGeom.reach_ok), or whose tables do not fit the
    // 32-bit lean indices, takes the literal path for every pose
    p.literal = (geom.reach_ok && geom.cells32 && geom.padded32) ? 0 : 1;
    p.inv_res_fine = 1.0 / geom.res_fine;
    const unsigned long long blocks = (p.items * 32ull + F110_SCAN_THREADS - 1) / F110_SCAN_THREADS;
    if (blocks > 0x7fffffffull) return F110_ERR_INVALID;
    const bool count = lookup_counter != nullptr;
    static const char *const names[3] = {"cells", "metres", "rot"};
    snprintf(g_launch_rec, sizeof(g_launch_rec), "scan=lean UNITS=%s layers=%u COUNT=%d LITERAL=%d PT=%d grid=%llu", names[units],
             layers, count ? 1 : 0, p.literal, F110_SCAN_THREADS, blocks);
    const cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid((unsigned)blocks), block(F110_SCAN_THREADS);
    if (units == F110_SCAN_UNITS_CELLS) {
        if (count) k_scan_lean<F110_SCAN_UNITS_CELLS, true><<<grid, block, 0, st>>>(p);
        else k_scan_lean<F110_SCAN_UNITS_CELLS, false><<<grid, block, 0, st>>>(p);
    } else if (units == F110_SCAN_UNITS_METRES) {
        if (count) k_scan_lean<F110_SCAN_UNITS_METRES, true><<<grid, block, 0, st>>>(p);
        else k_scan_lean<F110_SCAN_UNITS_METRES, false><<<grid, block, 0, st>>>(p);
    } else {
        if (count) k_scan_lean<F110_SCAN_UNITS_ROT, true><<<grid, block, 0, st>>>(p);
        else k_scan_lean<F110_SCAN_UNITS_ROT, false><<<grid, block, 0, st>>>(p);
    }
    LAUNCH_CHECK("k_scan_lean");
    return F110_OK;
}

int f110_render_views(const f110_sim *sim, const f110_map *map, const int32_t *agent_ids, int32_t V, int32_t height,
                      int32_t width, double metres_per_pixel, double forward_offset, int32_t heading_up, uint8_t *out,
                      void *stream) {
    return f110_render_views_obst(sim, map, nullptr, agent_ids, V, height, width, metres_per_pixel, forward_offset, heading_up, out,
                                  stream);
}
int f110_render_views_obst(const f110_sim *sim, const f110_map *map, const f110_obstacles *obst, const int32_t *agent_ids, int32_t V,
                           int32_t height, int32_t width, double metres_per_pixel, double forward_offset, int32_t heading_up,
                           uint8_t *out, void *stream) {
    if (!sim || !map || !agent_ids || !out || !sim->state) return F110_ERR_INVALID;
    if (V < 1 || height < 1 || height > F110_RENDER_MAX_SIZE || width < 1 || width > F110_RENDER_MAX_SIZE) return F110_ERR_INVALID;
    if (!isfinite(metres_per_pixel) || !(metres_per_pixel > 0.0) || !isfinite(forward_offset)) return F110_ERR_INVALID;
    if (sim->num_envs <= 0 || sim->num_agents <= 0 || sim->num_agents > F110_RENDER_MAX_AGENTS ||
        (long long)sim->num_envs * sim->num_agents > 0x7fffffffll)
        return F110_ERR_INVALID;
    if (!map->dt || map->height <= 0 || map->width <= 0) return F110_ERR_NO_MAP;
    if (!(map->resolution > 0.0)) return F110_ERR_INVALID;
    MapGeom geom;
    int rc;
    if ((rc = classify_map(map, &geom))) return rc;
    const bool het = geom.het;
    const unsigned layers = geom.layers;
    if (!geom.unrotated && layers > 1 && !map->layer_rot) return F110_ERR_INVALID;     // as f110_scan_layers
    if (layers > 1 && !sim->env_layer) return F110_ERR_INVALID;
    RenderK p;
    memset(&p, 0, sizeof(p));
    p.state = sim->state;
    p.env_layer = layers > 1 ? sim->env_layer : nullptr;
    p.agent_ids = agent_ids;
    p.dt = map->dt;
    p.layer_geom = het ? map->layer_geom : nullptr;
    p.layer_res = het ? map->layer_res : nullptr;
    p.layer_rot = het ? map->layer_rot : nullptr;
    p.out = out;
    p.orig = make_double2(map->orig_x, map->orig_y);
    p.ext = make_double2(map->width * map->resolution, map->height * map->resolution);    // make_view's x_max / y_max
    p.rot = make_double2(map->orig_c, map->orig_s);
    p.res = map->resolution;
    p.length = sim->sim_length; p.width = sim->sim_width;
    p.half = metres_per_pixel * 0.5; p.fwd = forward_offset;
    p.layer_stride = (unsigned long long)map->width * (unsigned long long)map->height;
    p.map_w = (unsigned)map->width; p.map_h = (unsigned)map->height;
    p.num_layers = layers;
    p.NA = sim->num_envs * sim->num_agents; p.A = sim->num_agents;
    p.V = V; p.H = height; p.W = width; p.heading_up = heading_up ? 1 : 0;
    if (obst) {
        ObstPlan ob;
        if ((rc = plan_obstacles(sim, obst, -1, &ob))) return rc;
        p.boxes = obst->boxes; p.active = obst->active; p.K = obst->per_env;
    }
    const unsigned long long tiles = ((unsigned long long)height * (unsigned long long)width + F110_RENDER_PIXELS - 1) /
                                     F110_RENDER_PIXELS;
    const dim3 grid((unsigned)tiles, (unsigned)(V < 65535 ? V : 65535)), block(F110_RENDER_THREADS);
    k_render_views<<<grid, block, 0, (cudaStream_t)stream>>>(p);
    LAUNCH_CHECK("k_render_views");
    return F110_OK;
}

int f110_vehicle_dynamics_st(const double *x, const double *u, const double *params, int32_t M, double *f, void *stream) {
    if (!x || !u || !params || !f || M <= 0) return F110_ERR_INVALID;
    k_rhs<<<(M + 127) / 128, 128, 0, (cudaStream_t)stream>>>(x, u, params, M, f);
    LAUNCH_CHECK("k_rhs");
    return F110_OK;
}

int f110_vehicle_dynamics_ks(const double *x, const double *u, const double *params, int32_t M, double *f, void *stream) {
    if (!x || !u || !params || !f || M <= 0) return F110_ERR_INVALID;
    k_rhs_ks<<<(M + 127) / 128, 128, 0, (cudaStream_t)stream>>>(x, u, params, M, f);
    LAUNCH_CHECK("k_rhs_ks");
    return F110_OK;
}

int f110_pid(const double *in, const double *params, int32_t M, double *out, void *stream) {
    if (!in || !params || !out || M <= 0) return F110_ERR_INVALID;
    k_pid<<<(M + 127) / 128, 128, 0, (cudaStream_t)stream>>>(in, params, M, out);
    LAUNCH_CHECK("k_pid");
    return F110_OK;
}

int f110_get_vertices(const double *poses, double length, double width, int32_t M, double *out, void *stream) {
    if (!poses || !out || M <= 0) return F110_ERR_INVALID;
    k_vertices<<<(M + 127) / 128, 128, 0, (cudaStream_t)stream>>>(poses, length, width, M, out);
    LAUNCH_CHECK("k_vertices");
    return F110_OK;
}

int f110_collision(const double *va, const double *vb, int32_t M, int32_t *out, void *stream) {
    if (!va || !vb || !out || M <= 0) return F110_ERR_INVALID;
    k_gjk<<<(M + 127) / 128, 128, 0, (cudaStream_t)stream>>>(va, vb, M, out);
    LAUNCH_CHECK("k_gjk");
    return F110_OK;
}

int f110_collision_multiple(const double *verts, int32_t M, int32_t n, double *collisions, double *collision_idx,
                            void *stream) {
    if (!verts || !collisions || !collision_idx || M <= 0 || n <= 0) return F110_ERR_INVALID;
    k_gjk_multiple<<<(M + 63) / 64, 64, 0, (cudaStream_t)stream>>>(verts, M, n, collisions, collision_idx);
    LAUNCH_CHECK("k_gjk_multiple");
    return F110_OK;
}

int f110_check_ttc(const f110_beams *beams, const double *scans, const double *vel, double ttc_thresh, int32_t M,
                   int32_t *out, void *stream) {
    int rc;
    if ((rc = check_beams(beams))) return rc;
    if (!scans || !vel || !out || M <= 0) return F110_ERR_INVALID;
    k_check_ttc<<<((long long)M * 32 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(make_view(beams), scans, vel,
                                                                                   ttc_thresh, M, out);
    LAUNCH_CHECK("k_check_ttc");
    return F110_OK;
}

int f110_ray_cast(const f110_beams *beams, const double *poses, const double *opp_vertices, int32_t M, float *scans,
                  int32_t *window, void *stream) {
    int rc;
    if ((rc = check_beams(beams))) return rc;
    if (!poses || !opp_vertices || !scans || M <= 0) return F110_ERR_INVALID;
    k_ray_cast<<<((long long)M * 32 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(make_view(beams), poses, opp_vertices,
                                                                                  M, scans, window);
    LAUNCH_CHECK("k_ray_cast");
    return F110_OK;
}

int f110_pure_pursuit(const double *wx, const double *wy, const double *wv, int32_t num_waypoints, const double *pose_x,
                      const double *pose_y, const double *pose_theta, int32_t M, double lookahead_distance, double vgain,
                      double wheelbase, double max_reacquire, double *actions_out, void *stream) {
    if (!wx || !wy || !wv || num_waypoints < 2 || !pose_x || !pose_y || !pose_theta || M <= 0 || !actions_out)
        return F110_ERR_INVALID;
    k_pure_pursuit<<<((long long)M * 32 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
        wx, wy, wv, num_waypoints, nullptr, nullptr, pose_x, pose_y, pose_theta, M, lookahead_distance, vgain, wheelbase,
        max_reacquire, actions_out);
    LAUNCH_CHECK("k_pure_pursuit");
    return F110_OK;
}

int f110_pure_pursuit_tables(const double *wx, const double *wy, const double *wv, const int32_t *table_start,
                             int32_t num_tables, const int32_t *pose_table, const double *pose_x, const double *pose_y,
                             const double *pose_theta, int32_t M, double lookahead_distance, double vgain, double wheelbase,
                             double max_reacquire, double *actions_out, void *stream) {
    if (!wx || !wy || !wv || !table_start || num_tables <= 0 || !pose_table || !pose_x || !pose_y || !pose_theta || M <= 0 ||
        !actions_out)
        return F110_ERR_INVALID;
    k_pure_pursuit<<<((long long)M * 32 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
        wx, wy, wv, 0, table_start, pose_table, pose_x, pose_y, pose_theta, M, lookahead_distance, vgain, wheelbase,
        max_reacquire, actions_out);
    LAUNCH_CHECK("k_pure_pursuit");
    return F110_OK;
}

static bool track_ok(const f110_track *track) {
    return track && track->num_tables >= 1 && track->min_segments >= 3 && track->table_start && track->segments;
}

int f110_track_project(const f110_track *track, const double *poses, const int32_t *table_ids, int32_t M, double *out,
                       void *stream) {
    if (!track_ok(track) || !poses || !out || M < 1 || (!table_ids && track->num_tables > 1)) return F110_ERR_INVALID;
    k_track_project<<<(unsigned)(((long long)M * 32 + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        track->segments, track->table_start, track->num_tables, poses, table_ids, M, out);
    LAUNCH_CHECK("k_track_project");
    return F110_OK;
}

int f110_track_progress(const f110_sim *sim, const f110_track *track, f110_progress *progress, void *stream) {
    if (!sim || !track_ok(track) || !progress || !sim->state || !sim->steer_cnt) return F110_ERR_INVALID;
    const f110_progress &g = *progress;
    if (!g.seg || !g.s || !g.d || !g.heading_error || !g.progress || !g.delta) return F110_ERR_INVALID;
    if (g.back < 0 || g.fwd < 0 || (long long)g.back + g.fwd + 1 > F110_TRACK_MAX_WINDOW) return F110_ERR_INVALID;
    if (!isfinite(g.reacquire_dist) || !(g.reacquire_dist > 0.0)) return F110_ERR_INVALID;
    if (sim->num_envs <= 0 || sim->num_agents <= 0 || (long long)sim->num_envs * sim->num_agents > 0x7fffffffll)
        return F110_ERR_INVALID;
    TrackK p;
    p.state = sim->state; p.steer_cnt = sim->steer_cnt; p.env_layer = sim->env_layer;
    p.segments = track->segments; p.table_start = track->table_start;
    p.seg = g.seg; p.s = g.s; p.d = g.d; p.e = g.heading_error; p.progress = g.progress; p.delta = g.delta;
    p.reacquire_dist = g.reacquire_dist;
    p.num_tables = track->num_tables;
    p.NA = sim->num_envs * sim->num_agents; p.A = sim->num_agents;
    p.back = g.back; p.window = g.back + g.fwd + 1;
    k_track_progress<<<(unsigned)(((long long)p.NA * 32 + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p);
    LAUNCH_CHECK("k_track_progress");
    return F110_OK;
}

int f110_track_progress_sum(const f110_sim *sim, const f110_track *track, f110_progress *progress, double *delta_sum,
                            int32_t restart, void *stream) {
    int rc;
    if (!delta_sum) return F110_ERR_INVALID;
    if ((rc = f110_track_progress(sim, track, progress, stream))) return rc;
    const int NA = sim->num_envs * sim->num_agents;
    k_delta_sum<<<(NA + 255) / 256, 256, 0, (cudaStream_t)stream>>>(progress->delta, delta_sum, NA, restart);
    LAUNCH_CHECK("k_delta_sum");
    return F110_OK;
}

int f110_edt(const uint8_t *occupied, int32_t height, int32_t width, double resolution, int32_t *scratch, double *dt_out,
             int64_t *k_out, void *stream) {
    if (!occupied || !scratch || !dt_out || height <= 0 || width <= 0 || !(resolution > 0)) return F110_ERR_INVALID;
    if ((size_t)width * sizeof(int32_t) > 200 * 1024) return F110_ERR_INVALID;      // one row of g must fit in shared memory
    cudaStream_t st = (cudaStream_t)stream;
    k_edt_columns<<<(width + 127) / 128, 128, 0, st>>>(occupied, height, width, scratch);
    LAUNCH_CHECK("k_edt_columns");
    const size_t smem = (size_t)width * sizeof(int32_t);
    if (smem > 48 * 1024)
        CUDA_TRY(cudaFuncSetAttribute(k_edt_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_edt_rows<<<height, 256, smem, st>>>(scratch, height, width, resolution, dt_out, k_out);
    LAUNCH_CHECK("k_edt_rows");
    return F110_OK;
}

int f110_rasterize_track(const double *segments, int32_t num_segments, double wall_inner, double wall_outer, int32_t height,
                          int32_t width, uint8_t *occupied, double *dist2_out, void *stream) {
    if (!segments || !occupied || num_segments <= 0 || height <= 0 || width <= 0 || !(wall_inner >= 0) ||
        !(wall_outer >= wall_inner))
        return F110_ERR_INVALID;
    const size_t smem = (size_t)num_segments * 5 * sizeof(double);
    if (smem > 200 * 1024) return F110_ERR_INVALID;
    if (smem > 48 * 1024)
        CUDA_TRY(cudaFuncSetAttribute(k_rasterize_track, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 block(32, 8), grid((width + 31) / 32, (height + 7) / 8);
    k_rasterize_track<<<grid, block, smem, (cudaStream_t)stream>>>(segments, num_segments, wall_inner * wall_inner,
                                                                    wall_outer * wall_outer, height, width, occupied, dist2_out);
    LAUNCH_CHECK("k_rasterize_track");
    return F110_OK;
}

int f110_pack_scans_u24(const float *scans, int64_t count, uint8_t *out, void *stream) {
    if (!scans || !out || count <= 0) return F110_ERR_INVALID;
    const long long groups = (count + 3) / 4;
    k_pack_u24<<<(unsigned)((groups + 255) / 256), 256, 0, (cudaStream_t)stream>>>(scans, (long long)count, out);
    LAUNCH_CHECK("k_pack_u24");
    return F110_OK;
}

int f110_scan_noise(float *scans, int64_t count, double std_dev, uint64_t seed, uint64_t offset, void *stream) {
    if (!scans || count <= 0) return F110_ERR_INVALID;
    k_scan_noise<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(scans, count, std_dev, seed, offset);
    LAUNCH_CHECK("k_scan_noise");
    return F110_OK;
}

}  // extern "C"
