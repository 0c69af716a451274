// march_het.cuh — k_march_lean_het: the lean ray march for a CANVAS STACK of maps that differ in size and origin
// (f110_map.layer_geom; multi-track batches such as berlin + vegas + skirk + levine).
//
// Same arithmetic, queue and per-agent record as k_march_lean<LAYERED> (march_lean.cuh), with the statically dealt queue
// and one entry per ticket; what differs is where the map geometry comes from.  Every layer sits in the low corner of its
// slice of one [Hc][Wc] canvas (Wc = max W_l, Hc = max H_l) and every other canvas cell holds that layer's dt[-1,-1], so
// the column / row clamps and the row stride stay the canvas' launch constants.  Per work item the kernel loads the layer
// of the agent's env once (layer_geom[env_layer[a / A]]):
//   * cell units: the origin in cells (ox, oy);
//   * metres: also the layer's own x_max = fl(W_l * res), y_max = fl(H_l * res).  The metre loop keeps both `c >= width`
//     and `tx >= x_max` because `tx >= fl(W * res)` is not the same predicate as `floor(RN(tx / res)) >= W`: the canvas
//     padding covers the first test, the second needs the layer's own bound.
// It is a separate kernel, not one more template argument of k_march_lean: the default instances keep their code and
// their mangled names (test_march_kernel_resource_budget), and the per-item constants live in registers here instead of
// the parameter bank, which needs its own register budget (launch bounds in launch_het, DESIGN.md §3.2).
#pragma once
#include "march_lean.cuh"

namespace f110 {

struct LayerGeomK {
    const double *__restrict__ layer_geom;  // [L][6] (orig_x, orig_y, x_max, y_max, W_l, H_l), metres
    const int32_t *__restrict__ env_layer;  // [num_envs]
    unsigned num_agents;
};

template <bool NOISE, bool COUNT, bool CELLS, int PT, int MINB>
__global__ void __launch_bounds__(PT, MINB) k_march_lean_het(const LeanK p, const LayerGeomK g, const MarchQueue mq) {
    __shared__ unsigned s_next;
    if (threadIdx.x == 0) s_next = 0u;
    pdl_wait();
    pdl_launch_dependents();
    __syncthreads();
    const unsigned lane = threadIdx.x & 31u;
    const unsigned nA = min(mq.count[0], mq.items), nB = min(mq.count[1], mq.items);
    const unsigned nAB = nA + nB;
    const unsigned total = min(nAB + min(mq.count[2], mq.items), mq.items);
    const unsigned cs = mq.chunk_shift;
    const unsigned qstride = gridDim.x << cs, qbase = blockIdx.x << cs, qmask = (1u << cs) - 1u;
    const unsigned s_next_addr = (unsigned)__cvta_generic_to_shared(&s_next);
    unsigned looks = 0u;
    for (;;) {
        unsigned k = 0, leader;
        asm volatile("{\n\t.reg .pred p;\n\telect.sync %1|p, 0xffffffff;\n\t@p atom.shared.add.u32 %0, [%2], 1;\n\t}"
                     : "+r"(k), "=r"(leader) : "r"(s_next_addr) : "memory");
        k = __shfl_sync(0xffffffffu, k, leader);
        const unsigned q = (k >> cs) * qstride + qbase + (k & qmask);
        if (q >= total) break;
        const unsigned it = mq.order[(q < nA) ? q : (q < nAB) ? (mq.items + (q - nA)) : (2u * mq.items + (q - nAB))];
        const unsigned a = it >> 8;
        const int i = (int)((it & 255u) * 32u + lane);
        const double2 *__restrict__ rp = p.rec + 4 * (size_t)a;
        const double2 r0 = __ldg(rp), r1 = __ldg(rp + 1);
        const unsigned long long ti0fx = (unsigned long long)__double_as_longlong(r1.y);
        // the agent's map layer: origin and extent (warp-uniform loads, once per item)
        const double *__restrict__ lg = g.layer_geom + 6 * (size_t)__ldg(g.env_layer + a / g.num_agents);
        const double2 lorig = __ldg(reinterpret_cast<const double2 *>(lg));
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
                const double *__restrict__ table = p.table + (unsigned long long)__double_as_longlong(__ldg(rp + 3).x);
                asm volatile("" : "+l"(table));
                const double MAGIC = 6755399441055744.0;   // 2^52 + 2^51: round-down add == floor in the low word
                double X = r0.x, Y = r0.y, T = r1.x, D = r1.x;
                n = 1;
                if (CELLS) {
                    const double ox = lorig.x * p.inv_res, oy = lorig.y * p.inv_res;     // exact: res = 2^-k
                    if (__double2hiint(D) != 0 && T <= p.tmax) {
#pragma unroll 1
                        do {
                            X = X + D * sc.y;
                            Y = Y + D * sc.x;
                            const unsigned c = (unsigned)__double2loint(__dadd_rd(X - ox, MAGIC));
                            const unsigned r = (unsigned)__double2loint(__dadd_rd(Y - oy, MAGIC));
                            // off the layer -> its padding on the canvas (or the extra row / column), which holds dt[-1,-1]
                            D = __ldg(table + min(r, p.height) * (p.width + 1u) + min(c, p.width));
                            T = T + D;
                            n++;
                        } while (__double2hiint(D) != 0 && T <= p.tmax);
                    }
                    range = ((T > p.tmax) ? p.tmax : T) * p.res;
                } else {
                    const double2 lmax = __ldg(reinterpret_cast<const double2 *>(lg) + 1);
                    if (__double2hiint(D) != 0 && T <= p.tmax) {
#pragma unroll 1
                        do {
                            X = X + D * sc.y;
                            Y = Y + D * sc.x;
                            const double tx = X - lorig.x, ty = Y - lorig.y;
                            double qx = tx * p.inv_res, qy = ty * p.inv_res;
                            qx = __fma_rn(__fma_rn(-qx, p.res, tx), p.inv_res, qx);     // RN(tx / res), see march.cuh
                            qy = __fma_rn(__fma_rn(-qy, p.res, ty), p.inv_res, qy);
                            const int c = __double2loint(__dadd_rd(qx, MAGIC));
                            const int r = __double2loint(__dadd_rd(qy, MAGIC));
                            unsigned idx = (unsigned)r * p.width + (unsigned)c;
                            if ((unsigned)c >= p.width || (unsigned)r >= p.height || tx >= lmax.x || ty >= lmax.y) idx = p.last;
                            D = __ldg(table + idx);
                            T = T + D;
                            n++;
                        } while (__double2hiint(D) != 0 && T <= p.tmax);
                    }
                    range = (T > p.tmax) ? p.tmax : T;
                }
            } else {
                // absurd coordinates (|x| >= 1e8 m): the literal reference arithmetic on the layer's geometry, out of line; the
                // canvas width is the row stride (the padding beyond the layer reads dt[-1,-1], as off the map)
                const double2 r3 = __ldg(rp + 3), lmax = __ldg(reinterpret_cast<const double2 *>(lg) + 1);
                const size_t lo = (size_t)((unsigned long long)__double_as_longlong(r3.x) / p.layer_stride_lean * p.layer_stride);
                const int ti = beam_theta_index(r3.y, i, p.inc, p.theta_dis_f, 1e-6);
                const double2 sc = __ldg(p.sincos2 + ti);
                range = march_generic(p.dt + lo, lorig.x, lorig.y, lmax.x, lmax.y, p.res, __ldg(p.dt + lo + p.last), p.eps_m,
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
    if (COUNT) {
        const unsigned nsum = __reduce_add_sync(0xffffffffu, looks);
        if (lane == 0 && nsum) atomicAdd(p.lookup_counter, (unsigned long long)nsum);
    }
}

// k_march_lean_het_res: a canvas stack whose layers also differ in resolution (f110_map.layer_res), metres only.  The metre
// loop of k_march_lean_het with the layer's own (res_l, RN(1/res_l)) in the quotient and in march_generic, loaded once per
// work item next to the origin and extent.  floor(RN(t / res_l)) through the FMA-corrected quotient is the reference's
// floor(t / res_l) at every resolution (test_boundary_inputs), so each layer keeps the single-map results.  A kernel of its
// own, not a template argument of k_march_lean_het, so that the existing instances keep their code and their names.
template <bool NOISE, bool COUNT, int PT, int MINB>
__global__ void __launch_bounds__(PT, MINB) k_march_lean_het_res(const LeanK p, const LayerGeomK g,
                                                                 const double *__restrict__ layer_res, const MarchQueue mq) {
    __shared__ unsigned s_next;
    if (threadIdx.x == 0) s_next = 0u;
    pdl_wait();
    pdl_launch_dependents();
    __syncthreads();
    const unsigned lane = threadIdx.x & 31u;
    const unsigned nA = min(mq.count[0], mq.items), nB = min(mq.count[1], mq.items);
    const unsigned nAB = nA + nB;
    const unsigned total = min(nAB + min(mq.count[2], mq.items), mq.items);
    const unsigned cs = mq.chunk_shift;
    const unsigned qstride = gridDim.x << cs, qbase = blockIdx.x << cs, qmask = (1u << cs) - 1u;
    const unsigned s_next_addr = (unsigned)__cvta_generic_to_shared(&s_next);
    unsigned looks = 0u;
    for (;;) {
        unsigned k = 0, leader;
        asm volatile("{\n\t.reg .pred p;\n\telect.sync %1|p, 0xffffffff;\n\t@p atom.shared.add.u32 %0, [%2], 1;\n\t}"
                     : "+r"(k), "=r"(leader) : "r"(s_next_addr) : "memory");
        k = __shfl_sync(0xffffffffu, k, leader);
        const unsigned q = (k >> cs) * qstride + qbase + (k & qmask);
        if (q >= total) break;
        const unsigned it = mq.order[(q < nA) ? q : (q < nAB) ? (mq.items + (q - nA)) : (2u * mq.items + (q - nAB))];
        const unsigned a = it >> 8;
        const int i = (int)((it & 255u) * 32u + lane);
        const double2 *__restrict__ rp = p.rec + 4 * (size_t)a;
        const double2 r0 = __ldg(rp), r1 = __ldg(rp + 1);
        const unsigned long long ti0fx = (unsigned long long)__double_as_longlong(r1.y);
        // the agent's map layer: origin, extent and resolution (warp-uniform loads, once per item)
        const unsigned l = (unsigned)__ldg(g.env_layer + a / g.num_agents);
        const double *__restrict__ lg = g.layer_geom + 6 * (size_t)l;
        const double2 lorig = __ldg(reinterpret_cast<const double2 *>(lg));
        const double2 lres = __ldg(reinterpret_cast<const double2 *>(layer_res) + l);     // (res_l, RN(1 / res_l))
        unsigned n = 0;
        if (i < p.B) {
            double range;
            const double2 lmax = __ldg(reinterpret_cast<const double2 *>(lg) + 1);
            if (ti0fx != ~0ull) {
                const unsigned long long vfx = ti0fx + (unsigned long long)(unsigned)i * p.inc_fx;
                unsigned ti = (unsigned)(vfx >> F110_FX_SHIFT);
                const unsigned fr = (unsigned)(vfx >> (F110_FX_SHIFT - 32));
                if (fr + p.guard32 <= 2u * p.guard32)
                    ti = (unsigned)replay_theta_index(__ldg(rp + 3).y, i, p.inc, p.theta_dis_f);
                const double2 sc = __ldg(p.sincos2 + ti);
                const double *__restrict__ table = p.table + (unsigned long long)__double_as_longlong(__ldg(rp + 3).x);
                asm volatile("" : "+l"(table));
                const double MAGIC = 6755399441055744.0;   // 2^52 + 2^51: round-down add == floor in the low word
                double X = r0.x, Y = r0.y, T = r1.x, D = r1.x;
                n = 1;
                if (__double2hiint(D) != 0 && T <= p.tmax) {
#pragma unroll 1
                    do {
                        X = X + D * sc.y;
                        Y = Y + D * sc.x;
                        const double tx = X - lorig.x, ty = Y - lorig.y;
                        double qx = tx * lres.y, qy = ty * lres.y;
                        qx = __fma_rn(__fma_rn(-qx, lres.x, tx), lres.y, qx);     // RN(tx / res_l), see march.cuh
                        qy = __fma_rn(__fma_rn(-qy, lres.x, ty), lres.y, qy);
                        const int c = __double2loint(__dadd_rd(qx, MAGIC));
                        const int r = __double2loint(__dadd_rd(qy, MAGIC));
                        unsigned idx = (unsigned)r * p.width + (unsigned)c;
                        if ((unsigned)c >= p.width || (unsigned)r >= p.height || tx >= lmax.x || ty >= lmax.y) idx = p.last;
                        D = __ldg(table + idx);
                        T = T + D;
                        n++;
                    } while (__double2hiint(D) != 0 && T <= p.tmax);
                }
                range = (T > p.tmax) ? p.tmax : T;
            } else {
                // absurd coordinates: the literal reference arithmetic on the layer's geometry and resolution (k_march_lean_het)
                const double2 r3 = __ldg(rp + 3);
                const size_t lo = (size_t)((unsigned long long)__double_as_longlong(r3.x) / p.layer_stride_lean * p.layer_stride);
                const int ti = beam_theta_index(r3.y, i, p.inc, p.theta_dis_f, 1e-6);
                const double2 sc = __ldg(p.sincos2 + ti);
                range = march_generic(p.dt + lo, lorig.x, lorig.y, lmax.x, lmax.y, lres.x, __ldg(p.dt + lo + p.last), p.eps_m,
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
    if (COUNT) {
        const unsigned nsum = __reduce_add_sync(0xffffffffu, looks);
        if (lane == 0 && nsum) atomicAdd(p.lookup_counter, (unsigned long long)nsum);
    }
}

}  // namespace f110
