// march_rot.cuh — k_march_lean_rot: the lean ray march for maps whose yaml origin has a yaw (orig_c, orig_s) != (1, 0):
// one such map alone, or a canvas stack that holds such maps (f110_map.layer_rot).
//
// The metre loop of k_march_lean_het_res (march_het.cuh) with the layer's rotation loaded once per work item next to its
// origin, extent and resolution.  Each lookup does the reference's xy_2_rc (laser_models.py:71-84) in the reference's
// order, every product and sum rounded on its own (no FMA):
//     tx = X - ox; ty = Y - oy; xr = tx*c + ty*s; yr = -tx*s + ty*c
// then floor(RN(xr / res_l)) through the FMA-corrected quotient and the magic-number add, as the other metre loops.  Off the
// map is `c >= W || r >= H || xr >= x_max_l || yr >= y_max_l`: a negative xr (yr) floors to a negative column (row), i.e. a
// huge unsigned one, and -0.0 floors to column 0 and stays on the map, as `x_rot < 0` leaves it in the reference.  The
// canvas row stride and clamps are those of k_march_lean_het; a single map is a canvas of one layer whose geometry comes
// from the launch parameters (RotGeomK.layer_geom == NULL), so it needs no device tables beyond the map's own.
// Scan poses at absurd coordinates take march_generic_rot: the literal trace_ray<false> of lidar.cuh, which is what
// k_raymarch computes, with the rotation and the row count.
// A kernel of its own, so that the k_march_lean, k_march_lean_het and k_march_lean_het_res instances keep their code.
#pragma once
#include "march_het.cuh"

namespace f110 {

struct RotGeomK {
    const double *__restrict__ layer_geom;  // canvas stack: [L][6] (orig_x, orig_y, x_max, y_max, W_l, H_l); NULL: one map
    const double *__restrict__ layer_res;   // canvas stack: [L][2] (res_l, RN(1 / res_l))
    const double *__restrict__ layer_rot;   // canvas stack: [L][2] (orig_c_l, orig_s_l)
    const int32_t *__restrict__ env_layer;  // canvas stack: [num_envs]
    unsigned num_agents;
    // one map (layer_geom == NULL): its geometry, by value
    double2 orig, ext, res, rot;            // (orig_x, orig_y), (x_max, y_max), (res, RN(1 / res)), (orig_c, orig_s)
};

// absurd coordinates on a rotated map: the literal reference arithmetic (k_raymarch's trace_ray<false>), out of line, all
// arguments by value.  Unlike march_generic it carries the row count, so it is exact wherever the ray goes.
__device__ __noinline__ double march_generic_rot(const double *dt, double2 orig, double2 rot, double2 ext, double res,
                                                 double dt_oob, double eps, double max_range, int width, int height,
                                                 double px, double py, double s, double c) {
    MapView m;
    m.dt = dt; m.orig_x = orig.x; m.orig_y = orig.y; m.orig_c = rot.x; m.orig_s = rot.y; m.resolution = res;
    m.x_max = ext.x; m.y_max = ext.y; m.dt_oob = dt_oob; m.eps = eps; m.max_range = max_range;
    m.width = width; m.height = height;
    int n;
    return trace_ray<false>(m, px, py, s, c, n);
}

template <bool NOISE, bool COUNT, int PT, int MINB>
__global__ void __launch_bounds__(PT, MINB) k_march_lean_rot(const LeanK p, const RotGeomK g, const MarchQueue mq) {
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
        // the agent's map: origin, resolution and rotation (warp-uniform loads, once per item, on a canvas stack)
        double2 lorig = g.orig, lres = g.res, lrot = g.rot;
        unsigned l = 0u;
        if (g.layer_geom) {
            l = (unsigned)__ldg(g.env_layer + a / g.num_agents);
            lorig = __ldg(reinterpret_cast<const double2 *>(g.layer_geom + 6 * (size_t)l));
            lres = __ldg(reinterpret_cast<const double2 *>(g.layer_res) + l);      // (res_l, RN(1 / res_l))
            lrot = __ldg(reinterpret_cast<const double2 *>(g.layer_rot) + l);      // (orig_c_l, orig_s_l)
        }
        unsigned n = 0;
        if (i < p.B) {
            double range;
            const double2 lmax = g.layer_geom ? __ldg(reinterpret_cast<const double2 *>(g.layer_geom + 6 * (size_t)l) + 1) : g.ext;
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
                        // x_rot, y_rot as the reference rounds them: two products and a sum each, never fused
                        const double xr = __dadd_rn(__dmul_rn(tx, lrot.x), __dmul_rn(ty, lrot.y));
                        const double yr = __dadd_rn(__dmul_rn(-tx, lrot.y), __dmul_rn(ty, lrot.x));
                        double qx = xr * lres.y, qy = yr * lres.y;
                        qx = __fma_rn(__fma_rn(-qx, lres.x, xr), lres.y, qx);     // RN(xr / res_l), see march.cuh
                        qy = __fma_rn(__fma_rn(-qy, lres.x, yr), lres.y, qy);
                        const int c = __double2loint(__dadd_rd(qx, MAGIC));
                        const int r = __double2loint(__dadd_rd(qy, MAGIC));
                        unsigned idx = (unsigned)r * p.width + (unsigned)c;
                        if ((unsigned)c >= p.width || (unsigned)r >= p.height || xr >= lmax.x || yr >= lmax.y) idx = p.last;
                        D = __ldg(table + idx);
                        T = T + D;
                        n++;
                    } while (__double2hiint(D) != 0 && T <= p.tmax);
                }
                range = (T > p.tmax) ? p.tmax : T;
            } else {
                // absurd coordinates: the literal reference arithmetic on the map's geometry, rotation and row count
                const double2 r3 = __ldg(rp + 3);
                const size_t lo = (size_t)((unsigned long long)__double_as_longlong(r3.x) / p.layer_stride_lean * p.layer_stride);
                const int ti = beam_theta_index(r3.y, i, p.inc, p.theta_dis_f, 1e-6);
                const double2 sc = __ldg(p.sincos2 + ti);
                range = march_generic_rot(p.dt + lo, lorig, lrot, lmax, lres.x, __ldg(p.dt + lo + p.last), p.eps_m, p.max_range,
                                          (int)p.width, (int)p.height, r0.x, r0.y, sc.x, sc.y);
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
