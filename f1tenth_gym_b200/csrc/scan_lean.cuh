// scan_lean.cuh — k_scan_lean: the stand-alone scan (ScanSimulator2D.scan without noise, laser_models.py:148-186, 429-454) of
// M arbitrary poses, each on its own layer of any map f110_step accepts (f110_scan_layers).
//
// One warp per 32-beam item of one pose, over a plain grid: a stand-alone scan has no previous tick whose costs could order a
// queue, and no per-agent record.  At the start of an item the warp loads the pose and its layer id, that layer's geometry
// (origin, own extent, (res_l, RN(1/res_l)), rotation; the struct's values on a single map or a same-size stack), and then
// every lane computes what k_dynamics computes once per agent for the tick: the LUT index of beam 0 as Q16.48 and the first
// lookup.  The per-lookup arithmetic is the tick kernel's for that map kind, one instance per kind:
//   UNITS_CELLS   fast_path maps and cell canvases: k_march_lean<CELLS> / k_march_lean_het<CELLS> on dt_cells_pad, with the
//                 layer origin in cells;
//   UNITS_METRES  the FMA-corrected quotient, the magic-number floor and the layer's own extent test of k_march_lean_het_res
//                 (the canvas x_max is not the layer's: march_het.cuh);
//   UNITS_ROT     the reference-ordered __dmul_rn / __dadd_rn rotation of k_march_lean_rot.
// Beam headings are the Q16.48 index with guard32 and the replay (march_lean.cuh), so every beam takes the reference's
// sequential walk.  Poses at absurd coordinates (k_dynamics' `sane` bound), and every pose of a map whose origin, extent or
// ray reach breaks step_impl's half-bound rule, take the literal trace_ray<false> with the row count on the layer's geometry,
// as march_generic_rot does; unlike it, scan_generic returns its lookup count, which the oracle's nlook includes.
// A layer id outside [0, num_layers) writes NaN to its pose's beams, reads no table and counts no lookup.
// There is no global state: two calls on two streams may run at once.
#pragma once
#include "march_rot.cuh"

namespace f110 {

#define F110_SCAN_UNITS_CELLS 0
#define F110_SCAN_UNITS_METRES 1
#define F110_SCAN_UNITS_ROT 2
#define F110_SCAN_THREADS 256

struct ScanLeanK {
    const double *__restrict__ table;       // CELLS: [L][(H+1)*(W+1)] dt_cells_pad; else [L][H*W] dt in metres
    const double *__restrict__ dt;          // [L][H*W] dt in metres (literal path)
    const double2 *__restrict__ sincos2;    // [2 * theta_dis] (sin, cos), the LUT stored twice
    const double *__restrict__ poses;       // [M][3]
    const int32_t *__restrict__ layer_ids;  // [M], or NULL: layer 0
    float *__restrict__ out_f32;            // [M][B] or NULL
    double *__restrict__ out_f64;           // [M][B] or NULL
    unsigned long long *lookup_counter;     // COUNT only
    // canvas stack: per-layer tables (f110_map.layer_geom / layer_res / layer_rot), or NULL: the values below
    const double *__restrict__ layer_geom;
    const double *__restrict__ layer_res;
    const double *__restrict__ layer_rot;
    double2 orig, ext, res, rot;            // (orig_x, orig_y), (W res, H res), (res, RN(1 / res)), (orig_c, orig_s)
    double tmax;                            // CELLS: max_range / res; else max_range
    double max_range, eps, fov, theta_dis_f, inc;
    double inv_res_fine;                    // 1 / finest resolution: the absurd-coordinate bound of k_dynamics
    unsigned long long inc_fx;              // theta_index_increment in Q16.48
    unsigned long long table_stride;        // elements between layers of `table`
    unsigned long long dt_stride;           // elements between layers of `dt`
    unsigned guard32;
    unsigned width, height, last;           // canvas; `last` = width * height - 1 (the metre table's dt[-1,-1])
    unsigned ipa;                           // items per pose: ceil(B / 32)
    unsigned long long items;               // M * ipa
    unsigned num_layers;                    // >= 1
    int B;
    int literal;                            // 1: every pose takes the literal path (half-bound rule broken)
};

// the literal reference arithmetic (k_raymarch's trace_ray<false>) on one layer, out of line, with its lookup count
__device__ __noinline__ double scan_generic(const double *dt, double2 orig, double2 rot, double2 ext, double res, double dt_oob,
                                            double eps, double max_range, int width, int height, double px, double py,
                                            double s, double c, unsigned *n_out) {
    MapView m;
    m.dt = dt; m.orig_x = orig.x; m.orig_y = orig.y; m.orig_c = rot.x; m.orig_s = rot.y; m.resolution = res;
    m.x_max = ext.x; m.y_max = ext.y; m.dt_oob = dt_oob; m.eps = eps; m.max_range = max_range;
    m.width = width; m.height = height;
    int n;
    const double r = trace_ray<false>(m, px, py, s, c, n);
    *n_out = (unsigned)n;
    return r;
}

template <int UNITS, bool COUNT>
__global__ void __launch_bounds__(F110_SCAN_THREADS) k_scan_lean(const ScanLeanK p) {
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long item = ((unsigned long long)blockIdx.x * F110_SCAN_THREADS + threadIdx.x) >> 5;
    unsigned n = 0;
    if (item < p.items) {
        const unsigned m = (unsigned)(item / p.ipa);
        const int i = (int)((unsigned)(item - (unsigned long long)m * p.ipa) * 32u + lane);
        // the pose and its layer (warp-uniform loads, once per item)
        const double px = __ldg(p.poses + 3 * (size_t)m), py = __ldg(p.poses + 3 * (size_t)m + 1);
        const double yaw = __ldg(p.poses + 3 * (size_t)m + 2);
        const unsigned l = p.layer_ids ? (unsigned)__ldg(p.layer_ids + m) : 0u;
        double range;
        if (l >= p.num_layers) {
            range = __longlong_as_double(0x7ff8000000000000ll);     // NaN: no such layer
        } else if (i < p.B) {
            double2 lorig = p.orig, lmax = p.ext, lres = p.res, lrot = p.rot;
            if (p.layer_geom) {
                lorig = __ldg(reinterpret_cast<const double2 *>(p.layer_geom + 6 * (size_t)l));
                lmax = __ldg(reinterpret_cast<const double2 *>(p.layer_geom + 6 * (size_t)l) + 1);
                if (p.layer_res) lres = __ldg(reinterpret_cast<const double2 *>(p.layer_res) + l);
                if (UNITS == F110_SCAN_UNITS_ROT) lrot = __ldg(reinterpret_cast<const double2 *>(p.layer_rot) + l);
            }
            const double ti0 = theta_index0(yaw, p.fov, p.theta_dis_f);
            // k_dynamics' `sane`: coordinates whose cell index stays below 2^31 along every ray (derivation there)
            const bool sane = !p.literal && (UNITS == F110_SCAN_UNITS_ROT ? (fabs(px) + fabs(py)) * p.inv_res_fine < 1e9
                                                                          : fabs(px) * p.inv_res_fine < 1e9 &&
                                                                            fabs(py) * p.inv_res_fine < 1e9);
            if (sane) {
                const unsigned long long vfx = __double2ull_rd(ti0 * 281474976710656.0) + (unsigned long long)(unsigned)i * p.inc_fx;
                unsigned ti = (unsigned)(vfx >> F110_FX_SHIFT);
                const unsigned fr = (unsigned)(vfx >> (F110_FX_SHIFT - 32));
                if (fr + p.guard32 <= 2u * p.guard32) ti = (unsigned)replay_theta_index(ti0, i, p.inc, p.theta_dis_f);
                const double2 sc = __ldg(p.sincos2 + ti);
                const double *__restrict__ table = p.table + (unsigned long long)l * p.table_stride;
                const double MAGIC = 6755399441055744.0;   // 2^52 + 2^51: round-down add == floor in the low word
                double T, D;
                if (UNITS == F110_SCAN_UNITS_CELLS) {
                    const double ox = lorig.x * p.res.y, oy = lorig.y * p.res.y;     // exact: res = 2^-k
                    double X = px * p.res.y, Y = py * p.res.y;
                    unsigned c = (unsigned)__double2loint(__dadd_rd(X - ox, MAGIC));
                    unsigned r = (unsigned)__double2loint(__dadd_rd(Y - oy, MAGIC));
                    // off the layer -> its padding on the canvas (or the extra row / column), which holds dt[-1,-1]
                    D = __ldg(table + min(r, p.height) * (p.width + 1u) + min(c, p.width));
                    T = D;
                    n = 1;
                    if (__double2hiint(D) != 0 && T <= p.tmax) {
#pragma unroll 1
                        do {
                            X = X + D * sc.y;
                            Y = Y + D * sc.x;
                            c = (unsigned)__double2loint(__dadd_rd(X - ox, MAGIC));
                            r = (unsigned)__double2loint(__dadd_rd(Y - oy, MAGIC));
                            D = __ldg(table + min(r, p.height) * (p.width + 1u) + min(c, p.width));
                            T = T + D;
                            n++;
                        } while (__double2hiint(D) != 0 && T <= p.tmax);
                    }
                    range = ((T > p.tmax) ? p.tmax : T) * p.res.x;
                } else {
                    double X = px, Y = py;
                    n = 0;
                    for (;;) {
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
                        T = (n == 0) ? D : T + D;
                        n++;
                        if (!(__double2hiint(D) != 0 && T <= p.tmax)) break;
                        X = X + D * sc.y;
                        Y = Y + D * sc.x;
                    }
                    range = (T > p.tmax) ? p.tmax : T;
                }
            } else {
                // absurd coordinates: the literal reference arithmetic on the layer's geometry, rotation and row count
                const size_t lo = (size_t)l * (size_t)p.dt_stride;
                const int ti = beam_theta_index(ti0, i, p.inc, p.theta_dis_f, 1e-6);
                const double2 sc = __ldg(p.sincos2 + ti);
                range = scan_generic(p.dt + lo, lorig, UNITS == F110_SCAN_UNITS_ROT ? lrot : make_double2(1.0, 0.0), lmax,
                                     lres.x, __ldg(p.dt + lo + p.last), p.eps, p.max_range, (int)p.width, (int)p.height, px, py,
                                     sc.x, sc.y, &n);
            }
        }
        if (i < p.B) {
            const size_t o = (size_t)m * (size_t)p.B + (size_t)i;
            if (p.out_f32) p.out_f32[o] = (float)range;
            if (p.out_f64) p.out_f64[o] = range;
        }
    }
    if (COUNT) {
        const unsigned nsum = __reduce_add_sync(0xffffffffu, n);
        if (lane == 0 && nsum) atomicAdd(p.lookup_counter, (unsigned long long)nsum);
    }
}

}  // namespace f110
