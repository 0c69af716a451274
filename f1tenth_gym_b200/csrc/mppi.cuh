// mppi.cuh — f110_mppi_sample / f110_mppi_update (include/f110_mppi.h): the two steps of an MPPI planner around
// f110_predict_scored, on the device, without host synchronisation.
//
// k_mppi_sample  thread per (m, k, h): the restart check of agent m, the nominal step, two draws of normal_sample and the clamp.
//                The thread of k = 0 writes the reset nominal back; every thread of a restarted agent uses (0, 0) whatever it
//                reads, so the result does not depend on the order of that write and the other threads' reads.
// k_mppi_update  block per agent m: min over the finite costs (a block reduction; min is exact in any order), the weights in
//                shared memory, then each thread sums whole columns (h, c) over k in k order, so repeated runs are bit-identical;
//                the weighted means go to shared memory before any nominal row is overwritten.  The means U [H] lie at the base
//                of the dynamic shared memory and the weights [K] after them, so U's double2 accesses are aligned for any K.
#pragma once

namespace f110 {

#define F110_MPPI_SAMPLE_THREADS 256
#define F110_MPPI_UPDATE_THREADS 256
// k_mppi_update's shared memory: the dynamic H double2 + K doubles and the static reduction arrays (ptxas reports 128 bytes
// for them: each padded as a double array), within the 48 KiB a block gets without an opt-in at the largest K and H the header
// allows
static_assert((2 * F110_MPPI_MAX_H + F110_MPPI_MAX_K) * sizeof(double) +
              2 * (F110_MPPI_UPDATE_THREADS / 32) * sizeof(double) <= 48 * 1024,
              "k_mppi_update needs more than 48 KiB of shared memory at F110_MPPI_MAX_K / F110_MPPI_MAX_H");

struct MppiK {
    const int32_t *__restrict__ agent_ids;    // [M]
    double2 *__restrict__ nominal;            // [M][H]
    int64_t *__restrict__ iteration;          // [1]
    int32_t *__restrict__ no_finite;          // [M]
    double2 sigma, lo, hi;                    // (steer, speed)
    double lambda;
    uint64_t seed;
    int M, K, H;
};

__device__ __forceinline__ double mppi_clamp(double v, double lo, double hi) {
    return v < lo ? lo : (v > hi ? hi : v);
}

__global__ void __launch_bounds__(F110_MPPI_SAMPLE_THREADS) k_mppi_sample(const MppiK p, const int32_t *__restrict__ steer_cnt,
                                                                         const uint8_t *__restrict__ terminated,
                                                                         const uint8_t *__restrict__ truncated, int NA, int A,
                                                                         double2 *__restrict__ actions) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)p.M * p.K * p.H) return;
    const int h = (int)(idx % p.H);
    const long long mk = idx / p.H;
    const int k = (int)(mk % p.K);
    const int m = (int)(mk / p.K);
    const int a = __ldg(p.agent_ids + m);
    bool restarted = false;
    if (a >= 0 && a < NA) {
        restarted = steer_cnt[a] == 0;
        if (terminated) restarted = restarted || terminated[a / A] != 0 || truncated[a / A] != 0;
    }
    double2 nom = make_double2(0.0, 0.0);
    if (!restarted) nom = p.nominal[(size_t)m * p.H + h];
    else if (k == 0) p.nominal[(size_t)m * p.H + h] = nom;
    double u0 = nom.x, u1 = nom.y;
    if (k != 0) {
        const uint64_t stream = (1ull << 63) | (uint64_t)*p.iteration;
        u0 = u0 + p.sigma.x * normal_sample(p.seed, stream, 2 * (uint64_t)idx);
        u1 = u1 + p.sigma.y * normal_sample(p.seed, stream, 2 * (uint64_t)idx + 1);
    }
    actions[idx] = make_double2(mppi_clamp(u0, p.lo.x, p.hi.x), mppi_clamp(u1, p.lo.y, p.hi.y));
}

__global__ void __launch_bounds__(F110_MPPI_UPDATE_THREADS) k_mppi_update(const MppiK p, const double2 *__restrict__ actions,
                                                                         const double *__restrict__ cost,
                                                                         double2 *__restrict__ action_out, int num_rows,
                                                                         double *__restrict__ weights_out,
                                                                         int32_t *__restrict__ argmin_out) {
    extern __shared__ double2 smem2[];
    double2 *U = smem2;                                      // [H], first: read as double2, so 16-byte aligned for any K
    double *w = reinterpret_cast<double *>(smem2 + p.H);     // [K]
    __shared__ double red_c[F110_MPPI_UPDATE_THREADS / 32];
    __shared__ int red_k[F110_MPPI_UPDATE_THREADS / 32];
    const int m = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double *c = cost + (size_t)m * p.K;
    // beta and the argmin: the smallest finite cost, its first k
    double bc = INFINITY;
    int bk = 0x7fffffff;
    for (int k = tid; k < p.K; k += F110_MPPI_UPDATE_THREADS) {
        const double v = c[k];
        if (isfinite(v) && v < bc) { bc = v; bk = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double oc = __shfl_xor_sync(0xffffffffu, bc, o);
        const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
        if (oc < bc || (oc == bc && ok < bk)) { bc = oc; bk = ok; }
    }
    if (lane == 0) { red_c[warp] = bc; red_k[warp] = bk; }
    __syncthreads();
    bc = red_c[0]; bk = red_k[0];
    for (int i = 1; i < F110_MPPI_UPDATE_THREADS / 32; i++)
        if (red_c[i] < bc || (red_c[i] == bc && red_k[i] < bk)) { bc = red_c[i]; bk = red_k[i]; }
    const bool any = bk != 0x7fffffff;
    const double beta = bc;
    for (int k = tid; k < p.K; k += F110_MPPI_UPDATE_THREADS) {
        const double v = c[k];
        const double wk = (any && isfinite(v)) ? exp(-(v - beta) / p.lambda) : 0.0;
        w[k] = wk;
        if (weights_out) weights_out[(size_t)m * p.K + k] = wk;
    }
    __syncthreads();
    // U[h] column by column: thread j takes (h, c) = (j / 2, j % 2), sums over k in order
    const double *A = reinterpret_cast<const double *>(actions) + (size_t)m * p.K * p.H * 2;
    for (int j = tid; j < 2 * p.H; j += F110_MPPI_UPDATE_THREADS) {
        double u;
        if (any) {
            double num = 0.0, den = 0.0;
            for (int k = 0; k < p.K; k++) {
                const double wk = w[k];
                den = den + wk;
                num = num + wk * __ldg(A + (size_t)k * p.H * 2 + j);
            }
            u = num / den;
        } else {
            const double v = reinterpret_cast<const double *>(p.nominal + (size_t)m * p.H)[j];
            u = (j & 1) ? mppi_clamp(v, p.lo.y, p.hi.y) : mppi_clamp(v, p.lo.x, p.hi.x);
        }
        reinterpret_cast<double *>(U)[j] = u;
    }
    __syncthreads();
    double2 *nom = p.nominal + (size_t)m * p.H;
    for (int h = tid; h < p.H; h += F110_MPPI_UPDATE_THREADS) nom[h] = U[h + 1 < p.H ? h + 1 : p.H - 1];
    if (tid == 0) {
        const int a = __ldg(p.agent_ids + m);
        if (a >= 0 && a < num_rows) action_out[a] = U[0];
        if (argmin_out) argmin_out[m] = any ? bk : -1;
        if (!any) p.no_finite[m] += 1;
        if (m == 0) *p.iteration += 1;
    }
}

}  // namespace f110
