// edt.cuh — exact Euclidean distance transform on the device (SURVEY.md 8f row 3; load-time, not per tick).
//
// Behavioural spec: reference laser_models.py:40-53 get_dt = resolution * scipy.ndimage.distance_transform_edt
// (bitmap): for every non-zero cell the Euclidean distance (in cells) to the nearest zero cell.  The squared
// distance is an integer; scipy returns sqrt of it in fp64, so `resolution * sqrt((double)k)` with the exact
// integer k reproduces the reference table bit for bit (checked against scipy on all bundled maps).
//   pass 1 (thread per column): g[r][c] = vertical distance to the nearest obstacle in column c (two sweeps)
//   pass 2 (block per row):     k[r][c] = min over c' of (c - c')^2 + g[r][c']^2   (exhaustive: O(W^2) per row;
//                               4.1e9 integer candidates for 1600x1600 on the GPU, replacing a 1-1.5 s
//                               host EDT; no lower-envelope bookkeeping, hence trivially exact)
#pragma once
#include <stdint.h>

namespace f110 {

#define F110_EDT_NONE 0x7fffffff      // no obstacle in this column

__global__ void k_edt_columns(const uint8_t *__restrict__ occupied, int H, int W, int32_t *__restrict__ g) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= W) return;
    int32_t d = F110_EDT_NONE;
    for (int r = 0; r < H; r++) {
        if (occupied[(size_t)r * W + c]) d = 0;
        else if (d != F110_EDT_NONE) d++;
        g[(size_t)r * W + c] = d;
    }
    d = F110_EDT_NONE;
    for (int r = H - 1; r >= 0; r--) {
        if (occupied[(size_t)r * W + c]) d = 0;
        else if (d != F110_EDT_NONE) d++;
        const int32_t up = g[(size_t)r * W + c];
        if (d < up) g[(size_t)r * W + c] = d;
    }
}

__global__ void __launch_bounds__(256) k_edt_rows(const int32_t *__restrict__ g, int H, int W, double resolution,
                                                  double *__restrict__ dt, int64_t *__restrict__ k_out) {
    extern __shared__ int32_t sg[];     // g[r][0..W)
    const int r = blockIdx.x;
    for (int c = threadIdx.x; c < W; c += blockDim.x) sg[c] = g[(size_t)r * W + c];
    __syncthreads();
    for (int c = threadIdx.x; c < W; c += blockDim.x) {
        unsigned long long best = ~0ull;
        for (int cc = 0; cc < W; cc++) {
            const int32_t gv = sg[cc];
            if (gv == F110_EDT_NONE) continue;
            const long long dx = (long long)(c - cc);
            const unsigned long long k = (unsigned long long)(dx * dx) + (unsigned long long)((long long)gv * gv);
            if (k < best) best = k;
        }
        // a map without any obstacle has no defined transform; report 0 there (scipy's result is unspecified)
        if (best == ~0ull) best = 0;
        dt[(size_t)r * W + c] = resolution * sqrt((double)best);
        if (k_out) k_out[(size_t)r * W + c] = (int64_t)best;
    }
}

}  // namespace f110
