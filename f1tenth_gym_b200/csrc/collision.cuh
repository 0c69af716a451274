// collision.cuh — car-body vertices and GJK overlap test of two convex 4-gons, fp64.
//
// Behavioural spec: reference gym/f110_gym/envs/collision_models.py:34-260.  GJK is kept as GJK
// (same support/simplex logic, same 1e3 iteration cap counted only on the triangle branch) rather
// than replaced by SAT so that boundary cases resolve the same way as the reference.
#pragma once
#include <math.h>

namespace f110 {

// collision_models.py:218-260 get_trmtx + get_vertices -> (rl, rr, fr, fl), v[2*i] = x, v[2*i+1] = y
// (cos, sin of the yaw are passed in: k_dynamics computes them once per agent and tick)
__device__ __forceinline__ void get_vertices_cs(double px, double py, double c, double s, double length, double width,
                                                double v[8]) {
    const double hl = length / 2, hw = width / 2;
    const double lx[4] = { -hl, -hl, hl, hl };
    const double ly[4] = { hw, -hw, -hw, hw };
#pragma unroll
    for (int i = 0; i < 4; i++) {
        v[2 * i] = (c * lx[i] + (-s) * ly[i]) + px;
        v[2 * i + 1] = (s * lx[i] + c * ly[i]) + py;
    }
}

// an obstacle slot (f110_obstacles.boxes row, active byte) takes part only when it is active, its pose is finite and its size finite and > 0
__device__ __forceinline__ bool box_present(const double *b, uint8_t act) {
    return act && isfinite(b[0]) && isfinite(b[1]) && isfinite(b[2]) && isfinite(b[3]) && isfinite(b[4]) && b[3] > 0.0 &&
           b[4] > 0.0;
}

__device__ __forceinline__ void get_vertices(double px, double py, double th, double length, double width,
                                             double v[8]) {
    double c = cos(th), s = sin(th);
    const double hl = length / 2, hw = width / 2;
    const double lx[4] = { -hl, -hl, hl, hl };
    const double ly[4] = { hw, -hw, -hw, hw };
#pragma unroll
    for (int i = 0; i < 4; i++) {
        v[2 * i] = (c * lx[i] + (-s) * ly[i]) + px;
        v[2 * i + 1] = (s * lx[i] + c * ly[i]) + py;
    }
}

// collision_models.py:81-92 indexOfFurthestPoint (np.argmax: first maximum)
__device__ __forceinline__ int furthest(const double v[8], double dx, double dy) {
    int best = 0;
    double bv = v[0] * dx + v[1] * dy;
#pragma unroll
    for (int i = 1; i < 4; i++) {
        double t = v[2 * i] * dx + v[2 * i + 1] * dy;
        if (t > bv) { bv = t; best = i; }
    }
    return best;
}

// collision_models.py:95-110 support
__device__ __forceinline__ void support(const double v1[8], const double v2[8], double dx, double dy,
                                        double &ox, double &oy) {
    int i = furthest(v1, dx, dy);
    int j = furthest(v2, -dx, -dy);
    ox = v1[2 * i] - v2[2 * j];
    oy = v1[2 * i + 1] - v2[2 * j + 1];
}

// collision_models.py:51-64 tripleProduct(a, b, c) = b*(a.c) - a*(b.c)
__device__ __forceinline__ void triple(double ax, double ay, double bx, double by, double cx, double cy,
                                       double &ox, double &oy) {
    double ac = ax * cx + ay * cy;
    double bc = bx * cx + by * cy;
    ox = bx * ac - ax * bc;
    oy = by * ac - ay * bc;
}

// collision_models.py:113-182 collision
__device__ __noinline__ bool gjk_collision(const double v1[8], const double v2[8]) {
    int index = 0;
    double sx[3], sy[3];
    double p1x = (v1[0] + v1[2] + v1[4] + v1[6]) / 4, p1y = (v1[1] + v1[3] + v1[5] + v1[7]) / 4;
    double p2x = (v2[0] + v2[2] + v2[4] + v2[6]) / 4, p2y = (v2[1] + v2[3] + v2[5] + v2[7]) / 4;
    double dx = p1x - p2x, dy = p1y - p2y;
    if (dx == 0 && dy == 0) dx = 1.0;
    double ax, ay;
    support(v1, v2, dx, dy, ax, ay);
    sx[0] = ax; sy[0] = ay;
    if (dx * ax + dy * ay <= 0) return false;
    dx = -ax; dy = -ay;
    int iter_count = 0;
    while (iter_count < 1000) {
        support(v1, v2, dx, dy, ax, ay);
        index += 1;
        if (index == 1) { sx[1] = ax; sy[1] = ay; } else { sx[2] = ax; sy[2] = ay; }
        if (dx * ax + dy * ay <= 0) return false;
        double aox = -ax, aoy = -ay;
        if (index < 2) {
            double abx = sx[0] - ax, aby = sy[0] - ay;
            triple(abx, aby, aox, aoy, abx, aby, dx, dy);
            if (sqrt(dx * dx + dy * dy) < 1e-10) { dx = aby; dy = -1 * abx; }   // perpendicular(ab) :34-48
            continue;
        }
        double abx = sx[1] - ax, aby = sy[1] - ay;
        double acx = sx[0] - ax, acy = sy[0] - ay;
        double px, py;
        triple(abx, aby, acx, acy, acx, acy, px, py);       // acperp
        if (px * aox + py * aoy >= 0) {
            dx = px; dy = py;
        } else {
            triple(acx, acy, abx, aby, abx, aby, px, py);   // abperp
            if (px * aox + py * aoy < 0) return true;
            sx[0] = sx[1]; sy[0] = sy[1];
            dx = px; dy = py;
        }
        sx[1] = sx[2]; sy[1] = sy[2];
        index -= 1;
        iter_count += 1;
    }
    return false;
}

}  // namespace f110
