// progress.cuh — projection of poses on closed centerlines (Frenet s, d, heading error) and the per-agent progress tracker.
//
// Behavioural spec of the projection: reference examples/waypoint_follow.py:16-47 nearest_point_on_trajectory on the closed
// polyline vstack(T, T[0]), in its operation order, fp64:
//   dot = fma(py - y_i, dy_i, (px - x_i) * dx_i);  t = dot / l2_i clamped to [0, 1];  q = (x_i + t * dx_i, y_i + t * dy_i);
//   ex = px - qx, ey = py - qy;  dist = sqrt(ex * ex + ey * ey);  the first minimum of dist wins.
// The one fused operation is the reference's own: its `np.dot(point - trajectory[i, :], diffs[i, :])` runs through BLAS ddot,
// which on x86-64 with FMA rounds (px - x) * dx and then fuses the second product into the sum.  With two separate roundings,
// 1057 of the 9600 reference t values of tests/golden/kat_progress.npz differ by an ulp, and one segment index differs; with
// this fma every seg, t and dist is equal.  Every other operation is rounded on its own (the library is built -fmad=false).
// Outputs: s = s_i + t * len_i;  d = +dist when dx_i * ey - dy_i * ex >= 0 (left of the direction of travel), else -dist;
// heading error e = yaw - h_i;  e = e - 2pi * floor((e + pi) / 2pi).  Nothing here evaluates a transcendental: the host
// precomputes every per-segment value (simulator.CenterlineTables).
//
// The per-segment arithmetic is k_pure_pursuit's (csrc/planner.cuh), but not shared with it: that kernel reads the waypoint
// columns and derives dx, dy, l2 itself, this one reads one precomputed 64-byte record per segment, and the tie order differs
// (window order here).  Keeping them apart leaves k_pure_pursuit's SASS as it is.
#pragma once
#include <math.h>
#include <stdint.h>

namespace f110 {

#define F110_TRACK_REC 8          // doubles per segment record: x, y, dx, dy, l2, s, len, heading
#define F110_TRACK_MAX_WINDOW 1024

struct TrackHit {
    double dist, t;
    int k;                        // window position of the first minimum, 0x7fffffff = none (every dist NaN)
};

// First minimum of dist over the window positions k = 0 .. W-1, segment i = (base + k) mod n (base in [0, n), W <= n).
// The whole warp calls it; every lane gets the result.
__device__ __forceinline__ TrackHit track_search(const double *__restrict__ rec, int n, int base, int W, double px, double py,
                                                 int lane) {
    double bd = INFINITY, bt = 0.0;
    int bk = 0x7fffffff;
    for (int k = lane; k < W; k += 32) {
        int i = base + k;
        if (i >= n) i -= n;
        const double2 *r = reinterpret_cast<const double2 *>(rec + (size_t)i * F110_TRACK_REC);
        const double2 xy = __ldg(r), dxy = __ldg(r + 1);
        const double l2 = __ldg(rec + (size_t)i * F110_TRACK_REC + 4);
        const double dot = __fma_rn(py - xy.y, dxy.y, (px - xy.x) * dxy.x);     // np.dot: see the top of this file
        double t = dot / l2;
        if (t < 0.0) t = 0.0;
        if (t > 1.0) t = 1.0;
        const double qx = xy.x + t * dxy.x, qy = xy.y + t * dxy.y;
        const double ex = px - qx, ey = py - qy;
        const double d = sqrt(ex * ex + ey * ey);
        if (d < bd) { bd = d; bt = t; bk = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double od = __shfl_xor_sync(0xffffffffu, bd, o);
        const double ot = __shfl_xor_sync(0xffffffffu, bt, o);
        const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
        if (od < bd || (od == bd && ok < bk)) { bd = od; bt = ot; bk = ok; }
    }
    TrackHit h;
    h.dist = bd; h.t = bt; h.k = bk;
    return h;
}

// track_search in one thread: the same per-segment statements over k = 0 .. W-1 in order, the first minimum kept.  For a
// caller whose lanes each track a pose of their own (k_scored_rollout).
__device__ __forceinline__ TrackHit track_search_thread(const double *__restrict__ rec, int n, int base, int W, double px,
                                                        double py) {
    double bd = INFINITY, bt = 0.0;
    int bk = 0x7fffffff;
    for (int k = 0; k < W; k++) {
        int i = base + k;
        if (i >= n) i -= n;
        const double2 *r = reinterpret_cast<const double2 *>(rec + (size_t)i * F110_TRACK_REC);
        const double2 xy = __ldg(r), dxy = __ldg(r + 1);
        const double l2 = __ldg(rec + (size_t)i * F110_TRACK_REC + 4);
        const double dot = __fma_rn(py - xy.y, dxy.y, (px - xy.x) * dxy.x);     // np.dot: see the top of this file
        double t = dot / l2;
        if (t < 0.0) t = 0.0;
        if (t > 1.0) t = 1.0;
        const double qx = xy.x + t * dxy.x, qy = xy.y + t * dxy.y;
        const double ex = px - qx, ey = py - qy;
        const double d = sqrt(ex * ex + ey * ey);
        if (d < bd) { bd = d; bt = t; bk = k; }
    }
    TrackHit h;
    h.dist = bd; h.t = bt; h.k = bk;
    return h;
}

struct TrackOut {
    double t, dist, s, d, e;
};

// Frenet outputs of a pose on segment i at parameter t (the values track_search compared, recomputed in the same order).
__device__ __forceinline__ TrackOut track_outputs(const double *__restrict__ rec, int i, double t, double px, double py,
                                                  double yaw) {
    const double *r = rec + (size_t)i * F110_TRACK_REC;
    const double x = r[0], y = r[1], dx = r[2], dy = r[3];
    const double qx = x + t * dx, qy = y + t * dy;
    const double ex = px - qx, ey = py - qy;
    TrackOut o;
    o.t = t;
    o.dist = sqrt(ex * ex + ey * ey);
    o.s = r[5] + t * r[6];
    o.d = (dx * ey - dy * ex >= 0.0) ? o.dist : -o.dist;
    const double two_pi = 6.283185307179586, pi = 3.141592653589793;    // 2 * np.pi, np.pi
    const double e = yaw - r[7];
    o.e = e - two_pi * floor((e + pi) / two_pi);
    return o;
}

// the rows [table_start[id], table_start[id + 1]) of table id, or false for an id outside [0, num_tables)
__device__ __forceinline__ bool track_table(const int32_t *__restrict__ table_start, int num_tables, int id,
                                            const double *__restrict__ &rec, int &n) {
    if (id < 0 || id >= num_tables) return false;
    const int off = table_start[id];
    n = table_start[id + 1] - off;
    rec += (size_t)off * F110_TRACK_REC;
    return true;
}

// f110_track_project: one warp per pose; out [M][5] = seg, t, d, s, e (all NaN for a non-finite pose or a bad table id).
__global__ void __launch_bounds__(128) k_track_project(const double *__restrict__ segments, const int32_t *__restrict__ table_start,
                                                       int num_tables, const double *__restrict__ poses,
                                                       const int32_t *__restrict__ table_ids, int M, double *__restrict__ out) {
    const int m = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (m >= M) return;
    const double px = poses[3 * (size_t)m], py = poses[3 * (size_t)m + 1], yaw = poses[3 * (size_t)m + 2];
    const double *rec = segments;
    int n = 0;
    const bool ok = isfinite(px) && isfinite(py) && isfinite(yaw) &&
                    track_table(table_start, num_tables, table_ids ? table_ids[m] : 0, rec, n);
    TrackHit h;
    h.k = 0x7fffffff;
    if (ok) h = track_search(rec, n, 0, n, px, py, lane);
    if (lane != 0) return;
    double *o = out + 5 * (size_t)m;
    if (h.k == 0x7fffffff) {
        o[0] = o[1] = o[2] = o[3] = o[4] = __longlong_as_double(0x7ff8000000000000ll);
        return;
    }
    const TrackOut r = track_outputs(rec, h.k, h.t, px, py, yaw);
    o[0] = (double)h.k; o[1] = r.t; o[2] = r.d; o[3] = r.s; o[4] = r.e;
}

struct TrackK {
    const double *state;              // [7][NA]
    const int32_t *steer_cnt;         // [NA]: 0 exactly when the agent was reset since its last step
    const int32_t *env_layer;         // [N] or NULL (table 0)
    const double *segments;
    const int32_t *table_start;
    int32_t *seg;
    double *s, *d, *e, *progress, *delta;
    double reacquire_dist;
    int num_tables, NA, A, back, window;   // window = back + fwd + 1
};

// f110_track_progress: one warp per agent.  Acquire (seg < 0, or a reset since the last step): global projection, progress
// and delta 0.  Track: first minimum over the window seg - back .. seg + fwd (clipped to n segments), in window order; a best
// dist above reacquire_dist (or none) falls back to the global projection; delta = s - s_prev unwrapped by half a lap.
__global__ void __launch_bounds__(128) k_track_progress(const TrackK p) {
    const int a = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (a >= p.NA) return;
    const int NA = p.NA;
    const double px = p.state[a], py = p.state[(size_t)NA + a], yaw = p.state[4 * (size_t)NA + a];
    const double *rec = p.segments;
    int n = 0;
    const bool ok = isfinite(px) && isfinite(py) && isfinite(yaw) &&
                    track_table(p.table_start, p.num_tables, p.env_layer ? p.env_layer[a / p.A] : 0, rec, n);
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    if (!ok) {
        if (lane == 0) {
            p.seg[a] = -1;
            p.s[a] = p.d[a] = p.e[a] = p.progress[a] = p.delta[a] = nan;
        }
        return;
    }
    const int sg = p.seg[a];
    bool acquire = sg < 0 || sg >= n || p.steer_cnt[a] == 0;
    TrackHit h;
    int base = 0;
    if (!acquire) {
        base = (sg - p.back) % n;
        if (base < 0) base += n;
        h = track_search(rec, n, base, p.window < n ? p.window : n, px, py, lane);
        if (h.k == 0x7fffffff || !(h.dist <= p.reacquire_dist)) base = -1;     // re-acquire, keep the progress
        else h.k = (base + h.k) % n;
    }
    if (acquire || base < 0) h = track_search(rec, n, 0, n, px, py, lane);
    if (lane != 0) return;
    if (h.k == 0x7fffffff) {
        p.seg[a] = -1;
        p.s[a] = p.d[a] = p.e[a] = p.progress[a] = p.delta[a] = nan;
        return;
    }
    const TrackOut r = track_outputs(rec, h.k, h.t, px, py, yaw);
    double delta = 0.0, prog = 0.0;
    if (!acquire) {
        const double *last = rec + (size_t)(n - 1) * F110_TRACK_REC;
        const double L = last[5] + last[6];          // = np.cumsum(len)[-1]: the same sum in the same order
        delta = r.s - p.s[a];
        if (delta > L * 0.5) delta -= L;
        else if (delta < -(L * 0.5)) delta += L;
        prog = p.progress[a] + delta;
    }
    p.seg[a] = h.k;
    p.s[a] = r.s; p.d[a] = r.d; p.e[a] = r.e;
    p.progress[a] = prog; p.delta[a] = delta;
}

}  // namespace f110
