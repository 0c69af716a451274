// render.cuh — k_render_views: top-down class rasters of the simulation (f110_render_views), one view per followed agent.
//
// A view of H x W pixels, row 0 at the top, s metres per pixel, follows agent a (flat index).  Every pixel gets one class code:
//   0 off-map, 1 free (dt != 0), 2 wall (dt == 0, what the lidar sees), 3 another agent of the env, 4 the followed agent,
//   255 the whole view is invalid (agent id outside [0, N*A), env layer outside [0, L), or the followed pose not finite: no table
//   is read).  Priority 4 > 3 > 2 > 1 / 0.
//
// Operation order (fp64, no FMA contraction: the library is built with -fmad=false; tests/test_views_host.py restates it):
//   x, y, yaw = state[0][a], state[1][a], state[4][a];   sincos(yaw) -> (sn, cs)   (as k_dynamics)
//   cx = x + f * cs;   cy = y + f * sn                                                 (f: forward offset)
//   h = s * 0.5;   u = (double)(2j + 1 - W) * h;   v = (double)(H - 2i - 1) * h        (pixel row i, column j)
//   world-aligned:  px = cx + u;                    py = cy + v
//   heading-up:     px = cx + (u * sn + v * cs);    py = cy + (v * sn - u * cs)
//   map class on layer l = env_layer[a / A] (0 without env_layer), the reference's xy_2_rc (laser_models.py:55-104):
//     tx = px - orig_x_l;  ty = py - orig_y_l;  x_rot = tx * c_l + ty * s_l;  y_rot = (-tx) * s_l + ty * c_l
//       ((c_l, s_l) = layer_rot[l], else the struct's (orig_c, orig_s); (1, 0) is the reference's own arithmetic)
//     off-map unless (x_rot >= 0 && x_rot < x_max_l && y_rot >= 0 && y_rot < y_max_l)   (NaN is off-map)
//     col = floor(x_rot / res_l), row = floor(y_rot / res_l) (IEEE quotients); off-map if col >= W_l or row >= H_l
//       (the oracle's deliberate deviation, DESIGN.md §4)
//     else wall if dt[l][row][col] == 0 (the metre table, canvas row pitch), free otherwise.
//     x_max_l, y_max_l, W_l, H_l are the layer's own (layer_geom), never the canvas: the canvas padding is off-map.
//   cars: every agent k of the env with a finite pose is the quad get_vertices(x_k, y_k, yaw_k, sim_length, sim_width)
//     (collision.cuh, the routine of k_vertices), vertices rl, rr, fr, fl (counter-clockwise).  Pixel centre p is inside when
//     bx0 <= px <= bx1 && by0 <= py <= by1 (the vertices' bounding box) and, for each edge (v0 -> v1) in that vertex order,
//     (v1x - v0x) * (py - v0y) - (v1y - v0y) * (px - v0x) >= 0.
//
// A block covers a tile of F110_RENDER_PIXELS consecutive pixels (row-major) of one view and loads the view's pose, its layer's
// geometry and the env's car quads into shared memory once per view; the grid's y dimension strides over the views.  Every
// thread writes four consecutive pixels, as one 32-bit store where the address allows.  Nothing but `out` is written.
#pragma once
#include "collision.cuh"

namespace f110 {

#define F110_RENDER_THREADS 256
#define F110_RENDER_PIXELS (4 * F110_RENDER_THREADS)
#define F110_RENDER_MAX_AGENTS 64      // car quads cached per block (agents per env)
#define F110_RENDER_MAX_SIZE 8192      // largest view height / width

struct RenderK {
    const double *__restrict__ state;       // [7][N*A]
    const int32_t *__restrict__ env_layer;  // [N], or NULL: layer 0
    const int32_t *__restrict__ agent_ids;  // [V]
    const double *__restrict__ dt;          // [L][Hc][Wc] metres
    const double *__restrict__ layer_geom;  // [L][6] or NULL
    const double *__restrict__ layer_res;   // [L][2] or NULL
    const double *__restrict__ layer_rot;   // [L][2] or NULL
    uint8_t *__restrict__ out;              // [V][H][W]
    double2 orig, ext, rot;                 // struct geometry: (orig_x, orig_y), (W res, H res), (orig_c, orig_s)
    double res;
    double length, width;                   // sim_length, sim_width
    double half, fwd;                       // metres per pixel / 2, forward offset
    unsigned long long layer_stride;        // Hc * Wc
    unsigned map_w, map_h;                  // canvas (or map) width / height
    unsigned num_layers;                    // >= 1
    int NA, A, V, H, W, heading_up;
};

struct RenderView {
    double cx, cy, sn, cs;
    double ox, oy, xmax, ymax, res, rc, rs;
    unsigned wl, hl;
    unsigned long long base;                // layer offset into dt
    int valid, self;                        // self: the followed agent's slot in the env
};

__global__ void __launch_bounds__(F110_RENDER_THREADS) k_render_views(const RenderK p) {
    __shared__ RenderView sv;
    __shared__ double4 s_box[F110_RENDER_MAX_AGENTS];          // bounding box (x0, x1, y0, y1); empty for a car not drawn
    __shared__ double s_vert[F110_RENDER_MAX_AGENTS][8];
    const unsigned long long HW = (unsigned long long)p.H * (unsigned long long)p.W;
    const unsigned long long lin0 = (unsigned long long)blockIdx.x * F110_RENDER_PIXELS + 4ull * threadIdx.x;
    for (long long vi = blockIdx.y; vi < p.V; vi += gridDim.y) {       // 64-bit: no overflow for V near INT32_MAX
        __syncthreads();                                        // the previous view's shared values are no longer read
        if (threadIdx.x == 0) {
            const int a = __ldg(p.agent_ids + vi);
            int valid = a >= 0 && a < p.NA;
            if (valid) {
                const double x = __ldg(p.state + a), y = __ldg(p.state + (size_t)p.NA + a);
                const double yaw = __ldg(p.state + 4 * (size_t)p.NA + a);
                valid = isfinite(x) && isfinite(y) && isfinite(yaw);
                const int env = a / p.A;
                const unsigned l = p.env_layer ? (unsigned)__ldg(p.env_layer + env) : 0u;
                valid = valid && l < p.num_layers;
                if (valid) {
                    double sn, cs;
                    sincos(yaw, &sn, &cs);
                    sv.sn = sn; sv.cs = cs;
                    sv.cx = x + p.fwd * cs;
                    sv.cy = y + p.fwd * sn;
                    double2 o = p.orig, e = p.ext, r = p.rot;
                    double res = p.res;
                    unsigned wl = p.map_w, hl = p.map_h;
                    if (p.layer_geom) {
                        const double *g = p.layer_geom + 6 * (size_t)l;
                        o = make_double2(__ldg(g), __ldg(g + 1));
                        e = make_double2(__ldg(g + 2), __ldg(g + 3));
                        wl = (unsigned)__ldg(g + 4); hl = (unsigned)__ldg(g + 5);
                        if (p.layer_res) res = __ldg(p.layer_res + 2 * (size_t)l);
                        if (p.layer_rot) r = make_double2(__ldg(p.layer_rot + 2 * (size_t)l), __ldg(p.layer_rot + 2 * (size_t)l + 1));
                    }
                    sv.ox = o.x; sv.oy = o.y; sv.xmax = e.x; sv.ymax = e.y; sv.res = res; sv.rc = r.x; sv.rs = r.y;
                    sv.wl = wl; sv.hl = hl;
                    sv.base = (unsigned long long)l * p.layer_stride;
                    sv.self = a - env * p.A;
                }
            }
            sv.valid = valid;
        }
        __syncthreads();
        if (sv.valid && threadIdx.x < (unsigned)p.A) {
            const int a = __ldg(p.agent_ids + vi);
            const int k = (a / p.A) * p.A + (int)threadIdx.x;
            const double x = __ldg(p.state + k), y = __ldg(p.state + (size_t)p.NA + k);
            const double yaw = __ldg(p.state + 4 * (size_t)p.NA + k);
            double v[8];
            get_vertices(x, y, yaw, p.length, p.width, v);
            double4 b = make_double4(INFINITY, -INFINITY, INFINITY, -INFINITY);
            if (isfinite(x) && isfinite(y) && isfinite(yaw)) {
                b.x = fmin(fmin(v[0], v[2]), fmin(v[4], v[6]));
                b.y = fmax(fmax(v[0], v[2]), fmax(v[4], v[6]));
                b.z = fmin(fmin(v[1], v[3]), fmin(v[5], v[7]));
                b.w = fmax(fmax(v[1], v[3]), fmax(v[5], v[7]));
            }
            s_box[threadIdx.x] = b;
#pragma unroll
            for (int q = 0; q < 8; q++) s_vert[threadIdx.x][q] = v[q];
        }
        __syncthreads();
        if (lin0 >= HW) continue;
        uint8_t cls[4];
        const bool valid = sv.valid != 0;
        unsigned i = (unsigned)(lin0 / (unsigned)p.W), j = (unsigned)(lin0 - (unsigned long long)i * (unsigned)p.W);
#pragma unroll
        for (int q = 0; q < 4; q++) {
            uint8_t c = 255;
            if (valid && lin0 + q < HW) {
                const double u = (double)(2 * (int)j + 1 - p.W) * p.half;
                const double w = (double)(p.H - 2 * (int)i - 1) * p.half;
                double px, py;
                if (p.heading_up) {
                    px = sv.cx + (u * sv.sn + w * sv.cs);
                    py = sv.cy + (w * sv.sn - u * sv.cs);
                } else {
                    px = sv.cx + u;
                    py = sv.cy + w;
                }
                c = 0;
                for (int k = 0; k < p.A; k++) {
                    const double4 b = s_box[k];
                    if (!(px >= b.x && px <= b.y && py >= b.z && py <= b.w)) continue;
                    const double *vk = s_vert[k];
                    bool in = true;
#pragma unroll
                    for (int e = 0; e < 4; e++) {
                        const int e2 = (e + 1) & 3;
                        const double ex = vk[2 * e2] - vk[2 * e], ey = vk[2 * e2 + 1] - vk[2 * e + 1];
                        in = in && (ex * (py - vk[2 * e + 1]) - ey * (px - vk[2 * e]) >= 0.0);
                    }
                    if (in) {
                        if (k == sv.self) { c = 4; break; }
                        c = 3;
                    }
                }
                if (c == 0) {
                    const double tx = px - sv.ox, ty = py - sv.oy;
                    const double xr = tx * sv.rc + ty * sv.rs;
                    const double yr = (-tx) * sv.rs + ty * sv.rc;
                    if (xr >= 0.0 && xr < sv.xmax && yr >= 0.0 && yr < sv.ymax) {
                        const double col = floor(xr / sv.res), row = floor(yr / sv.res);
                        if (col < (double)sv.wl && row < (double)sv.hl) {
                            const double d = __ldg(p.dt + sv.base + (unsigned long long)row * p.map_w + (unsigned long long)col);
                            c = (d == 0.0) ? 2 : 1;
                        }
                    }
                }
            }
            cls[q] = c;
            if (++j == (unsigned)p.W) { j = 0; i++; }
        }
        uint8_t *o = p.out + (unsigned long long)vi * HW + lin0;
        if (lin0 + 4 <= HW && ((size_t)o & 3u) == 0) {
            *reinterpret_cast<uint32_t *>(o) = (uint32_t)cls[0] | ((uint32_t)cls[1] << 8) | ((uint32_t)cls[2] << 16) |
                                              ((uint32_t)cls[3] << 24);
        } else {
#pragma unroll
            for (int q = 0; q < 4; q++)
                if (lin0 + q < HW) o[q] = cls[q];
        }
    }
}

}  // namespace f110
