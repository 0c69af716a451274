// obstacles.cuh — static box obstacles (f110_obstacles, include/f110_b200.h): parked cars of an env that have no sensor and
// never move.  Included by f110_b200.cu after the tail kernels, whose device functions it reuses.
//
// With obstacles bound, a tick runs its usual tail without the env-level part, then
//   k_obstacles       warp per agent   GJK of the agent's body against the env's boxes, ORed into collisions / collision_idx
//                                      (a box in slot k has the index A + k of a parked agent), then the scan clipped against
//                                      every box with the opponent ray-cast's arithmetic (ray_cast_agents :206-227)
//   k_env_tail_obst   thread per env   lap logic, repeat bookkeeping, auto-reset, and the respawn of the boxes of the envs the
//                                      auto-reset restarted
// so that contact is known before `done` and before the auto-reset, as it would be if the boxes were agents.
#pragma once

namespace f110 {

struct ObstK {
    const double *boxes;         // [N][K][5] (x, y, yaw, length, width)
    const uint8_t *active;       // [N][K]
    int32_t *hit;                // [N*A] or NULL: the highest slot the agent touches, -1 = none
    int K;
    uint32_t lidar;              // k_obstacles<true, true>: the lidar mask (f110_lidar); only those slots' scans are clipped
};

// the respawn draw (f110_obstacles.candidates / cand_offsets / count_* / clearance / seed), by value
struct ObstDraw {
    double *boxes;
    uint8_t *active;
    const double *cand;          // [C][5], NULL = no respawn
    int K, num_cand, num_tables; // num_tables 0: one table for every env; L: env on layer l draws from rows [off[l], off[l + 1])
    int count_min, count_max;
    double clearance;
    uint64_t seed;
    int32_t off[F110_MAX_START_TABLES + 1];
};

// the beams i0 .. i1 of one box, lane-strided: the cone test of finalize_agent, then `min(scan, fp32(get_range))` over the four
// edges (the beam loop of the opponent ray-cast, kept apart from the tuned tail kernels)
__device__ __forceinline__ void obst_cast_beams(float *scan, const BeamView &bv, int lane, double px, double py, double yaw,
                                                double phi, double cone, const double v[8], int i0, int i1) {
    for (int i = i0 + lane; i <= i1; i += 32) {
        const float cur = scan[i];
        const double bt = yaw + bv.scan_angles[i];
        double dl = bt - phi;
        dl = dl - (2 * M_PI) * rint(dl * (1.0 / (2 * M_PI)));
        const double adl = fabs(dl);
        if (adl > cone && (M_PI - adl) > cone) continue;
        double v3x, v3y;
        sincos(bt + M_PI / 2., &v3y, &v3x);
        const double curd = (double)cur;
        double r = INFINITY;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int e2 = (e + 1) & 3;
            const double d = get_range_below(px, py, v3x, v3y, v[2 * e], v[2 * e + 1], v[2 * e2], v[2 * e2 + 1], curd);
            if (d < r) r = d;
        }
        const float rf = (float)r;
        if (rf < cur) scan[i] = rf;
    }
}

// SCAN = false: the contact part alone (the intermediate ticks of f110_tick_repeat, whose scans nobody reads).  LIDAR: a tick
// with a lidar mask, where the scan of an agent whose slot has no lidar does not exist and is not touched.
// obstacles_agent: the work of agent a's warp, shared with the restarted envs' instance (k_episode_obstacles, episodes.cuh)
template <bool SCAN, bool LIDAR>
__device__ __forceinline__ void obstacles_agent(const f110_sim &s, const BeamView &bv, const ObstK &o, double max_scan_range,
                                                int a, int lane) {
    const int A = s.num_agents, env = a / A;
    const double *pa = s.agent_poses + 5 * (size_t)a;
    const double *boxes = o.boxes + (size_t)env * o.K * 5;
    const uint8_t *act = o.active + (size_t)env * o.K;

    // GJK (collision_multiple :184-212): lane k tests slot k.  The agent's index is below every box's, so the agent's body is
    // the first argument.  Bounding circles farther apart than the sum of their radii (with a 0.1 % margin) cannot overlap.
    int hk = -1;
    if (lane < o.K) {
        const double *b = boxes + 5 * lane;
        if (box_present(b, act[lane])) {
            const double ddx = b[0] - pa[0], ddy = b[1] - pa[1];
            const double reach = 0.5 * sqrt(s.sim_length * s.sim_length + s.sim_width * s.sim_width) +
                                 0.5 * sqrt(b[3] * b[3] + b[4] * b[4]);
            if (ddx * ddx + ddy * ddy <= reach * reach * 1.001) {
                double vme[8], vb[8], sb, cb;
                sincos(b[2], &sb, &cb);
                get_vertices_cs(pa[0], pa[1], pa[3], pa[4], s.sim_length, s.sim_width, vme);
                get_vertices_cs(b[0], b[1], cb, sb, b[3], b[4], vb);
                if (gjk_collision(vme, vb)) hk = lane;
            }
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) hk = max(hk, __shfl_xor_sync(0xffffffffu, hk, d));
    if (lane == 0) {
        if (hk >= 0) {
            s.collisions[a] = 1.0;
            s.collision_idx[a] = max(s.collision_idx[a], A + hk);
        }
        if (o.hit) o.hit[a] = hk;
    }
    if (!SCAN) return;
    if (LIDAR && !((o.lidar >> (a - env * A)) & 1u)) return;

    // the scan, clipped against every box as against an opponent; check_ttc has zeroed the yaw of an agent whose iTTC fired
    const int hit = s.wall_flag[a];
    const double px = pa[0], py = pa[1];
    const double yaw = hit ? 0.0 : pa[2];
    const double cyaw = hit ? 1.0 : pa[3], syaw = hit ? 0.0 : pa[4];
    float *scan = s.scans + (size_t)a * bv.num_beams;
    for (int k = 0; k < o.K; k++) {
        const double *b = boxes + 5 * k;
        if (!box_present(b, act[k])) continue;
        const double half_diag = 0.5 * sqrt(b[3] * b[3] + b[4] * b[4]);
        const double ddx = b[0] - px, ddy = b[1] - py;
        const double far = max_scan_range + half_diag;
        if (ddx * ddx + ddy * ddy > far * far) continue;      // cannot shorten any beam (see finalize_agent)
        double v[8], sb, cb;
        sincos(b[2], &sb, &cb);
        get_vertices_cs(b[0], b[1], cb, sb, b[3], b[4], v);
        int lo, hi;
        double phi;
        blocked_view_indices_warp(px, py, cyaw, syaw, v, bv.scan_angles, bv.num_beams, bv.fov, bv.angle_increment, lane, b[0],
                                  b[1], lo, hi, phi);
        // the rear-cut cone filter of finalize_agent: a wide window visits only the beams around the centres (phi - yaw) + m pi
        double cone = 4.0;
        const bool wide = hi - lo >= 96;
        if (wide) {
            const double dist = sqrt(ddx * ddx + ddy * ddy);
            if (dist > 1.25 * half_diag) cone = asin(half_diag / dist) + 0.05;
        }
        if (cone < 3.5 && wide) {
            const double base = wrap_2pi_diff(phi - yaw), half = bv.fov / 2., inv_inc = 1.0 / bv.angle_increment;
            const int m0 = max(-3, (int)floor((-half - cone - 0.02 - base) * (1.0 / M_PI))),
                      m1 = min(5, (int)ceil((half + cone + 0.02 - base) * (1.0 / M_PI)));
            for (int m = m0; m <= m1; m++) {
                const double c = base + (double)m * M_PI;
                const double f0 = (c - cone + half) * inv_inc - 2.0, f1 = (c + cone + half) * inv_inc + 2.0;
                if (f1 < (double)lo || f0 > (double)hi) continue;
                const int i0 = max(lo, (int)floor(fmax(f0, (double)lo))), i1 = min(hi, (int)ceil(fmin(f1, (double)hi)));
                obst_cast_beams(scan, bv, lane, px, py, yaw, phi, cone, v, i0, i1);
            }
        } else {
            obst_cast_beams(scan, bv, lane, px, py, yaw, phi, cone, v, lo, hi);
        }
        __syncwarp();
    }
}

template <bool SCAN, bool LIDAR = false>
__global__ void __launch_bounds__(128) k_obstacles(f110_sim s, BeamView bv, ObstK o, double max_scan_range) {
    const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (a >= s.num_envs * s.num_agents) return;
    obstacles_agent<SCAN, LIDAR>(s, bv, o, max_scan_range, a, lane);
}

// u in [0, 1) from the top 53 bits of a hash, as the auto-reset's start-pose draw
__device__ __forceinline__ double hash_unit(uint64_t h) { return (double)(h >> 11) * (1.0 / 9007199254740992.0); }

// The respawn draw of env `env` at tick counter `tick` (f1tenth_gym_b200/obstacles.py restates it in numpy): the active count
// c = count_min + floor(u * (count_max - count_min + 1)) from one hash of (tick, env); slot k takes candidate row
// min(floor(u_k * C_l), C_l - 1) of the env's table from a hash of (tick, env, k) and is active when k < c and its centre is
// not closer than `clearance` to any agent's position in sim->state.  No retry.
__device__ __forceinline__ void obst_respawn_one(const f110_sim &s, int env, const ObstDraw &d, uint64_t tick) {
    const int A = s.num_agents, NA = s.num_envs * A;
    const double *cand = d.cand;
    int C = d.num_cand;
    if (d.num_tables) {
        const int l = s.env_layer[env];
        if (l < 0 || l >= d.num_tables) {       // a layer without a candidate table: the env gets no boxes
            for (int k = 0; k < d.K; k++) d.active[(size_t)env * d.K + k] = 0;
            return;
        }
        cand += 5 * (size_t)d.off[l];
        C = d.off[l + 1] - d.off[l];
    }
    const uint64_t base = d.seed + 0xA0761D6478BD642Full * (tick + 1) + 0xE7037ED1A0B428DBull * (uint64_t)(env + 1);
    const int span = d.count_max - d.count_min + 1;
    int c = (int)(hash_unit(mix64(base + 0x589965CC75374CC3ull)) * span);
    if (c >= span) c = span - 1;
    c += d.count_min;
    const double clr2 = d.clearance * d.clearance;
    for (int k = 0; k < d.K; k++) {
        int j = (int)(hash_unit(mix64(base + 0x8EBC6AF09C88C6E3ull * (uint64_t)(k + 1))) * C);
        if (j >= C) j = C - 1;
        const double *src = cand + 5 * (size_t)j;
        double *dst = d.boxes + ((size_t)env * d.K + k) * 5;
#pragma unroll
        for (int q = 0; q < 5; q++) dst[q] = src[q];
        bool on = k < c;
        for (int i = 0; i < A && on; i++) {
            const size_t a = (size_t)env * A + i;
            const double dx = src[0] - s.state[a], dy = src[1] - s.state[(size_t)NA + a];
            if (dx * dx + dy * dy < clr2) on = false;
        }
        d.active[(size_t)env * d.K + k] = on ? 1 : 0;
    }
}

// per env: the env-level part of the tail after k_obstacles.  The respawn follows the auto-reset's own predicate, read before
// the auto-reset runs, so that both act on the same envs.
__global__ void k_env_tail_obst(f110_sim s, int env_level, AutoResetArgs ar, RepeatDone rd, ObstDraw d) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= s.num_envs) return;
    if (env_level) {
        env_post_step_one(s, env);
        if (rd.done_any || rd.done_tick) repeat_done_one(s, env, rd);
    }
    if (!ar.start_poses) return;
    const bool fired = s.collisions[(size_t)env * s.num_agents + s.ego_idx] != 0.0;
    autoreset_one(s, env, ar);
    if (fired && d.cand) obst_respawn_one(s, env, d, s.tick_counter ? (uint64_t)*s.tick_counter : ar.tick_host);
}

// f110_obstacles_respawn: the draw for the masked envs at a given tick counter
__global__ void k_obst_respawn(f110_sim s, ObstDraw d, const uint8_t *__restrict__ mask, uint64_t tick) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= s.num_envs || (mask && !mask[env])) return;
    obst_respawn_one(s, env, d, tick);
}

}  // namespace f110
