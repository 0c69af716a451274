// episode_repeat.cuh — episodes under a held action (f110_tick_repeat_episodes, include/f110_episode_repeat.h): K ticks under
// one action in which an env's episode stops at the first tick that ends it, keeps that tick's final observation, and restarts
// after the K ticks as f110_tick_episodes restarts it.  Included by f110_b200.cu after episodes.cuh, whose kernels it reuses.
//
// After every tick j of the call (the tick of f110_tick_repeat: the short path on j < K-1 when the plan allows it, else the
// plain tick; env_level, no auto-reset):
//   k_episode_latch      warp per env        for an env still in its episode: the tick counted, terminated / truncated,
//                                            done_any / done_tick; when it ends here end_tick = j, length, the final_* copies
//                                            and either its scan rows (a tick whose scans exist) or a snapshot of every input
//                                            the scan of tick j reads (a short-path tick: march_rec, agent_poses, wall_flag),
//                                            with its id appended to the final-scan list.  Envs that ended earlier in the call
//                                            are not touched: nothing after their end tick is visible.
// After the last tick, on the final-scan list (built on the device; empty on the full path):
//   k_restart_march      the scan of tick j from the snapshot records, to final_scans (noise off on the short path; the
//                        snapshot's iTTC threshold is -inf, so no wall flag is written)
//   k_episode_cast       the opponent ray-cast against the snapshot poses, with the yaw the snapshot's wall flag gives
//   k_episode_obstacles  the box clip (the boxes have not moved: the call has no auto-reset); its contact part rewrites
//                        final_collisions / final_collision_idx with the values they already hold
// each launched with an f110_sim whose agent_poses / wall_flag / scans point at the snapshot and final_scans.
// Then the restart of every env that ended anywhere in the call:
//   k_episode_restart    thread per env      done = the done of its end tick, track_seg = -1, track_delta_sum = 0, the start-pose
//                                            draw and the box respawn at the counter of the call's last tick; the restart list
//   k_episode_dyn, k_restart_march, k_episode_cast, k_episode_tail, k_episode_obstacles on that list, as f110_tick_episodes
//                        launches them.  k_restart_march runs without its crash-scan move: the latch already copied the scans
//                        of the envs that ended on the last tick, and the others have theirs from their end tick.
// An ended env keeps ticking under the held action after its end tick; the restart overwrites everything it changes, and the
// tick kernels stay exactly as they are.
#pragma once

namespace f110 {

struct LatchK {
    EpisodeK ep;                 // ticks, flags, length, final_*, max_ticks (list / count / track_seg unused here)
    int32_t *end_tick;           // [N]
    uint8_t *done_any;           // [N] or NULL
    int32_t *done_tick;          // [N] or NULL
    const float *scans;
    float *final_scans;
    double2 *snap_rec;           // [N*A][4]
    double *snap_poses;          // [N*A][5]
    int32_t *snap_flag;          // [N*A]
    uint32_t *scan_list, *scan_count;
    int tick;                    // index of this tick in the call
    int num_beams;
    uint32_t final_slots;        // slots that have a lidar: their scan rows go to final_scans
    int scans_exist;             // 1: this tick computed the scans of final_slots; 0: a short-path tick
};

__global__ void __launch_bounds__(128) k_episode_latch(f110_sim s, LatchK k) {
    const int env = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = (int)(threadIdx.x & 31u);
    if (env >= s.num_envs) return;                                  // warp-uniform
    const int A = s.num_agents, NA = s.num_envs * A;
    if (k.tick != 0 && k.end_tick[env] >= 0) return;                // its episode ended on an earlier tick of the call
    const int d = s.done[env] ? 1 : 0;
    const int t = k.ep.ticks[env] + 1;
    const bool term = d != 0;
    const bool trunc = !term && k.ep.max_ticks > 0 && t >= k.ep.max_ticks;
    const bool ended = term || trunc;
    __syncwarp();                                                   // every lane has read what lane 0 overwrites
    if (lane == 0) {
        k.ep.terminated[env] = term ? 1 : 0;
        k.ep.truncated[env] = trunc ? 1 : 0;
        if (k.done_any) k.done_any[env] = (uint8_t)((k.tick == 0 ? 0 : k.done_any[env]) | d);
        if (k.done_tick) {
            const int first = k.tick == 0 ? -1 : k.done_tick[env];
            k.done_tick[env] = (first < 0 && d) ? k.tick : first;
        }
        k.end_tick[env] = ended ? k.tick : -1;
        if (ended) k.ep.length[env] = t;
        k.ep.ticks[env] = ended ? 0 : t;                            // the restart's zero-action tick does not count
    }
    if (!ended) return;
    if (lane < A) {
        const size_t a = (size_t)env * A + lane;
#pragma unroll
        for (int q = 0; q < 7; q++) k.ep.final_state[(size_t)q * NA + a] = s.state[(size_t)q * NA + a];
        k.ep.final_collisions[a] = s.collisions[a];
        k.ep.final_collision_idx[a] = s.collision_idx[a];
        k.ep.final_lap_times[a] = s.lap_times[a];
        k.ep.final_lap_counts[a] = s.lap_counts[a];
        if (!k.scans_exist) {
            const double2 *rp = reinterpret_cast<const double2 *>(s.march_rec) + 4 * a;
            double2 *sp = k.snap_rec + 4 * a;
            sp[0] = rp[0];
            sp[1] = rp[1];
            sp[2] = make_double2(-INFINITY, rp[2].y);               // the scan alone: no iTTC predicate on the replay
            sp[3] = rp[3];
#pragma unroll
            for (int q = 0; q < 5; q++) k.snap_poses[5 * a + q] = s.agent_poses[5 * a + q];
            k.snap_flag[a] = s.wall_flag[a];
        }
    }
    if (k.scans_exist) {
        // four loads in flight per lane before their stores: one warp copies the env's rows, so its round trips are the cost
        for (int slot = 0; slot < A; slot++) {
            if (!((k.final_slots >> slot) & 1u)) continue;
            const size_t row = ((size_t)env * A + slot) * (size_t)k.num_beams;
            for (int i0 = lane; i0 < k.num_beams; i0 += 128) {
                float v[4];
#pragma unroll
                for (int q = 0; q < 4; q++) v[q] = i0 + 32 * q < k.num_beams ? k.scans[row + i0 + 32 * q] : 0.0f;
#pragma unroll
                for (int q = 0; q < 4; q++)
                    if (i0 + 32 * q < k.num_beams) k.final_scans[row + i0 + 32 * q] = v[q];
            }
        }
    } else if (lane == 0 && k.final_slots) {
        k.scan_list[atomicAdd(k.scan_count, 1u)] = (uint32_t)env;
    }
}

// thread per env that ended anywhere in the call: what k_episode_end does after its end decision, at the call's last tick
__global__ void k_episode_restart(f110_sim s, AutoResetArgs ar, LatchK k, ObstDraw d, int32_t *track_seg, double *delta_sum,
                                  uint32_t *list, uint32_t *count) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= s.num_envs || k.end_tick[env] < 0) return;
    const int A = s.num_agents;
    s.done[env] = k.ep.terminated[env];                             // done of the end tick (terminated == done there)
    for (int i = 0; i < A; i++) {
        const size_t a = (size_t)env * A + i;
        if (track_seg) track_seg[a] = -1;
        if (delta_sum) delta_sum[a] = 0.0;                         // a restarted env earns 0 on the call
    }
    episode_place(s, env, ar);
    if (d.cand) obst_respawn_one(s, env, d, s.tick_counter ? (uint64_t)*s.tick_counter : ar.tick_host);
    list[atomicAdd(count, 1u)] = (uint32_t)env;
}

}  // namespace f110
