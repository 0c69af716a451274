// param_draw.cuh — per-episode dynamics randomisation (f110_params_draw*, include/f110_param_draw.h): redraw the per-env
// parameter rows of the envs that start a new episode.  Included by f110_b200.cu after episode_repeat.cuh; uses its mix64.
//
// One kernel, launched after the call that restarted the envs (the tick and restart kernels stay as they are):
//   k_param_draw   thread per (env, slot)   the env's rule (a host mask, the auto-reset's collision predicate, or the episode
//                                           flags) picks it; then the final_params copy (episode rule) and the draw of every
//                                           drawn key of the slot at the tick counter read on the device.
// The draw is restated in numpy by f1tenth_gym_b200.simulator.param_draw_rows.
#pragma once

namespace f110 {

enum ParamDrawRule { PARAM_DRAW_MASK = 0, PARAM_DRAW_AUTORESET = 1, PARAM_DRAW_EPISODES = 2 };

struct ParamDrawK {
    const double *lo, *hi;                  // [A][F110_NPARAM]
    double *params;                         // [N*A][F110_NPARAM]
    double *final_params;                   // [N*A][F110_NPARAM] or NULL
    const unsigned long long *tick_counter;
    const uint8_t *mask;                    // PARAM_DRAW_MASK: [N] or NULL (all)
    const double *collisions;               // PARAM_DRAW_AUTORESET: [N*A]
    const uint8_t *terminated, *truncated;  // PARAM_DRAW_EPISODES: [N]
    uint64_t seed;
    int num_envs, num_agents, ego, rule, per_env;
    uint32_t keys[32];
    int32_t group[F110_NPARAM];
};

// __grid_constant__: keys[i] is indexed at run time; read in place from the parameter bank rather than copied to the stack
__global__ void __launch_bounds__(128) k_param_draw(const __grid_constant__ ParamDrawK k) {
    const int A = k.num_agents;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= k.num_envs * A) return;
    const int e = t / A, i = t - e * A;
    bool hit;
    if (k.rule == PARAM_DRAW_MASK) hit = !k.mask || k.mask[e] != 0;
    else if (k.rule == PARAM_DRAW_AUTORESET) hit = k.collisions[(size_t)e * A + k.ego] != 0.0;
    else hit = (k.terminated[e] | k.truncated[e]) != 0;
    if (!hit) return;
    double *row = k.params + (size_t)t * F110_NPARAM;
    if (k.final_params) {
        double *f = k.final_params + (size_t)t * F110_NPARAM;
#pragma unroll
        for (int q = 0; q < F110_NPARAM; q++) f[q] = row[q];
    }
    const uint32_t keys = k.keys[i];
    if (!keys) return;
    const uint64_t tick = (uint64_t)*k.tick_counter;
    const uint64_t base = k.seed + F110_PARAM_DRAW_C1 * (tick + 1) + F110_PARAM_DRAW_C2 * (uint64_t)(e + 1) +
                          F110_PARAM_DRAW_C3 * (uint64_t)((k.per_env ? 0 : i) + 1);
    const double *lo = k.lo + (size_t)i * F110_NPARAM, *hi = k.hi + (size_t)i * F110_NPARAM;
#pragma unroll
    for (int q = 0; q < F110_PARAM_DRAW_KEYS; q++) {
        if (!((keys >> q) & 1u)) continue;
        const uint64_t h = mix64(base + F110_PARAM_DRAW_C4 * (uint64_t)(k.group[q] + 1));
        const double u = (double)(h >> 11) * (1.0 / 9007199254740992.0);
        row[q] = lo[q] + u * (hi[q] - lo[q]);
    }
}

}  // namespace f110
