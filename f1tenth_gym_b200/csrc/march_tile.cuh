// march_tile.cuh — k_march_tile: the north_star's ray-march design (BASELINE.json): the occupancy-grid tile around
// each agent's scan pose is staged into SHARED memory by TMA (cp.async.bulk.tensor.2d, mbarrier completion) and the
// agent's beams march through it on chip; lookups that leave the tile fall back to the global table.
//
// Why: k_march_lean is latency bound (long-scoreboard 11 warps per issue, L1 hit rate 53 %, 21.8 cycles
// per instruction per warp): every sphere-tracing step is a dependent, divergent 8-byte gather that misses L1 half of
// the time because the ~10 agents an SM works on at once have a 40-130 KB footprint each in the 8-byte table.  The
// tile holds the near field (where the lookups are dense) as 1-byte rank codes: TILE x TILE cells = 16 KB, decoded
// through the 2 KB fp64 LUT that also lives in shared memory -> two LDS (29 cycles each) instead of an L1/L2 gather.
//
// Organisation (a block = 512 threads, 4 blocks per SM, NSLOT tile slots per block):
//   * agents are claimed from a global longest-first queue (agent-level classes built by k_dynamics from last tick's
//     per-slice lookup maxima), one claim per slot refill; the claimer computes the tile origin (scan cell - TILE/2,
//     clamped into the padded table so that the box never leaves it), arms the slot's mbarrier with the byte count
//     and issues the TMA load;
//   * the block's warps take (sequence, slice) tickets from a shared counter, IN ORDER: ticket g belongs to the
//     (g / ipa)-th agent this block claimed, slice g % ipa.  A warp waits for the slot's publication word and then for
//     the mbarrier phase of that fill, marches its 32 beams in a warp-synchronous loop while ANY of its live beams is
//     still inside the tile, then gives the slot back (a ray that has left a convex box around its origin never
//     re-enters it) and finishes the stragglers on the global fp64 table exactly like k_march_lean;
//   * the warp that returns the last slice of a slot refills it (claim, origin, fence.proxy.async, TMA), so there is
//     no producer warp and no block barrier after the prologue.
// Results are bit-identical to k_march_lean / the oracle (same arithmetic, same lookups; tests/test_gpu_round2.py).
// Behavioural spec: reference laser_models.py:106-217.
#pragma once
#include <cuda.h>
#include "march_lean.cuh"

namespace f110 {

struct TileK {
    LeanK l;                                // tables, record, outputs, constants (CELLS flavour)
    const unsigned *__restrict__ order;     // [3][M] agent classes (very heavy | heavy | light)
    const unsigned *__restrict__ count;     // [4]: [0..2] class sizes, [3] the global claim counter
    unsigned *claim;                        // = count + 3
    unsigned *__restrict__ cost;            // [M << 8] per-slice lookup maxima (written here, read by next tick's k_dynamics)
    unsigned agents;                        // M
    unsigned ipa;                           // 32-beam slices per agent
    unsigned ipa_magic;                     // floor(2^32 / ipa) + 1: g / ipa == umulhi(g, magic) for g < 2^24
    unsigned codes_pitch;                   // row pitch of the padded code table (multiple of 16)
    int c_max, r_max;                       // largest legal tile origin: pitch - TILE, (H + 1) - TILE
    unsigned long long *tile_counter;       // COUNT only: lookups served from the tile (debug), or NULL
};

#define F110_TILE_END 0xFFFFFFFFu

__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\tLAB_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\tbra LAB_WAIT;\n\tDONE:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(unsigned dst, const CUtensorMap *tm, int c0, int r0, unsigned bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(dst), "l"(tm), "r"(c0), "r"(r0), "r"(bar) : "memory");
}

template <int TILE, int NSLOT>
struct TileSmem {
    alignas(128) unsigned char tile[NSLOT][TILE * TILE];
    alignas(16) double lut[256];
    alignas(8) unsigned long long bar[NSLOT];
    int org_c[NSLOT], org_r[NSLOT];
    unsigned agent[NSLOT];
    unsigned left[NSLOT];
    unsigned ready[NSLOT];                  // sequence number published for the slot; F110_TILE_END = no more agents, ever
    unsigned next;                          // ticket counter
    unsigned ended;                         // slots that reached F110_TILE_END
};

// claim the next agent of the global queue for `slot` (sequence `seq`), start its tile load and publish it
template <int TILE, int NSLOT>
__device__ __forceinline__ void tile_refill(const TileK &p, const CUtensorMap *tm, TileSmem<TILE, NSLOT> *s, unsigned slot,
                                            unsigned seq) {
    const unsigned nA = min(p.count[0], p.agents), nB = min(p.count[1], p.agents);
    const unsigned nAB = nA + nB;
    const unsigned total = min(nAB + min(p.count[2], p.agents), p.agents);
    const unsigned q = atomicAdd(p.claim, 1u);
    if (q >= total) {
        s->agent[slot] = F110_TILE_END;
        atomicAdd(&s->ended, 1u);
        __threadfence_block();
        *(volatile unsigned *)&s->ready[slot] = F110_TILE_END;
        return;
    }
    const unsigned a = p.order[(q < nA) ? q : (q < nAB) ? (p.agents + (q - nA)) : (2u * p.agents + (q - nAB))];
    const double2 r0 = __ldg(p.l.rec + 4 * (size_t)a);
    // cell of the scan pose (absurd coordinates hold metres here: the origin is clamped, the tile is simply not used)
    const double fx = floor(r0.x - p.l.ox), fy = floor(r0.y - p.l.oy);
    int cc = (fx > -1e9 && fx < 1e9) ? (int)fx : 0, rr = (fy > -1e9 && fy < 1e9) ? (int)fy : 0;
    // TMA: the box start must be 16-byte aligned in the innermost dimension (an unaligned start coordinate faults as an
    // illegal instruction at the UTMALDG): 1-byte cells -> a multiple of 16 columns; c_max is one (pitch and TILE are)
    cc = max(0, min(cc - TILE / 2, p.c_max)) & ~15;
    rr = max(0, min(rr - TILE / 2, p.r_max));
    s->agent[slot] = a;
    s->org_c[slot] = cc;
    s->org_r[slot] = rr;
    s->left[slot] = p.ipa;
    const unsigned bar = (unsigned)__cvta_generic_to_shared(&s->bar[slot]);
    const unsigned dst = (unsigned)__cvta_generic_to_shared(&s->tile[slot][0]);
    // the slot's previous tile was read through the generic proxy; order those reads before the async-proxy write
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    mbar_expect_tx(bar, (unsigned)(TILE * TILE));
    tma_load_2d(dst, tm, cc, rr, bar);
    __threadfence_block();
    *(volatile unsigned *)&s->ready[slot] = seq;
}

template <bool NOISE, bool COUNT, int TILE, int NSLOT, int PT, int MINB>
__global__ void __launch_bounds__(PT, MINB) k_march_tile(const TileK p, const __grid_constant__ CUtensorMap tmap) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    TileSmem<TILE, NSLOT> *s = reinterpret_cast<TileSmem<TILE, NSLOT> *>(smem_raw);
    const unsigned lane = threadIdx.x & 31u;
    for (unsigned t = threadIdx.x; t < 256u; t += PT) s->lut[t] = p.l.lut[t];
    if (threadIdx.x == 0) {
        s->next = 0u;
        s->ended = 0u;
        for (int k = 0; k < NSLOT; k++) mbar_init((unsigned)__cvta_generic_to_shared(&s->bar[k]), 1u);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int k = 0; k < NSLOT; k++) tile_refill<TILE, NSLOT>(p, &tmap, s, (unsigned)k, (unsigned)k);
    }
    __syncthreads();
    const unsigned next_addr = (unsigned)__cvta_generic_to_shared(&s->next);
    const double MAGIC = 6755399441055744.0;   // 2^52 + 2^51
    unsigned looks = 0u, tile_looks = 0u;
    for (;;) {
        unsigned g = 0, leader;
        asm volatile("{\n\t.reg .pred p;\n\telect.sync %1|p, 0xffffffff;\n\t@p atom.shared.add.u32 %0, [%2], 1;\n\t}"
                     : "+r"(g), "=r"(leader) : "r"(next_addr) : "memory");
        g = __shfl_sync(0xffffffffu, g, leader);
        const unsigned seq = __umulhi(g, p.ipa_magic);
        const unsigned slice = g - seq * p.ipa;
        const unsigned fill = seq / (unsigned)NSLOT;
        const unsigned slot = seq - fill * (unsigned)NSLOT;
        // wait until the slot carries this sequence number (or the end marker)
        unsigned rdy;
        while ((rdy = *(volatile unsigned *)&s->ready[slot]) != seq && rdy != F110_TILE_END) __nanosleep(32);
        if (rdy == F110_TILE_END) {
            if (*(volatile unsigned *)&s->ended >= (unsigned)NSLOT) break;
            continue;
        }
        __threadfence_block();
        const unsigned a = s->agent[slot];
        const int c0 = s->org_c[slot], r0c = s->org_r[slot];
        const int i = (int)(slice * 32u + lane);
        const double2 *__restrict__ rp = p.l.rec + 4 * (size_t)a;
        const double2 r0 = __ldg(rp), r1 = __ldg(rp + 1);
        const unsigned long long ti0fx = (unsigned long long)__double_as_longlong(r1.y);
        const bool valid = i < p.l.B;
        unsigned n = 0;
        double range = 0.0;
        if (ti0fx != ~0ull) {                                   // warp-uniform (per agent)
            double2 sc = make_double2(0.0, 0.0);
            if (valid) {
                const unsigned long long vfx = ti0fx + (unsigned long long)(unsigned)i * p.l.inc_fx;
                unsigned ti = (unsigned)(vfx >> F110_FX_SHIFT);
                const unsigned fr = (unsigned)(vfx >> (F110_FX_SHIFT - 32));
                if (fr + p.l.guard32 <= 2u * p.l.guard32)
                    ti = (unsigned)replay_theta_index(__ldg(rp + 3).y, i, p.l.inc, p.l.theta_dis_f);
                sc = __ldg(p.l.sincos2 + ti);
            }
            const double *__restrict__ table = p.l.table;
            asm volatile("" : "+l"(table));
            double X = r0.x, Y = r0.y, T = r1.x, D = r1.x;
            n = valid ? 1u : 0u;
            bool alive = valid && __double2hiint(D) != 0 && T <= p.l.tmax;
            if (alive) { X = X + D * sc.y; Y = Y + D * sc.x; }
            // phase 1: the tile is resident -- wait for its TMA load, then march while any live beam is inside it
            mbar_wait((unsigned)__cvta_generic_to_shared(&s->bar[slot]), fill & 1u);
            const unsigned char *__restrict__ tile = s->tile[slot];
            for (;;) {
                unsigned c = 0, r = 0;
                bool in = false;
                if (alive) {
                    c = (unsigned)__double2loint(__dadd_rd(X - p.l.ox, MAGIC));
                    r = (unsigned)__double2loint(__dadd_rd(Y - p.l.oy, MAGIC));
                    in = (((c - (unsigned)c0) | (r - (unsigned)r0c)) < (unsigned)TILE);
                }
                if (!__any_sync(0xffffffffu, in)) break;
                if (alive) {
                    if (in) {
                        D = s->lut[tile[(r - (unsigned)r0c) * (unsigned)TILE + (c - (unsigned)c0)]];
                        if (COUNT) tile_looks++;
                    } else {
                        D = __ldg(table + min(r, p.l.height) * (p.l.width + 1u) + min(c, p.l.width));
                    }
                    T = T + D;
                    n++;
                    alive = __double2hiint(D) != 0 && T <= p.l.tmax;
                    if (alive) { X = X + D * sc.y; Y = Y + D * sc.x; }
                }
            }
            // give the slot back; the warp that returns the last slice refills it
            if (lane == leader) {
                if (atomicSub(&s->left[slot], 1u) == 1u) tile_refill<TILE, NSLOT>(p, &tmap, s, slot, seq + (unsigned)NSLOT);
            }
            // phase 2: stragglers on the global fp64 table (same loop as k_march_lean, lookup pending at (X, Y))
            while (alive) {
                const unsigned c = (unsigned)__double2loint(__dadd_rd(X - p.l.ox, MAGIC));
                const unsigned r = (unsigned)__double2loint(__dadd_rd(Y - p.l.oy, MAGIC));
                D = __ldg(table + min(r, p.l.height) * (p.l.width + 1u) + min(c, p.l.width));
                T = T + D;
                n++;
                alive = __double2hiint(D) != 0 && T <= p.l.tmax;
                if (alive) { X = X + D * sc.y; Y = Y + D * sc.x; }
            }
            if (T != T)      // an escape code (NaN from the LUT) ended the beam: redo it on the fp64 table
                T = redo_beam_cells(table, r0.x, r0.y, r1.x, sc.x, sc.y, p.l.ox, p.l.oy, p.l.tmax, p.l.width, p.l.height, &n);
            range = ((T > p.l.tmax) ? p.l.tmax : T) * p.l.res;
        } else {
            if (lane == leader) {
                mbar_wait((unsigned)__cvta_generic_to_shared(&s->bar[slot]), fill & 1u);     // the load must land before the slot is reused
                if (atomicSub(&s->left[slot], 1u) == 1u) tile_refill<TILE, NSLOT>(p, &tmap, s, slot, seq + (unsigned)NSLOT);
            }
            if (valid) {
                const double2 r3 = __ldg(rp + 3);
                const int ti = beam_theta_index(r3.y, i, p.l.inc, p.l.theta_dis_f, 1e-6);
                const double2 sc = __ldg(p.l.sincos2 + ti);
                range = march_generic(p.l.dt, p.l.orig_x, p.l.orig_y, p.l.x_max, p.l.y_max, p.l.res, __ldg(p.l.dt + p.l.last),
                                      p.l.eps_m, p.l.max_range, (int)p.l.width, r0.x, r0.y, sc.x, sc.y);
                n = 1;
            }
        }
        if (valid) {
            if (NOISE) {
                const unsigned long long tick = p.l.tick_counter ? *p.l.tick_counter : 0ull;
                range = range + p.l.noise_std * normal_sample(p.l.noise_seed, tick, (uint64_t)a * (uint64_t)p.l.B + (uint64_t)i);
            }
            const double2 r2 = __ldg(rp + 2);
            if (range <= r2.x) {
                const double2 cs2 = __ldg(p.l.cos_side + i);
                ttc_exact(range, r2.y, cs2.x, cs2.y, p.l.ttc_thresh, p.l.ttc_margin, p.l.wall_flag + a);
            }
            p.l.out[a * (unsigned)p.l.B + (unsigned)i] = (float)range;
        }
        if (COUNT) looks += n;
        const unsigned mx = __reduce_max_sync(0xffffffffu, n);
        if (lane == 0) p.cost[(a << 8) | slice] = mx;
    }
    if (COUNT) {
        const unsigned nsum = __reduce_add_sync(0xffffffffu, looks);
        if (lane == 0 && nsum) atomicAdd(p.l.lookup_counter, (unsigned long long)nsum);
        if (p.tile_counter) {
            const unsigned tsum = __reduce_add_sync(0xffffffffu, tile_looks);
            if (lane == 0 && tsum) atomicAdd(p.tile_counter, (unsigned long long)tsum);
        }
    }
}

}  // namespace f110
