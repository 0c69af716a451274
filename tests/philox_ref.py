"""Plain numpy restatement of the scan-noise stream of the CUDA path (csrc/lidar.cuh normal_sample): Philox4x32-10
(Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11; the Random123 round function) keyed by the 64-bit
seed, counter (index lo, index hi, stream lo, stream hi), then Box-Muller on the first two output words.

All words are held in uint64 arrays, so the 32 x 32 -> 64-bit products are exact and the high / low halves are plain
shifts and masks.  Test infrastructure only."""
import os

import numpy as np

M32 = np.uint64(0xFFFFFFFF)
PHILOX_M0, PHILOX_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
PHILOX_W0, PHILOX_W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Ten rounds on the counter words (arrays or scalars < 2^32) with key (k0, k1); returns four uint64 arrays."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) for x in (c0, c1, c2, c3))
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0 = PHILOX_M0 * c0
        p1 = PHILOX_M1 * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & M32
        hi1, lo1 = p1 >> np.uint64(32), p1 & M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + PHILOX_W0) & M32
        k1 = (k1 + PHILOX_W1) & M32
    return c0, c1, c2, c3


def normal_sample(seed, stream, index):
    """One standard normal per (seed, stream, index), fp64; `index` may be an array (uint64), seed and stream scalars."""
    seed, stream = int(seed) & 0xFFFFFFFFFFFFFFFF, int(stream) & 0xFFFFFFFFFFFFFFFF
    index = np.asarray(index, dtype=np.uint64)
    c0, c1, _, _ = philox4x32_10(index & M32, index >> np.uint64(32), stream & 0xFFFFFFFF, stream >> 32,
                                 seed & 0xFFFFFFFF, seed >> 32)
    u1 = (c0.astype(np.float64) + 1.0) * (1.0 / 4294967296.0)      # (0, 1]
    u2 = c1.astype(np.float64) * (1.0 / 4294967296.0)              # [0, 1)
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(np.pi * (2.0 * u2))


def tick_noise(seed, tick, num_agents_total, num_beams, std, threads=None):
    """The additive noise of one tick of the march kernels: std * normal_sample(seed, tick, a * B + i) for every agent
    a of the batch (flat index env * A + slot) and beam i -> (NA, B) fp64.  Chunks run on a thread pool (numpy releases
    the GIL inside its ufuncs)."""
    from concurrent.futures import ThreadPoolExecutor
    n = num_agents_total * num_beams
    out = np.empty(n)
    step = 1 << 20

    def fill(lo):
        hi = min(n, lo + step)
        out[lo:hi] = std * normal_sample(seed, tick, np.arange(lo, hi, dtype=np.uint64))
    with ThreadPoolExecutor(threads or os.cpu_count() or 1) as ex:
        list(ex.map(fill, range(0, n, step)))
    return out.reshape(num_agents_total, num_beams)
