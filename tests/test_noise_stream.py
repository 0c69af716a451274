"""The scan-noise stream (csrc/lidar.cuh normal_sample: Philox4x32-10, then Box-Muller) against a plain numpy
restatement (tests/philox_ref.py).

CPU tier: the restated Philox reproduces the published Random123 known-answer vectors of philox4x32_10.
GPU tier: f110_scan_noise on zeros with std 1 is the numpy draw, for seeds with the high word set and index offsets on
both sides of 2^32 (the counter's second word)."""
import numpy as np
import pytest

import philox_ref

# Random123 kat_vectors, philox4x32 10 rounds: counter[4], key[2] -> output[4]
KAT = [((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000),
        (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff),
        (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize('ctr,key,want', KAT)
def test_philox_known_answers(ctr, key, want):
    got = philox_ref.philox4x32_10(*ctr, *key)
    assert tuple(int(x) for x in got) == want


def test_normal_sample_is_keyed_by_every_word():
    """Seed lo / hi, stream lo / hi and index lo / hi all change the draw; the marginal is standard normal."""
    base = float(philox_ref.normal_sample(1, 2, 3))
    for seed, stream, index in [(1 + (1 << 32), 2, 3), (0, 2, 3), (1, 2 + (1 << 32), 3), (1, 3, 3), (1, 2, 3 + (1 << 32)),
                                (1, 2, 4)]:
        assert float(philox_ref.normal_sample(seed, stream, index)) != base
    z = philox_ref.normal_sample(0xDEADBEEF12345678, 7, np.arange(1 << 18, dtype=np.uint64))
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1.0) < 0.01 and abs((z ** 4).mean() - 3.0) < 0.05


def fp32_bracket(z, rel=1e-12):
    """fp32 values a device result may take if its fp64 draw is within rel * max(1, |z|) of z (the numpy log and cos may
    differ from CUDA's log and cospi by a few ulps): [fp32(z - tol), fp32(z + tol)]."""
    tol = rel * np.maximum(1.0, np.abs(z))
    return (z - tol).astype(np.float32), (z + tol).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize('seed', [12345, 0xFFFFFFFF00000001, 0x8000000000000000, 0x0123456789ABCDEF])
@pytest.mark.parametrize('offset', [0, (1 << 32) - 1500, (1 << 33) + 7])
def test_scan_noise_kernel_equals_numpy_draw(seed, offset):
    import torch
    import f1tenth_gym_b200 as f110
    L = f110._native.lib()
    n = 3000
    out = torch.zeros(n, dtype=torch.float32, device='cuda:0')
    f110._native.check(L.f110_scan_noise(out.data_ptr(), n, 1.0, seed, offset, None))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    # f110_scan_noise draws from stream 0xFFFFFFFF (no tick) at index offset + i
    z = philox_ref.normal_sample(seed, 0xFFFFFFFF, np.uint64(offset) + np.arange(n, dtype=np.uint64))
    lo, hi = fp32_bracket(z)
    bad = np.flatnonzero((got < lo) | (got > hi))
    assert bad.size == 0, [(int(i), float(got[i]), float(z[i])) for i in bad[:5]]
    assert np.abs(got - z).max() < 1e-6 * max(1.0, np.abs(z).max())
