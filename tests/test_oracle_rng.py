"""The Philox oracle (oracle/rng.py) on the CPU: the Random123 known-answer vectors of philox4x32-10, and the counter
conventions of the per-kernel helpers restated from the words."""
import numpy as np
import pytest

from oracle import rng as R


def _philox(counter, key):
    """Philox on a raw 4-word counter and 2-word key, through this repository's (seed, offset, ctr) layout."""
    seed = key[0] | (key[1] << 32)
    ctr = counter[0] | (counter[1] << 32)
    offset = counter[2] | (counter[3] << 32)
    return [int(v) for v in R.philox4x32_10(seed, offset, [ctr])[0]]


@pytest.mark.parametrize("counter,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(counter, key, want):
    assert _philox(counter, key) == list(want)


def test_helpers_follow_the_kernels_counter_conventions():
    seed, off = 0x1234_5678_9ABC_DEF0, (3 << 32) + 7
    blk = R.philox4x32_10(seed, off, np.arange(3))
    bits = R.binary_source(seed, off, 300)
    assert bits.shape == (300,)
    for i in (0, 31, 32, 127, 128, 200, 299):
        k, r = divmod(i, 128)
        assert bits[i] == (blk[k, r // 32] >> (r % 32)) & 1
    u = R.uniform(seed, off, 9, -2.0, 3.0)
    assert u.dtype == np.float32 and u[5] == np.float32(-2.0) + np.float32(5.0) * np.float32((blk[1, 1] >> 8) * 2.0 ** -24)
    assert np.all(R.uniform(seed, off, 9, 1.5, 1.5) == np.float32(1.5))
    g = R.normal(seed, off, 7)
    c, s = R.box_muller(blk[1, 2], blk[1, 3])
    assert g[6] == c and g.shape == (7,)
    w = R.awgn(seed, off, 5)
    c, s = R.box_muller(blk[2, 0], blk[2, 1])
    assert w[4] == c + 1j * s
    c, s = R.box_muller(blk[1, 2], blk[1, 3])
    assert w[3] == c + 1j * s
    z = R.channel_noise(seed, off, 3)
    c, s = R.box_muller(blk[2, 0], blk[2, 1])
    assert z[2] == c + 1j * s
    # u1 = 1 gives radius 0; u1 = 2^-24 the largest radius
    assert R.box_muller(np.uint32(0xFFFFFF00), np.uint32(0))[0] == 0.0
    assert np.isclose(R.box_muller(np.uint32(0), np.uint32(0))[0], np.sqrt(48 * np.log(2)))
