"""Oracle: the device random streams (csrc/rng.cuh, csrc/phy_kernels.cu, csrc/channel.cu) rebuilt from (seed, offset).
TEST INFRASTRUCTURE (NumPy). Philox4x32-10 restated from the published algorithm (Salmon, Moraes, Dror, Shaw, "Parallel
random numbers: as easy as 1, 2, 3", SC'11): ten rounds of two 32 x 32 -> 64-bit multiplications with the Weyl-sequence
key schedule. This repository's layout: key = (seed_lo, seed_hi), counter = (ctr_lo, ctr_hi, offset_lo, offset_hi).

The streams are this repository's own; they are not TensorFlow's (rng.cuh says why they cannot be). Each helper follows
the counter convention of one kernel, so a test can ask for the exact values a launch with (seed, offset) must produce.
Box-Muller is evaluated in float64 on the kernel's own integer words; the kernels evaluate it in float32.
"""
import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32_10(seed, offset, ctr):
    """Philox4x32-10 blocks: key (seed & 0xffffffff, seed >> 32), counter (ctr_lo, ctr_hi, offset_lo, offset_hi) for
    every counter value in ``ctr`` (array of integers < 2^64) -> uint32 array [len(ctr), 4]."""
    seed, offset = int(seed), int(offset)
    ctr = np.asarray(ctr, dtype=np.uint64).reshape(-1)
    c0, c1 = ctr & _LO, ctr >> _S32
    c2 = np.full_like(ctr, offset & 0xFFFFFFFF)
    c3 = np.full_like(ctr, offset >> 32)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2                              # exact: both factors < 2^32
        c0, c1, c2, c3 = ((p1 >> _S32) ^ c1 ^ np.uint64(k0), p1 & _LO, (p0 >> _S32) ^ c3 ^ np.uint64(k1), p0 & _LO)
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def box_muller(a, b):
    """Two N(0, 1) values from two 32-bit words, float64: u1 = ((a >> 8) + 1) 2^-24 in (0, 1], u2 = (b >> 8) 2^-24
    in [0, 1); r = sqrt(-2 log u1) -> (r cos 2 pi u2, r sin 2 pi u2)."""
    u1 = ((np.asarray(a, np.uint32) >> 8).astype(np.float64) + 1.0) * 2.0 ** -24
    u2 = (np.asarray(b, np.uint32) >> 8).astype(np.float64) * 2.0 ** -24
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2.0 * np.pi * u2), r * np.sin(2.0 * np.pi * u2)


def binary_source(seed, offset, n):
    """sb_binary_source: block k -> bits 128 k .. 128 k + 127, bit 32 w + b = bit b of word w. float32 0 / 1 [n]."""
    blocks = philox4x32_10(seed, offset, np.arange((n + 127) // 128))
    bits = (blocks[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1
    return bits.reshape(-1)[:n].astype(np.float32)


def _words(seed, offset, n, per_block):
    return philox4x32_10(seed, offset, np.arange((n + per_block - 1) // per_block)).reshape(-1)


def uniform(seed, offset, n, lo, hi):
    """sb_uniform: block k -> values 4 k .. 4 k + 3, lo + (hi - lo) u with u = (word >> 8) 2^-24, evaluated as the
    kernel does in float32 (w = hi - lo, then lo + w * u, each operation rounded: the kernel is built without FMA
    contraction). float32 [n]."""
    u = ((_words(seed, offset, n, 4)[:n] >> 8).astype(np.float32) * np.float32(2.0 ** -24)).astype(np.float32)
    lo, hi = np.float32(lo), np.float32(hi)
    w = np.float32(hi - lo)
    return (lo + (w * u).astype(np.float32)).astype(np.float32)


def normal(seed, offset, n):
    """sb_normal before its affine map: block k -> values 4 k .. 4 k + 3 = (g0.x, g0.y, g1.x, g1.y), g0 from words
    (x, y), g1 from (z, w). float64 [n]."""
    w = _words(seed, offset, n, 4).reshape(-1, 2)
    c, s = box_muller(w[:, 0], w[:, 1])
    return np.stack([c, s], -1).reshape(-1)[:n]


def awgn(seed, offset, n):
    """sb_awgn's unit noise before the scaling by sqrt(no / 2): block k -> complex samples 2 k (words x, y) and 2 k + 1
    (words z, w). complex128 [n]."""
    w = _words(seed, offset, n, 2).reshape(-1, 2)
    c, s = box_muller(w[:, 0], w[:, 1])
    return (c + 1j * s)[:n]


def channel_noise(seed, offset, n):
    """Unit noise of sb_apply_ofdm_channel / sb_apply_time_channel: output element i uses block i (counter = flat output
    index) and the Box-Muller pair of its words (x, y). complex128 [n]."""
    blk = philox4x32_10(seed, offset, np.arange(n))
    c, s = box_muller(blk[:, 0], blk[:, 1])
    return c + 1j * s
