"""OFDM (de)modulation and signal.fft / ifft over the whole fft_size range the library accepts (1 ... 8192), held to
the single-precision error envelope rather than a fixed tolerance.

For every size both directions are compared with complex128 NumPy (oracle/ofdm.py for OFDM: cyclic prefix, l_min,
(i)fftshift; np.fft for signal.fft / ifft, where the shift is off). The error of the kernel against complex128 must be
at most 2x (rms) and 3x (max) the error of scipy.fft run in complex64 on the same input, both normalised by the rms of
the exact output. The worst ratios measured on an H100 80GB HBM3 are 1.84x / 2.09x over all sizes but two, which
have their own bar (SIZE_BARS). These are the generic kernel's sizes with many odd stages: 2187 = 3^7 at 2.35x / 2.71x
and 4095 = 3^2 * 5 * 7 * 13 at 2.94x / 3.40x. That kernel's odd radices are direct p-term butterflies. All its twiddles
are sincospif of the fp32 quotient -2k/N, which carries up to 2^-24 relative rounding unless N is a power of two.
An arithmetic slip (a conjugated twiddle, a shift by (N+1)/2) makes the ratio about 10^7.

A transform whose size has a prime factor p > 19 contains a direct p-term DFT (sb_ofdm_modulate's butterflies for
p <= 19 are specialised, larger primes are summed term by term), whose fp32 rounding error grows like sqrt(p) while an
FFT's grows like sqrt(log p); for those sizes the envelope is the larger of scipy's error and that of a length-p DFT
summed term by term in complex64 NumPy.

Which branch of the dispatcher (csrc/ofdm_mimo.cu, ofdm_fft) each size reaches:
  N <= 1024             warp-per-transform kernel, 4 / 2 / 1 transforms per warp for N <= 128 / <= 256 / larger;
                        radices 2, 4, odd primes <= 19 (specialised) and larger primes (direct sums: 23, 97, 127,
                        257, 529 = 23^2, 1009, 1022 = 2 * 7 * 73)
  N = 2048, 4096        in-place radix-16 kernel
  other N <= 8192       one CTA per transform (1025 = 5^2 * 41, 1031 prime, 2187 = 3^7, 4095, 5000, 6144, 7264,
                        7265 = 5 * 1453, 8192, and one transform of the prime 8191)
Tests: test_fft_sizes_within_fp32_envelope[N] runs every size in both directions with shift 1 (OFDM) and shift 0
(signal.fft / ifft); test_fft_prime_8191_single_transform; test_fft_partial_batches[N] runs job counts 1, 3, 5 and one
more than whole grid-stride passes in each kernel (N = 76, 200, 600: 4 / 2 / 1 per warp; 2048, 4096; 1536 generic);
test_fft_size_above_8192_is_refused.
"""
import numpy as np
import pytest
import scipy.fft as sfft
import torch

from oracle import ofdm as F
from oracle.parity import cnormal, envelope

pytestmark = pytest.mark.gpu

WARP_SIZES = [1, 2, 23, 46, 97, 127, 128, 129, 256, 257, 529, 1000, 1009, 1022, 1024]
R16_SIZES = [2048, 4096]
GENERIC_SIZES = [1025, 1031, 2187, 4095, 5000, 6144, 7264, 7265, 8192]
DEFAULT_BAR = (2.0, 3.0)                       # (rms, max)
SIZE_BARS = {2187: (3.0, 3.5), 4095: (3.5, 4.0)}


def _rms(a):
    return float(np.sqrt(np.mean(np.abs(a) ** 2)))


def _largest_prime_factor(n):
    p, big = 2, 1
    while n > 1:
        if p * p > n:
            return max(big, n)
        while n % p == 0:
            big, n = p, n // p
        p += 1
    return big


def _direct_dft_floor(n, size, rng):
    """Floor (rms, max) of the fp32 envelope of a size-n transform of `size` outputs: none unless n has a prime factor
    p > 19, else the error of min(16, size // p) (at least one) length-p DFTs summed term by term in complex64 (x_0 w^0
    + x_1 w^c + ... in that order, roots rounded to complex64) against complex128, normalised by the rms of the exact
    output."""
    p = _largest_prime_factor(n)
    if p <= 19:
        return 0.0, 0.0
    x = cnormal(rng, (max(1, min(16, size // p)), p))
    k = np.arange(p)
    w = np.exp(-2j * np.pi * k / p).astype(np.complex64)
    out = np.empty(x.shape, np.complex64)
    for c0 in range(0, p, 64):
        c = np.arange(c0, min(p, c0 + 64))
        terms = x[:, None, :] * w[(c[:, None] * k[None, :]) % p][None]
        out[:, c] = np.cumsum(terms, axis=-1)[..., -1]
    ref = np.fft.fft(x.astype(np.complex128), axis=-1)
    e = np.abs(out - ref) / _rms(ref)
    return _rms(e), float(e.max())


def _envelope_n(what, n, got, f32, ref, rng):
    """The envelope of a size-n transform, errors relative to the rms of the whole exact output."""
    return envelope(f"{what} N={n}", got, f32, ref, SIZE_BARS.get(n, DEFAULT_BAR), _direct_dft_floor(n, got.size, rng),
                    axis=None)


def _modulate_f32(x, cp):
    """oracle.ofdm_modulate evaluated in complex64 with scipy.fft."""
    n = x.shape[-1]
    t = sfft.ifft(np.fft.ifftshift(x, axes=-1), axis=-1, norm="ortho")
    assert t.dtype == np.complex64
    return np.concatenate([np.concatenate([t[..., l, n - cp[l]:], t[..., l, :]], -1) for l in range(len(cp))], -1)


def _demodulate_f32(x, n, l_min, cp):
    """oracle.ofdm_demodulate evaluated in complex64 with scipy.fft."""
    off = np.concatenate([[0], np.cumsum(n + cp)[:-1]])
    sym = np.stack([x[..., off[l] + cp[l]: off[l] + cp[l] + n] for l in range(len(cp))], axis=-2)
    f = sfft.fft(sym, axis=-1, norm="ortho")
    tmp = (-2 * np.pi * np.float32(l_min) / np.float32(n) * np.arange(n, dtype=np.float32)).astype(np.float32)
    f = f * np.exp(1j * tmp).astype(np.complex64)
    assert f.dtype == np.complex64
    return np.fft.fftshift(f, axes=-1)


def _check_ofdm(dev, x, cp, l_mins, rng):
    """Modulate x [..., nsym, n] with per-symbol cyclic prefixes cp, demodulate the result for each l_min: each
    direction against the oracle within the fp32 envelope; demodulate(modulate(x)) with l_min = 0 returns x."""
    from sionna_b200.phy.ofdm import OFDMModulator, OFDMDemodulator
    n = x.shape[-1]
    t = OFDMModulator(cp)(torch.from_numpy(x).to(dev))
    got_t = t.cpu().numpy()
    ref_t = F.ofdm_modulate(x.astype(np.complex128), cp)
    assert got_t.shape == ref_t.shape
    bad = [_envelope_n("modulate", n, got_t, _modulate_f32(x, cp), ref_t, rng)]
    for l_min in l_mins:
        xh = OFDMDemodulator(n, l_min, cp)(t).cpu().numpy()
        assert xh.shape == x.shape
        ref = F.ofdm_demodulate(got_t.astype(np.complex128), n, l_min, cp)
        bad.append(_envelope_n(f"demodulate l_min={l_min}", n, xh, _demodulate_f32(got_t, n, l_min, cp), ref, rng))
    back = OFDMDemodulator(n, 0, cp)(t).cpu().numpy()
    assert np.abs(back - x).max() < 3e-5 * np.sqrt(max(n, 72) / 72)
    return [b for b in bad if b]


def _check_signal_fft(dev, x, rng):
    """signal.fft / ifft (no shift, no cyclic prefix) along the last axis against np.fft, within the fp32 envelope."""
    from sionna_b200.phy.signal import fft, ifft
    n = x.shape[-1]
    xd = torch.from_numpy(x).to(dev)
    ref = np.fft.fft(x.astype(np.complex128), axis=-1) / np.sqrt(n)
    bad = [_envelope_n("fft", n, fft(xd).cpu().numpy(), sfft.fft(x, axis=-1, norm="ortho"), ref, rng)]
    ref = np.fft.ifft(x.astype(np.complex128), axis=-1) * np.sqrt(n)
    bad.append(_envelope_n("ifft", n, ifft(xd).cpu().numpy(), sfft.ifft(x, axis=-1, norm="ortho"), ref, rng))
    return [b for b in bad if b]


@pytest.mark.parametrize("n", WARP_SIZES + R16_SIZES + GENERIC_SIZES)
def test_fft_sizes_within_fp32_envelope(cuda_device, n):
    """3 rows x 5 OFDM symbols = 15 transforms, not a multiple of 2 or 4 transforms per warp; per-symbol cyclic
    prefixes (up to the full symbol for small N), l_min = 0 and -7; odd N exercise floor(N/2) in the (i)fftshift."""
    rng = np.random.default_rng(n)
    x = cnormal(rng, (3, 5, n))
    cp = rng.integers(0, min(n, 40) + 1, 5).astype(np.int32)
    cp[0] = min(n, 40)
    bad = _check_ofdm(cuda_device, x, cp, (0, -7), rng) + _check_signal_fft(cuda_device, x.reshape(15, n), rng)
    assert not bad, "\n".join(bad)


def test_fft_prime_8191_single_transform(cuda_device):
    """The largest prime the generic kernel accepts: one direct 8191-term DFT per direction, O(N^2) in one thread."""
    rng = np.random.default_rng(8191)
    x = cnormal(rng, (1, 1, 8191))
    bad = _check_ofdm(cuda_device, x, np.array([37], np.int32), (-7,), rng)
    assert not bad, "\n".join(bad)


def _grid_stride(n, dev):
    """Transforms one full grid-stride pass of the kernel that size n dispatches to covers (the launch rules of
    launch_fft_small_fpw / launch_fft_r16 / ofdm_fft), for every occupancy of 1 ... 4 CTAs per SM."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    if n <= 1024:
        fpw = 4 if n <= 128 else (2 if n <= 256 else 1)
        return 8 * fpw * sms * 12
    if n in (2048, 4096):
        return sms * (2 if n == 4096 else 4)
    return sms * 8


@pytest.mark.parametrize("n", [76, 200, 600, 2048, 4096, 1536])
def test_fft_partial_batches(cuda_device, n):
    """Job counts that leave the last batch of a warp (4 or 2 transforms per warp), a CTA or a grid-stride pass
    partly filled: 1, 3, 5 OFDM symbols of one row, and one transform more than whole grid-stride passes."""
    rng = np.random.default_rng(1000 + n)
    bad = []
    for shape in ((1, 1, n), (1, 3, n), (1, 5, n), (_grid_stride(n, cuda_device) + 1, 1, n)):
        x = cnormal(rng, shape)
        cp = np.full(shape[1], 11, np.int32)
        bad += _check_ofdm(cuda_device, x, cp, (-3,), rng)
    assert not bad, "\n".join(bad)


def test_fft_size_above_8192_is_refused(cuda_device):
    from sionna_b200._lib import SbError
    from sionna_b200.phy.ofdm import OFDMModulator, OFDMDemodulator
    from sionna_b200.phy.signal import fft
    x = torch.zeros((2, 1, 8193), dtype=torch.complex64, device=cuda_device)
    with pytest.raises(SbError, match="fft_size <= 8192"):
        OFDMModulator(0)(x)
    with pytest.raises(SbError, match="fft_size <= 8192"):
        OFDMDemodulator(8193, 0, 0)(x[:, 0])
    with pytest.raises(SbError, match="fft_size <= 8192"):
        fft(x)
