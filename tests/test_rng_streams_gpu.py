"""Every random-drawing kernel against the Philox oracle (oracle/rng.py), value by value: the bits of sb_binary_source,
the uniforms of sb_uniform, the Box-Muller normals of sb_normal and sb_awgn, and the noise that sb_apply_ofdm_channel and
sb_apply_time_channel add. Moment tests cannot tell a wrong key or counter word, two elements sharing a counter or a lost
tail element from a correct stream; these tests can.

Calls go through the C-ABI with explicit (seed, offset), with seeds whose high word is not zero and offsets >= 2^32 so
that every key and counter word takes part, and through the blocks with the (seed, offset) that config hands out.

Exactness:
  sb_binary_source  bit for bit.
  sb_uniform        exact: lo + (hi - lo) u in float32 with every operation rounded (phy_kernels.cu is built with
                    -fmad=false, so the compiler does not contract it into an FMA).
  Box-Muller        the kernels evaluate it in float32: logf (1 ulp, CUDA Math API), sqrtf (correctly rounded),
                    sincospif (1 ulp each) and the product (0.5 ulp) put r cos / r sin within 2.5 ulp of the float64 value
                    on the same integer words. The scaling by sqrt(no) * 0.70710678f (sqrtf 0.5 ulp, the constant 0.14 ulp,
                    two roundings) and the final addition bring the bound to BOUND_ULP = 5 ulp (2^-23 relative) of
                    |signal| + |noise|. The worst measured error is printed (pytest -s).
"""
import numpy as np
import pytest
import torch

from oracle import rng as R

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -23
BOUND_ULP = 5.0
SIZES = [1, 2, 3, 4, 5, 127, 128, 129, 2_000_003]
SEEDS = [(0x0000_0000_0000_0007, 0),
         (0xFEDC_BA98_7654_3210, (0xABCD << 32) | 0x1234),          # k1 and c3 both matter
         (0x7FFF_FFFF_FFFF_FFFF, (1 << 63) + 5)]


def _lib():
    from sionna_b200._lib import lib
    return lib()


def _call(fn, *args):
    """C-ABI call; tensor arguments are passed as device pointers and stay referenced until the kernel has finished."""
    from sionna_b200._lib import check, ptr, current_stream
    check(getattr(_lib(), fn)(*[ptr(x) if isinstance(x, torch.Tensor) else x for x in args], current_stream()), fn)
    torch.cuda.synchronize()


def _within(what, got, ref, scale, bound=BOUND_ULP):
    """max |got - ref| / (ULP * scale) <= bound; prints the worst value."""
    err = np.abs(np.asarray(got, np.complex128) - ref) / (ULP * np.maximum(scale, np.finfo(np.float32).tiny))
    worst = float(err.max()) if err.size else 0.0
    print(f"{what}: worst {worst:.2f} ulp (bound {bound:g})")
    assert worst <= bound, f"{what}: {worst:.2f} ulp"


def _sizes_and_seeds():
    return [(n, s, o) for n in SIZES for (s, o) in (SEEDS if n < 1000 else SEEDS[1:2])]


@pytest.mark.parametrize("n,seed,offset", _sizes_and_seeds())
def test_binary_source_bits(cuda_device, n, seed, offset):
    from sionna_b200._lib import ptr
    out = torch.full((n + 1,), -1.0, device=cuda_device)
    _call("sb_binary_source", ptr(out), n, seed, offset)
    got = out.cpu().numpy()
    assert np.array_equal(got[:n], R.binary_source(seed, offset, n))
    assert got[n] == -1.0                                            # nothing written past the end


@pytest.mark.parametrize("lo,hi", [(-np.pi, np.pi), (0.0, 1.0), (2.5, 2.5), (-1e-3, 7.0)])
@pytest.mark.parametrize("n,seed,offset", _sizes_and_seeds())
def test_uniform_exact(cuda_device, n, seed, offset, lo, hi):
    from sionna_b200._lib import ptr
    out = torch.full((n + 1,), -7.0, device=cuda_device)
    _call("sb_uniform", ptr(out), n, lo, hi, seed, offset)
    got = out.cpu().numpy()
    ref = R.uniform(seed, offset, n, lo, hi)
    assert np.array_equal(got[:n], ref), f"max diff {np.abs(got[:n] - ref).max()}"
    assert got[n] == -7.0


@pytest.mark.parametrize("mean,std", [(0.0, 1.0), (-3.0, 0.25)])
@pytest.mark.parametrize("n,seed,offset", _sizes_and_seeds())
def test_normal_box_muller(cuda_device, n, seed, offset, mean, std):
    from sionna_b200._lib import ptr
    out = torch.full((n + 1,), -7.0, device=cuda_device)
    _call("sb_normal", ptr(out), n, mean, std, seed, offset)
    got = out.cpu().numpy()
    g = std * R.normal(seed, offset, n)
    _within(f"sb_normal n={n}", got[:n], mean + g, abs(mean) + np.abs(g))
    assert got[n] == -7.0


def _awgn_c(dev, x, no, inner, seed, offset, y=None):
    from sionna_b200._lib import ptr
    y = torch.empty_like(x) if y is None else y
    _call("sb_awgn", ptr(x), ptr(no), inner, ptr(y), x.numel(), seed, offset)
    return y


@pytest.mark.parametrize("n,seed,offset", _sizes_and_seeds())
def test_awgn_values(cuda_device, n, seed, offset):
    """Per-element no (inner = 1), out of place; the element after the end stays untouched."""
    rng = np.random.default_rng(n)
    x = (rng.normal(size=n + 1) + 1j * rng.normal(size=n + 1)).astype(np.complex64)
    no = rng.uniform(0.01, 4.0, n).astype(np.float32)
    xd = torch.from_numpy(x).to(cuda_device)
    y = torch.full((n + 1,), 9.0 + 0j, dtype=torch.complex64, device=cuda_device)
    from sionna_b200._lib import ptr
    _call("sb_awgn", ptr(xd), torch.from_numpy(no).to(cuda_device), 1, ptr(y), n, seed, offset)
    got = y.cpu().numpy()
    w = np.sqrt(no.astype(np.float64) / 2) * R.awgn(seed, offset, n)
    _within(f"sb_awgn n={n}", got[:n], x[:n] + w, np.abs(x[:n]) + np.abs(w))
    assert got[n] == 9.0 + 0j


def test_awgn_in_place(cuda_device):
    """x and y the same buffer (complex_normal draws this way), odd n, one scalar no (inner = n)."""
    n, seed, offset = 1001, SEEDS[1][0], SEEDS[1][1]
    rng = np.random.default_rng(5)
    x = (rng.normal(size=n) + 1j * rng.normal(size=n)).astype(np.complex64)
    buf = torch.from_numpy(x).to(cuda_device)
    no = torch.tensor([0.3], device=cuda_device)
    _awgn_c(cuda_device, buf, no, n, seed, offset, y=buf)
    w = np.sqrt(np.float64(np.float32(0.3)) / 2) * R.awgn(seed, offset, n)
    _within("sb_awgn in place", buf.cpu().numpy(), x + w, np.abs(x) + np.abs(w))


def _take_philox():
    """The (seed, offset) the next block call will receive from config, leaving config's state as it was."""
    from sionna_b200.phy import config
    off0 = config._philox_offset
    seed, off = config.next_philox()
    config._philox_offset = off0
    return seed, off


def _no_patterns(shape, rng):
    """Every form of `no` that _broadcast_inner distinguishes: scalar, leading dimensions (inner > 1), a middle singleton
    (materialised, inner = 1), the full shape. -> list of (label, no array float32)."""
    out = [("scalar", np.float32(0.37))]
    for k in range(1, len(shape)):
        out.append((f"lead{k}", rng.uniform(0.05, 2.0, shape[:k]).astype(np.float32)))
    if len(shape) >= 3:
        mid = list(shape[:3])
        mid[1] = 1
        out.append(("mid1", rng.uniform(0.05, 2.0, mid).astype(np.float32)))
    out.append(("full", rng.uniform(0.05, 2.0, shape).astype(np.float32)))
    return out


def _expand_no(no, shape):
    no = np.asarray(no, np.float64)
    return np.broadcast_to(no.reshape(no.shape + (1,) * (len(shape) - no.ndim)), shape)


def test_awgn_block_every_no_pattern(cuda_device):
    from sionna_b200.phy.channel import AWGN
    shape = (3, 5, 7)                                                # 105 samples: odd n
    rng = np.random.default_rng(11)
    x = (rng.normal(size=shape) + 1j * rng.normal(size=shape)).astype(np.complex64)
    xd = torch.from_numpy(x).to(cuda_device)
    awgn = AWGN()
    for label, no in _no_patterns(shape, rng):
        seed, off = _take_philox()
        y = awgn(xd, torch.as_tensor(no).to(cuda_device)).cpu().numpy()
        w = np.sqrt(_expand_no(no, shape) / 2) * R.awgn(seed, off, x.size).reshape(shape)
        _within(f"AWGN no {label}", y, x + w, np.abs(x) + np.abs(w))


def _rand_c(rng, shape, scale=1.0):
    return ((rng.normal(size=shape) + 1j * rng.normal(size=shape)) * scale / np.sqrt(2)).astype(np.complex64)


@pytest.mark.parametrize("b,rx,ra,tx,ta,s,f", [(2, 2, 3, 1, 2, 3, 37), (1, 1, 1, 1, 1, 1, 1), (3, 1, 2, 2, 1, 14, 72)])
def test_apply_ofdm_channel_noise(cuda_device, b, rx, ra, tx, ta, s, f):
    """y_noisy - y_noiseless = sqrt(no / 2) * channel_noise for every `no` pattern; [b, rx, ra, s] takes the per-element
    path of the kernel (no_inner = f is not a multiple of the RE count), [b, rx, ra] the per-row path."""
    from sionna_b200.phy.channel import ApplyOFDMChannel
    rng = np.random.default_rng(b * 100 + f)
    h = torch.from_numpy(_rand_c(rng, (b, rx, ra, tx, ta, s, f))).to(cuda_device)
    x = torch.from_numpy(_rand_c(rng, (b, tx, ta, s, f))).to(cuda_device)
    app = ApplyOFDMChannel()
    y0 = app(x, h).cpu().numpy()
    shape = y0.shape
    for label, no in _no_patterns(shape, rng):
        seed, off = _take_philox()
        y = app(x, h, torch.as_tensor(no).to(cuda_device)).cpu().numpy()
        w = np.sqrt(_expand_no(no, shape) / 2) * R.channel_noise(seed, off, y.size).reshape(shape)
        _within(f"ApplyOFDMChannel no {label}", y, y0 + w, np.abs(y0) + np.abs(w))


@pytest.mark.parametrize("b,rx,ra,tx,ta,n,l", [(2, 1, 2, 2, 1, 50, 7), (1, 1, 1, 1, 1, 3, 5), (2, 2, 1, 1, 1, 1, 1)])
def test_apply_time_channel_noise(cuda_device, b, rx, ra, tx, ta, n, l):
    from sionna_b200.phy.channel import ApplyTimeChannel
    rng = np.random.default_rng(n * 10 + l)
    h = torch.from_numpy(_rand_c(rng, (b, rx, ra, tx, ta, n + l - 1, l))).to(cuda_device)
    x = torch.from_numpy(_rand_c(rng, (b, tx, ta, n))).to(cuda_device)
    app = ApplyTimeChannel(n, l)
    y0 = app(x, h).cpu().numpy()
    shape = y0.shape
    for label, no in _no_patterns(shape, rng):
        seed, off = _take_philox()
        y = app(x, h, torch.as_tensor(no).to(cuda_device)).cpu().numpy()
        w = np.sqrt(_expand_no(no, shape) / 2) * R.channel_noise(seed, off, y.size).reshape(shape)
        _within(f"ApplyTimeChannel no {label}", y, y0 + w, np.abs(y0) + np.abs(w))


@pytest.mark.parametrize("kernel", ["sb_apply_ofdm_channel", "sb_apply_time_channel"])
def test_channel_noise_c_abi_large_offsets(cuda_device, kernel):
    """Zero input through the C-ABI with a 64-bit seed and offset: y is the scaled noise alone, and element i of the
    output uses counter i."""
    from sionna_b200._lib import ptr
    seed, off = SEEDS[2]
    rng = np.random.default_rng(3)
    bsz, r, tt = 3, 4, 2
    if kernel == "sb_apply_ofdm_channel":
        re = 1000
        x = torch.zeros((bsz, tt, re), dtype=torch.complex64, device=cuda_device)
        h = torch.from_numpy(_rand_c(rng, (bsz, r, tt, re))).to(cuda_device)
        n_out = re
        no = rng.uniform(0.1, 3.0, (bsz, r)).astype(np.float32)
        y = torch.empty((bsz, r, n_out), dtype=torch.complex64, device=cuda_device)
        _call(kernel, ptr(x), ptr(h), torch.from_numpy(no).to(cuda_device), n_out, ptr(y), bsz, r, tt, re, 1, seed, off)
    else:
        n, l = 600, 9
        x = torch.zeros((bsz, tt, n), dtype=torch.complex64, device=cuda_device)
        h = torch.from_numpy(_rand_c(rng, (bsz, r, tt, n + l - 1, l))).to(cuda_device)
        n_out = n + l - 1
        no = rng.uniform(0.1, 3.0, (bsz, r)).astype(np.float32)
        y = torch.empty((bsz, r, n_out), dtype=torch.complex64, device=cuda_device)
        _call(kernel, ptr(x), ptr(h), torch.from_numpy(no).to(cuda_device), n_out, ptr(y), bsz, r, tt, n, l, 1, seed,
              off)
    w = np.sqrt(no.astype(np.float64)[..., None] / 2) * R.channel_noise(seed, off, bsz * r * n_out).reshape(bsz, r, n_out)
    _within(f"{kernel} noise", y.cpu().numpy(), w, np.abs(w))


def test_config_streams_disjoint_and_per_rank(cuda_device):
    """Consecutive draws through config take consecutive offsets (so disjoint counter ranges: the offset is a counter
    word); the blocks that draw use exactly the pair config hands out; per-rank streams mix the rank into the key."""
    from sionna_b200.phy import config
    from sionna_b200.phy.channel.tdl import _uniform
    from sionna_b200.phy.mapping import BinarySource
    from sionna_b200.phy.utils import complex_normal
    config.seed = 1234
    seed, off = config.next_philox()
    config.seed = 1234
    u = _uniform([1000], -1.0, 1.0).cpu().numpy()
    bits = BinarySource()([7, 33]).cpu().numpy()
    z = complex_normal([5, 9], var=2.0).cpu().numpy()
    assert config._philox_offset == off + 3
    assert np.array_equal(u, R.uniform(seed, off, 1000, -1.0, 1.0))
    assert np.array_equal(bits.reshape(-1), R.binary_source(seed, off + 1, 231))
    w = R.awgn(seed, off + 2, 45).reshape(5, 9)
    _within("complex_normal", z, w, np.abs(w))
    assert not np.array_equal(u, R.uniform(seed, off + 1, 1000, -1.0, 1.0))
    # per-rank seed: seed_r = (seed_0 + 0x9E3779B97F4A7C15 * r) mod 2^63, which changes both key words
    try:
        config.seed = 1234
        seeds = []
        for rank in range(3):
            config.rank_offset = rank
            s_r, o_r = config.next_philox()
            config._philox_offset = o_r
            seeds.append(s_r)
            v = _uniform([257], 0.0, 1.0).cpu().numpy()
            assert np.array_equal(v, R.uniform(s_r, o_r, 257, 0.0, 1.0)), rank
        assert seeds[0] == seed
        for rank in (1, 2):
            assert seeds[rank] == (seed + 0x9E3779B97F4A7C15 * rank) & 0x7FFFFFFFFFFFFFFF
            assert (seeds[rank] & 0xFFFFFFFF) != (seed & 0xFFFFFFFF) and (seeds[rank] >> 32) != (seed >> 32)
    finally:
        config.rank_offset = 0
    # a seeded BinarySource keeps its own stream: offsets 0, 1, ... of its own key
    src = BinarySource(seed=99)
    key = (99 * 0x9E3779B97F4A7C15 + 0xABCDEF) & 0x7FFFFFFFFFFFFFFF
    for k in range(2):
        assert np.array_equal(src([300]).cpu().numpy(), R.binary_source(key, k, 300))
