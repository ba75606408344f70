"""Both demapper kernels and the mapper over the whole range they accept, through Mapper / Demapper and the C-ABI.

Every LLR tensor is compared twice:
  * bit for bit with the oracle's kernel-math mode (oracle.mapping.demapper, math_mode=1: the operation order and the
    sb_math.h functions of the kernel that ran);
  * against the float64 reference oracle.mapping.demapper_f64 (the reference's 2-D formula, per-group logsumexp), held
    to the single-precision envelope (oracle.parity.envelope): the kernel's rms and max error, relative to the rms of
    each row's reference LLRs, must be at most 2x and 3x the error of the libm 2-D formula in float32
    (math_mode=0). Every comparison prints its ratios (pytest -s).

Kernels and the cases that reach them (csrc/phy_kernels.cu):
  sb_demap_qam   square QAM and other separable constellations without prior, m = 2 ... 10 (demap_qam.cuh), app and
                 maxlog: noisy points at 40 noise variances from 1e-4 to 3, and inputs whose |LLR| sweeps 60 ... 100,
                 where a bit group's members fall below exp's underflow relative to the dimension's largest exponent
                 (the per-group path); levels that differ between the real and the imaginary dimension; hard_out
  sb_demap       every m = 1 ... 12: PAM, a custom constellation, QAM(12) (never separable), QAM with priors of shape
                 [m], [..., S, m] and [..., 1, m] (the last also through the C-ABI with prior_inner = S)
  both           no as a scalar, per batch row and per symbol; symbol counts 1, 31, 33, 129, 4097 (the warp tails of
                 store_llrs_warp) and one batch longer than a grid pass (the grid-stride loop with a tail);
                 no = 0 and no below float32 tiny, including a dimension whose exponents all overflow to -inf (the
                 reference gives -inf - -inf = NaN there)
  sb_qam_map     m = 1 ... 12, QAM / PAM / custom, tails: points and indices exact
"""
import numpy as np
import pytest
import torch

from oracle import mapping as M
from oracle.parity import constellation, demap_noisy, demap_window, envelope

pytestmark = pytest.mark.gpu

DEFAULT_BAR = (2.0, 3.0)
METHODS = ("app", "maxlog")
TINY = np.finfo(np.float32).tiny


def _run(dem, y, no, dev, prior=None):
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    no_arg = float(no) if np.ndim(no) == 0 else t(np.asarray(no, np.float32))
    return dem(t(y), no_arg, t(prior)).cpu().numpy()


def _check(tag, llr, y, no, pts, method, prior=None, bar=DEFAULT_BAR):
    """llr equals the kernel-math oracle bit for bit and is within the envelope of the float32 2-D formula. Returns ''
    or the failing measurement line."""
    assert np.array_equal(llr, M.demapper(y, no, pts, method, prior=prior, math_mode=1)), f"{tag}: not the oracle's bits"
    return envelope(tag, llr, M.demapper(y, no, pts, method, prior=prior, math_mode=0),
                    M.demapper_f64(y, no, pts, method, prior), bar)


def _separable(dem):
    pts = dem.constellation().to(torch.complex64)
    return dem._separable_levels(pts) is not None


# ---- sb_demap_qam -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("m", [2, 4, 6, 8, 10])
def test_separable_qam(cuda_device, m, method):
    from sionna_b200.phy.mapping import Demapper
    rng = np.random.default_rng(200 + m)
    dem = Demapper(method, "qam", m)
    assert _separable(dem)
    pts = M.qam(m)
    bad = []
    for inputs, gen in (("noisy", demap_noisy), ("window", demap_window)):
        y, no = gen(rng, pts, 256)
        no = no[:, None]                                                    # one noise variance per batch row
        llr = _run(dem, y, no, cuda_device)
        bad.append(_check(f"qam{m} {method} {inputs}", llr, y, no, pts, method))
        if inputs == "window":
            ref = M.demapper_f64(y, no, pts, method)
            assert np.mean((np.abs(ref) > 60) & (np.abs(ref) < 100)) > 0.05
    hard = _run(Demapper(method, "qam", m, hard_out=True), y, no, cuda_device)
    assert np.array_equal(hard, (llr > 0).astype(np.float32))
    assert not any(bad), "\n".join(b for b in bad if b)


def _asym_constellation(m):
    """A separable constellation whose imaginary levels are the real ones reversed and scaled by 0.75."""
    from sionna_b200.phy.mapping import Constellation, separable_levels_np
    h = m // 2
    lev_re, _ = separable_levels_np(M.qam(m), m)
    lev_im = (0.75 * lev_re[::-1]).astype(np.float32)
    j = np.arange(1 << m)
    bits = (j[:, None] >> np.arange(m - 1, -1, -1)) & 1
    w = 1 << np.arange(h - 1, -1, -1)
    pts = (lev_re[bits[:, 0::2] @ w] + 1j * lev_im[bits[:, 1::2] @ w]).astype(np.complex64)
    return Constellation("custom", m, points=pts), lev_re, lev_im


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("m", [4, 6, 8])
def test_separable_levels_that_differ(cuda_device, m, method):
    """Real and imaginary levels differ: the two dimensions cannot be confused. Through Demapper and through the C-ABI
    with the noise variance given once per row (no_inner = S)."""
    from sionna_b200.phy.mapping import Demapper
    from sionna_b200._lib import lib, check, ptr, current_stream
    const, lev_re, lev_im = _asym_constellation(m)
    dem = Demapper(method, constellation=const)
    assert _separable(dem)
    pts = const().cpu().numpy()
    rng = np.random.default_rng(300 + m)
    bad = []
    for inputs, gen in (("noisy", demap_noisy), ("window", demap_window)):
        y, no = gen(rng, pts, 128)
        llr = _run(dem, y, no[:, None], cuda_device)
        bad.append(_check(f"asym{m} {method} {inputs}", llr, y, no[:, None], pts, method))
        yd = torch.from_numpy(y).to(cuda_device)
        nd = torch.from_numpy(no).to(cuda_device)
        lr, li = torch.from_numpy(lev_re).to(cuda_device), torch.from_numpy(lev_im).to(cuda_device)
        out = torch.empty((y.shape[0], y.shape[1] * m), dtype=torch.float32, device=cuda_device)
        check(lib().sb_demap_qam(ptr(yd), ptr(nd), y.shape[1], ptr(lr), ptr(li), m, METHODS.index(method), ptr(out),
                                 y.size, 0, current_stream()), "sb_demap_qam")
        assert np.array_equal(out.cpu().numpy(), llr)
    assert not any(bad), "\n".join(b for b in bad if b)


# ---- sb_demap ---------------------------------------------------------------------------------------------------------
GENERIC = [(m, kind) for m in range(1, 13) for kind in ("pam", "custom")] + [(12, "qam")]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("m,kind", GENERIC, ids=[f"{k}{m}" for m, k in GENERIC])
def test_generic(cuda_device, m, kind, method):
    from sionna_b200.phy.mapping import Demapper
    const = constellation(kind, m)
    dem = Demapper(method, constellation=const)
    assert not _separable(dem)
    pts = const().cpu().numpy()
    rng = np.random.default_rng(400 + m)
    y, no = demap_noisy(rng, pts, 64)
    llr = _run(dem, y, no[:, None], cuda_device)
    bad = _check(f"{kind}{m} {method}", llr, y, no[:, None], pts, method)
    assert not bad, bad


PRIORED = [(m, shape) for m in (2, 4, 6, 8, 10, 12) for shape in ("bits", "full", "lead")]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("m,shape", PRIORED, ids=[f"qam{m}-{s}" for m, s in PRIORED])
def test_generic_priors(cuda_device, m, shape, method):
    """QAM with priors takes the generic kernel. Prior shapes [m], [..., S, m] and [..., 1, m] (broadcast from the
    leading dimensions; also through the C-ABI with one prior row per batch row, prior_inner = S)."""
    from sionna_b200.phy.mapping import Demapper
    from sionna_b200._lib import lib, check, ptr, current_stream
    rng = np.random.default_rng(500 + m)
    pts = M.qam(m)
    y, no = demap_noisy(rng, pts, 64)
    no = no[:, None]
    pshape = {"bits": (m,), "full": y.shape + (m,), "lead": (y.shape[0], 1, m)}[shape]
    prior = (3.0 * rng.normal(size=pshape)).astype(np.float32)
    dem = Demapper(method, "qam", m)
    llr = _run(dem, y, no, cuda_device, prior)
    bad = _check(f"qam{m} {method} prior {shape}", llr, y, no, pts, method, prior)
    if shape == "lead":                                                    # device copies stay referenced until read
        yd, nd, pd, prd = (torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
                           for a in (y, no.reshape(-1), pts, prior.reshape(-1)))
        out = torch.empty(llr.shape, dtype=torch.float32, device=cuda_device)
        check(lib().sb_demap(ptr(yd), ptr(nd), y.shape[1], ptr(pd), m, METHODS.index(method), ptr(prd), y.shape[1],
                             ptr(out), y.size, 0, current_stream()), "sb_demap")
        assert np.array_equal(out.cpu().numpy(), llr)
    assert not bad, bad


# ---- both kernels: noise shapes, launch edges, degenerate noise -------------------------------------------------------
def _both(method, hard_out=False):
    """(tag, Demapper, points, prior) for the separable kernel (16-QAM) and the generic one (16-QAM with a prior)."""
    from sionna_b200.phy.mapping import Demapper
    dem = Demapper(method, "qam", 4, hard_out=hard_out)
    return (("sb_demap_qam", dem, M.qam(4), None),
            ("sb_demap", dem, M.qam(4), np.array([0.5, -1.0, 2.0, 0.0], np.float32)))


@pytest.mark.parametrize("method", METHODS)
def test_noise_shapes(cuda_device, method):
    rng = np.random.default_rng(600)
    pts = M.qam(4)
    y, no_rows = demap_noisy(rng, pts, 96, num_no=6, no_range=(0.01, 1.0))
    bad = []
    for what, no in (("scalar", np.float32(0.05)), ("per batch", no_rows[:, None]),
                     ("per symbol", (no_rows[:, None] * rng.uniform(0.5, 2.0, y.shape)).astype(np.float32))):
        for kern, dem, p, prior in _both(method):
            llr = _run(dem, y, no, cuda_device, prior)
            bad.append(_check(f"{kern} {method} no {what}", llr, y, no, p, method, prior))
    assert not any(bad), "\n".join(b for b in bad if b)


@pytest.mark.parametrize("method", METHODS)
def test_launch_edges(cuda_device, method):
    """Symbol counts around the warp tiles of store_llrs_warp and one batch longer than a grid pass (8 CTAs per SM of
    128 symbols): bit for bit with the kernel-math oracle, hard_out equal to soft > 0."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    big = 300001
    assert big > 2 * 8 * sms * 128 and big % 128
    rng = np.random.default_rng(700)
    for n in (1, 31, 33, 129, 4097, big):
        y = (rng.normal(size=n) + 1j * rng.normal(size=n)).astype(np.complex64)
        no = np.float32(0.1)
        for (kern, dem, p, prior), (_, hdem, _, _) in zip(_both(method), _both(method, hard_out=True)):
            llr = _run(dem, y, no, cuda_device, prior)
            assert llr.shape == (n * 4,)
            assert np.array_equal(llr, M.demapper(y, no, p, method, prior=prior, math_mode=1)), f"{kern} n={n}"
            assert np.array_equal(_run(hdem, y, no, cuda_device, prior), (llr > 0).astype(np.float32)), f"{kern} n={n}"


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("no", [0.0, 1e-39], ids=["zero", "below-tiny"])
def test_degenerate_noise(cuda_device, method, no):
    """no = 0 and no below float32 tiny are floored to tiny. Far from every point all exponents of a dimension overflow
    to -inf and the reference's logsumexp (or max) difference is -inf - -inf = NaN; exactly on a point the LLRs are
    huge (or infinite) with the sign of the point's label bits. Both kernels equal the kernel-math oracle bit for bit,
    NaN for NaN."""
    no = np.float32(no)
    assert no < TINY
    pts = M.qam(4)
    rng = np.random.default_rng(800)
    far = np.array([100 + 100j, -100 + 100j, 100 - 100j, -100 - 100j], np.complex64)
    y = np.concatenate([far, pts, (pts + 1e-3 * (rng.normal(size=16) + 1j * rng.normal(size=16))).astype(np.complex64)])
    for kern, dem, p, prior in _both(method):
        llr = _run(dem, y, no, cuda_device, prior)
        ref = M.demapper(y, no, p, method, prior=prior, math_mode=1)
        assert np.array_equal(llr, ref, equal_nan=True), kern
        assert np.isnan(llr[:4 * 4]).all(), kern                          # the far symbols: every LLR NaN
        bits = (np.arange(16)[:, None] >> np.arange(3, -1, -1)) & 1
        exact = llr[16:16 + 64].reshape(16, 4)
        assert np.array_equal(exact > 0, bits.astype(bool)), kern         # exactly on a point: its label
        assert not np.isnan(llr[16:]).any(), kern


# ---- sb_qam_map -------------------------------------------------------------------------------------------------------
MAPPER = [(m, kind) for m in range(1, 13) for kind in ("qam", "pam", "custom") if kind != "qam" or m % 2 == 0]


@pytest.mark.parametrize("m,kind", MAPPER, ids=[f"{k}{m}" for m, k in MAPPER])
def test_mapper_exact(cuda_device, m, kind):
    from sionna_b200.phy.mapping import Mapper
    const = constellation(kind, m)
    mp = Mapper(constellation=const, return_indices=True)
    pts = const().cpu().numpy()
    rng = np.random.default_rng(900 + m)
    for shape in ((1, 1), (3, 31), (2, 129), (4097,)):
        bits = rng.integers(0, 2, shape[:-1] + (shape[-1] * m,)).astype(np.float32)
        x, idx = mp(torch.from_numpy(bits).to(cuda_device))
        xr, ir = M.mapper(bits, pts)
        assert np.array_equal(x.cpu().numpy(), xr) and np.array_equal(idx.cpu().numpy(), ir), shape
