"""The dense LMMSE kernels over the whole (M antennas, K streams) range they accept, held to the single-precision error
envelope: the error of the CUDA result against complex128 NumPy, relative per element (per vector or matrix for
whitened and factor outputs), must be at most a bar times the error of the same formula evaluated by numpy.linalg in
complex64, in rms and in max. "The same formula" is the reference's step sequence (oracle/ofdm.py: inv_cholesky,
whiten_channel, lmmse_matrix, lmmse_equalizer_cholesky: Cholesky factorisations and cholesky_solve, as
mimo/equalization.py and mimo/utils.py evaluate them), run once in complex128 and once in complex64.

The bar is 2x (rms) / 3x (max) unless BARS names an exception. Worst ratios measured on an H100 80GB HBM3 are given
beside each bar. The exceptions are results that the kernels obtain by forward substitution (whiten_channel,
inv_cholesky and the whitening inside lmmse_equalizer), where the reference forms L^-1 and multiplies. Another is
the register kernel's x_hat, which whitens with rsqrt (<= 2 ulp) and solves through A^-1 = C^-H C^-1. The last is
the square systems M = K, where the condition number of H amplifies any difference in rounding. An arithmetic
slip (the wrong operand conjugated in the Cholesky solve) makes the ratio about 10^6.

Entry points and the branches they reach (csrc/ofdm_mimo.cu):
  lmmse_equalizer(whiten_interference=True)    sb_lmmse_equalize -> lmmse_kernel (lmmse_core)
  lmmse_equalizer(whiten_interference=False)   sb_mimo_linalg mode 3: (H H^H + S) Cholesky, chol_solve_col, epilogue
  lmmse_matrix(h, s) / lmmse_matrix(h)         sb_mimo_linalg mode 2, receive side (M x M) / transmit side (K x K)
  whiten_channel, inv_cholesky                 sb_mimo_linalg modes 1 / 0
  LMMSEEqualizer                               sb_ofdm_lmmse: ofdm_lmmse_diag_kernel<K> for K <= 4 streams without
                                               interferers (antennas in chunks of 4, then a tail loop), else
                                               ofdm_lmmse_kernel (lmmse_core)
Tests per branch: test_lmmse_equalizer_envelope (lmmse_kernel, mode 3), test_whiten_channel_and_lmmse_matrix_envelope
(modes 1, 2), test_inv_cholesky_envelope (mode 0), test_ofdm_lmmse_equalizer_envelope[M-K-False] with K <= 4 (diag
kernel: M < 4 tail loop only, M = 5, 6, 7, 13 both loops, M = 32, 64 chunks only), [M-{5,8,16}-False] and
[32-{1,4}-True] (ofdm_lmmse_kernel without / with interferers), test_lmmse_shapes_beyond_the_scratch_limit_are_refused.
The thread-per-vector kernels keep their matrices in shared memory; from M = 24 at K = 4, or K >= 15 at any M, fewer
than 32 vectors fit in a CTA and the launch uses 16 ... 1 threads. Batches of 1 and 33 vectors (a partly filled CTA)
must return exactly the first rows of the 4097-vector batch.
"""
import numpy as np
import pytest
import torch

from oracle import mapping as MAP
from oracle import ofdm as F
from oracle.parity import cnormal, envelope, mimo_problem, noise_covariance

pytestmark = pytest.mark.gpu

KS = (1, 2, 3, 4, 5, 8, 12, 15, 16)
PAIRS = [(m, k) for k in KS for m in sorted({k, k + 1, 13, 16, 23, 24, 32}) if m >= k]
NUM = 4097
NO = 10 ** (-15.0 / 10)                         # 15 dB
DEFAULT_BAR = (2.0, 3.0)
BARS = {                                        # (rms, max) bar: worst measured ratio
    "lmmse_equalizer": (2.5, 3.5),              # tall systems 2.01 / 3.00 (whitening by forward substitution)
    "lmmse_equalizer square": (3.2, 4.3),       # M = K: 2.65 / 3.55 (x_hat at M = K = 15)
    "whiten_channel": (3.0, 6.0),               # forward substitution: whitened H 2.42 / 4.88, y 1.95 / 2.98
    "inv_cholesky": (2.5, 4.2),                 # column-wise forward substitution: 1.91 / 3.42
    "ofdm diag x_hat": (3.2, 4.0),              # register kernel: 2.65 / 3.34
}                                               # default: lmmse_matrix 1.58 / 2.36, ofdm general 1.64 / 1.96,
                                                # ofdm diag no_eff 1.44 / 1.68


def _prefix_identical(fn, args, full):
    """fn on the first 1 and 33 vectors returns exactly the first rows of fn on all of them."""
    for num in (1, 33):
        part = fn(*(a[:num] for a in args))
        for p, f in zip(part if isinstance(part, tuple) else (part,), full if isinstance(full, tuple) else (full,)):
            assert torch.equal(p, f[:num]), num


@pytest.mark.parametrize("whiten", [True, False])
@pytest.mark.parametrize("m,k", PAIRS)
def test_lmmse_equalizer_envelope(cuda_device, m, k, whiten):
    from sionna_b200.phy.mimo import lmmse_equalizer
    rng = np.random.default_rng(1000 * m + 10 * k + whiten)
    y, h, s = mimo_problem(rng, NUM, m, k, MAP.qam(4), NO)
    x64, n64 = F.lmmse_equalizer_cholesky(y.astype(np.complex128), h.astype(np.complex128), s.astype(np.complex128),
                                          whiten)
    x32, n32 = F.lmmse_equalizer_cholesky(y, h, s, whiten)
    args = tuple(torch.from_numpy(v).to(cuda_device) for v in (y, h, s))
    fn = lambda y_, h_, s_: lmmse_equalizer(y_, h_, s_, whiten_interference=whiten)   # noqa: E731
    xg, ng = fn(*args)
    bar = BARS["lmmse_equalizer square" if m == k else "lmmse_equalizer"]
    bad = [envelope(f"x_hat M={m} K={k} whiten={whiten}", xg.cpu().numpy(), x32, x64, bar, scale=np.abs(x64)),
           envelope(f"no_eff M={m} K={k} whiten={whiten}", ng.cpu().numpy(), n32, n64, bar, scale=np.abs(n64))]
    _prefix_identical(fn, args, (xg, ng))
    assert not any(bad), "\n".join(b for b in bad if b)


@pytest.mark.parametrize("m,k", PAIRS)
def test_whiten_channel_and_lmmse_matrix_envelope(cuda_device, m, k):
    from sionna_b200.phy.mimo import whiten_channel, lmmse_matrix
    rng = np.random.default_rng(2000 * m + k)
    y, h, s = mimo_problem(rng, NUM, m, k, MAP.qam(4), NO)
    mats = (-2, -1)
    c128 = [v.astype(np.complex128) for v in (y, h, s)]
    yd, hd, sd = (torch.from_numpy(v).to(cuda_device) for v in (y, h, s))
    yw, hw, _ = whiten_channel(yd, hd, sd)
    (yw64, hw64), (yw32, hw32) = F.whiten_channel(*c128), F.whiten_channel(y, h, s)
    bad = [envelope(f"whiten y M={m} K={k}", yw.cpu().numpy(), yw32, yw64, BARS["whiten_channel"], axis=-1),
           envelope(f"whiten H M={m} K={k}", hw.cpu().numpy(), hw32, hw64, BARS["whiten_channel"], axis=mats)]
    _prefix_identical(lambda *a: whiten_channel(*a, return_s=False), (yd, hd, sd), (yw, hw))
    g = lmmse_matrix(hd, sd)
    bad.append(envelope(f"lmmse_matrix(h, s) M={m} K={k}", g.cpu().numpy(), F.lmmse_matrix(h, s),
                        F.lmmse_matrix(c128[1], c128[2]), DEFAULT_BAR, axis=mats))
    _prefix_identical(lmmse_matrix, (hd, sd), g)
    g = lmmse_matrix(hd)
    bad.append(envelope(f"lmmse_matrix(h) M={m} K={k}", g.cpu().numpy(), F.lmmse_matrix(h), F.lmmse_matrix(c128[1]),
                        DEFAULT_BAR, axis=mats))
    _prefix_identical(lmmse_matrix, (hd,), g)
    assert not any(bad), "\n".join(b for b in bad if b)


@pytest.mark.parametrize("m", sorted({m for m, _ in PAIRS}))
def test_inv_cholesky_envelope(cuda_device, m):
    from sionna_b200.phy.utils import inv_cholesky
    rng = np.random.default_rng(3000 + m)
    s = noise_covariance(rng, NUM, m, 1.0)
    sd = torch.from_numpy(s).to(cuda_device)
    li = inv_cholesky(sd)
    ref = F.inv_cholesky(s.astype(np.complex128))
    f32 = F.inv_cholesky(s)
    assert f32.dtype == np.complex64
    got = li.cpu().numpy()
    assert np.all(np.triu(got, 1) == 0)
    bad = envelope(f"inv_cholesky M={m}", got, f32, ref, BARS["inv_cholesky"], axis=(-2, -1))
    _prefix_identical(inv_cholesky, (sd,), li)
    assert not bad, bad


def _ofdm_cases():
    for k in (1, 2, 3, 4):                       # register kernel: chunks of 4 antennas, then the tail loop
        for m in sorted({k, 5, 6, 7, 13, 32, 64}):
            if m >= k:
                yield m, k, False
    for k in (5, 8, 16):                         # shared-memory kernel, no interferers
        for m in sorted({k, 32}):
            yield m, k, False
    for k in (1, 4):                             # shared-memory kernel, interference from a second transmitter
        yield 32, k, True


@pytest.mark.parametrize("m,k,interf", list(_ofdm_cases()))
def test_ofdm_lmmse_equalizer_envelope(cuda_device, m, k, interf):
    """LMMSEEqualizer on a Kronecker-pilot grid of 3 OFDM symbols (one carries pilots only, so its REs are skipped):
    8 batches x 3 symbols x F subcarriers, F the multiple of the stream count nearest 60 (not a multiple of 128
    resource elements). With interference there are two transmitters and two receivers, each receiver decoding one
    transmitter's K streams and treating the other's as interference."""
    from sionna_b200.phy.ofdm import LMMSEEqualizer, ResourceGrid
    from sionna_b200.phy.mimo import StreamManagement
    num_tx, rx = (2, 2) if interf else (1, 1)
    assoc = np.eye(2, dtype=int) if interf else np.ones((1, 1), int)
    txs = num_tx * k
    f_ = txs * max(1, round(60 / txs))
    b, s_ = 8, 3
    rg = ResourceGrid(s_, f_, 15e3, num_tx=num_tx, num_streams_per_tx=k, pilot_pattern="kronecker",
                      pilot_ofdm_symbol_indices=[1])
    sm = StreamManagement(assoc, k)
    rng = np.random.default_rng(4000 + 100 * m + 10 * k + interf)
    h = cnormal(rng, (b, rx, m, num_tx, k, s_, f_))
    x = MAP.qam(4)[rng.integers(0, 16, (b, num_tx, k, s_, f_))]
    no = rng.uniform(0.02, 0.06, size=(b, rx, m)).astype(np.float32)
    y = np.einsum("brmtksf,btksf->brmsf", h.astype(np.complex128), x)
    y = (y + cnormal(rng, y.shape) * np.sqrt(no)[..., None, None]).astype(np.complex64)
    ev = (0.01 * rng.uniform(size=h.shape)).astype(np.float32)
    mask = rg.pilot_pattern.mask.astype(bool)
    smr = F.stream_management(assoc, k)
    x64, n64 = F.ofdm_lmmse_equalize(y.astype(np.complex128), h.astype(np.complex128), ev.astype(np.float64), no,
                                     mask, smr)
    x32, n32 = F.ofdm_lmmse_equalize_f32(y, h, ev, no, mask, smr)
    eq = LMMSEEqualizer(rg, sm)
    args = [torch.from_numpy(v).to(cuda_device) for v in (y, h, ev, no)]
    xg, ng = eq(*args)
    assert xg.shape == x64.shape == (b, num_tx, k, rg.num_data_symbols)
    diag = not interf and k <= 4
    bad = [envelope(f"ofdm x_hat M={m} K={k} interf={interf}", xg.cpu().numpy(), x32, x64,
                    BARS["ofdm diag x_hat"] if diag else DEFAULT_BAR, scale=np.abs(x64)),
           envelope(f"ofdm no_eff M={m} K={k} interf={interf}", ng.cpu().numpy(), n32, n64, DEFAULT_BAR,
                    scale=np.abs(n64))]
    x1, n1 = eq(*(a[:1] for a in args))
    assert torch.equal(x1, xg[:1]) and torch.equal(n1, ng[:1])
    assert not any(bad), "\n".join(b for b in bad if b)


def test_lmmse_shapes_beyond_the_scratch_limit_are_refused(cuda_device):
    """A matrix whose per-vector scratch exceeds the shared-memory cap returns the library's error naming the limit."""
    from sionna_b200._lib import SbError
    from sionna_b200.phy.mimo import lmmse_equalizer
    from sionna_b200.phy.utils import inv_cholesky
    m, k = 159, 1                                 # 8 (M^2 + 3 M + 1) bytes > 200 KB
    y = torch.zeros((1, m), dtype=torch.complex64, device=cuda_device)
    h = torch.zeros((1, m, k), dtype=torch.complex64, device=cuda_device)
    s = torch.eye(m, dtype=torch.complex64, device=cuda_device)[None]
    with pytest.raises(SbError, match="the limit is 204800"):
        lmmse_equalizer(y, h, s)
    with pytest.raises(SbError, match="shared-memory scratch per matrix"):
        inv_cholesky(torch.eye(99, dtype=torch.complex64, device=cuda_device)[None])
