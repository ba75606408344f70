"""ZF / MF equalisation, the pseudo-inverse, unwhitened OFDM LMMSE, SymbolDemapper and LinearDetector on the GPU.

Envelope tests hold each kernel to the single-precision error envelope of oracle/parity.py: its error against the
complex128 / float64 evaluation of the reference's step sequence (oracle/linear.py) must be at most a bar times the
error of the same sequence evaluated in complex64 / float32, in rms and in max. The bar is 2x (rms) / 3x (max) unless
BARS names an exception, with the worst ratio measured on an H100 80GB HBM3 beside it.

Entry points and the branches they reach (csrc/ofdm_mimo.cu, csrc/phy_kernels.cu):
  zf_equalizer / mf_equalizer / matrix_pinv       sb_mimo_linalg modes 4 / 5 / 6
  ZFEqualizer, MFEqualizer                        sb_ofdm_equalize: ofdm_linear_diag_kernel<EQ, K> for K <= 4 streams
                                                  without interferers (antennas in chunks of 4, then a tail loop), else
                                                  ofdm_linear_kernel<EQ>
  LMMSEEqualizer(whiten_interference=False)       sb_ofdm_equalize: the LMMSE register kernel for K <= 4 without
                                                  interferers and M >= K + 2, else ofdm_linear_kernel<1>
  SymbolDemapper                                  sb_symbol_demap: symbol_demap_kernel<G>, G = min(P, 32) lanes/symbol
"""
import numpy as np
import pytest
import torch

from oracle import linear as L
from oracle import mapping as MAP
from oracle import ofdm as F
from oracle.parity import cnormal, constellation, demap_noisy, demap_window, envelope, mimo_problem

pytestmark = pytest.mark.gpu

KS = (1, 2, 3, 4, 5, 8, 12, 15, 16)
PAIRS = [(m, k) for k in KS for m in sorted({k, k + 1, 13, 16, 23, 24, 32}) if m >= k]
NUM = 4097
NO = 10 ** (-15.0 / 10)                         # 15 dB
DEFAULT_BAR = (2.0, 3.0)
BARS = {                                        # (rms, max) bar, the shapes it applies to: worst measured ratio
    "zf square": (6.0, 6.5),                    # dense, M <= K + 1: 5.47 / 5.67 at M = K = 16 (cond(H^H H) = cond(H)^2)
    "pinv square": (5.0, 5.5),                  # M <= K + 1: 4.53 / 4.69 at M = K = 16
    "mf M=32": (2.5, 3.0),                      # dense, M = 32: 2.02 / 2.17 at K = 1 (sums over M in one chain)
    "ofdm zf": (4.0, 5.0),                      # OFDM, M <= K + 1 or the shared-memory kernel (interferers or K > 4):
}                                               # 3.44 / 4.31 at M = K = 8, 2.23 / 4.12 at M = 32, K = 1 with interferers
# default bar elsewhere: dense zf tall 1.70 / 1.84, dense mf M < 32 below 2 / 3, pinv tall 1.46 / 1.84, OFDM zf tall
# register kernel 1.67 / 2.50, OFDM mf 1.88 / 2.55, SymbolDemapper 0.81 / 1.18


def _dense_bar(name, m, k):
    if name == "zf" and m <= k + 1:
        return BARS["zf square"]
    if name == "mf" and m >= 32:
        return BARS["mf M=32"]
    return DEFAULT_BAR


def _ofdm_bar(eq, m, k, interf):
    if eq == "zf" and (m <= k + 1 or interf or k > 4):
        return BARS["ofdm zf"]
    return DEFAULT_BAR


def _prefix_identical(fn, args, full):
    """fn on the first 1 and 33 problems returns exactly the first rows of fn on all of them."""
    for num in (1, 33):
        part = fn(*(a[:num] for a in args))
        for p, f in zip(part if isinstance(part, tuple) else (part,), full if isinstance(full, tuple) else (full,)):
            assert torch.equal(p, f[:num]), num


# ---- dense ZF / MF / pinv ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,k", PAIRS)
def test_dense_zf_mf_pinv_envelope(cuda_device, m, k):
    from sionna_b200.phy.mimo import zf_equalizer, mf_equalizer
    from sionna_b200.phy.utils import matrix_pinv
    rng = np.random.default_rng(5000 * m + k)
    y, h, s = mimo_problem(rng, NUM, m, k, MAP.qam(4), NO)
    c128 = [v.astype(np.complex128) for v in (y, h, s)]
    args = tuple(torch.from_numpy(v).to(cuda_device) for v in (y, h, s))
    bad = []
    for name, fn, ref in (("zf", zf_equalizer, L.zf_equalizer), ("mf", mf_equalizer, L.mf_equalizer)):
        xg, ng = fn(*args)
        (x64, n64), (x32, n32) = ref(*c128), ref(y, h, s)
        bar = _dense_bar(name, m, k)
        bad += [envelope(f"{name} x_hat M={m} K={k}", xg.cpu().numpy(), x32, x64, bar, axis=-1),
                envelope(f"{name} no_eff M={m} K={k}", ng.cpu().numpy(), n32, n64, bar, scale=np.abs(n64))]
        _prefix_identical(fn, args, (xg, ng))
    g = matrix_pinv(args[1])
    assert g.shape == (NUM, k, m)
    bad.append(envelope(f"matrix_pinv M={m} K={k}", g.cpu().numpy(), L.matrix_pinv(h), L.matrix_pinv(c128[1]),
                        BARS["pinv square"] if m <= k + 1 else DEFAULT_BAR, axis=(-2, -1)))
    _prefix_identical(matrix_pinv, (args[1],), g)
    assert not any(bad), "\n".join(b for b in bad if b)


# ---- OFDM equalisers --------------------------------------------------------------------------------------------------
def _ofdm_cases():
    for k in (1, 2, 3, 4):                       # register kernel: M < 4 tail loop only, 5 / 13 both loops, 32 chunks
        for m in sorted({k, 5, 13, 32}):
            yield m, k, False, False
    for k in (5, 8):                             # shared-memory kernel, no interferers
        for m in sorted({k, 32}):
            yield m, k, False, False
    for k in (1, 4):                             # shared-memory kernel, interference from a second transmitter
        yield 32, k, True, False
    yield 13, 2, False, True                     # broadcast err_var / no, register kernel
    yield 16, 2, True, True                      # broadcast err_var / no, shared-memory kernel


def _ofdm_problem(m, k, interf, bcast, seed):
    from sionna_b200.phy.ofdm import ResourceGrid
    from sionna_b200.phy.mimo import StreamManagement
    num_tx, rx = (2, 2) if interf else (1, 1)
    assoc = np.eye(2, dtype=int) if interf else np.ones((1, 1), int)
    txs = num_tx * k
    f_ = txs * max(1, round(60 / txs))
    b, s_ = 8, 3
    rg = ResourceGrid(s_, f_, 15e3, num_tx=num_tx, num_streams_per_tx=k, pilot_pattern="kronecker",
                      pilot_ofdm_symbol_indices=[1])
    sm = StreamManagement(assoc, k)
    rng = np.random.default_rng(seed)
    h = cnormal(rng, (b, rx, m, num_tx, k, s_, f_))
    x = MAP.qam(4)[rng.integers(0, 16, (b, num_tx, k, s_, f_))]
    no = rng.uniform(0.02, 0.06, size=(b, rx, m)).astype(np.float32)
    y = np.einsum("brmtksf,btksf->brmsf", h.astype(np.complex128), x)
    y = (y + cnormal(rng, y.shape) * np.sqrt(no)[..., None, None]).astype(np.complex64)
    ev = (0.01 * rng.uniform(size=h.shape)).astype(np.float32)
    if bcast:                                    # err_var one value per (tx, stream), no one value per batch
        ev = np.ascontiguousarray(ev[:1, :1, :1, :, :, :1, :1])
        no = np.ascontiguousarray(no[:, 0, 0])
    return rg, sm, F.stream_management(assoc, k), y, h, ev, no


@pytest.mark.parametrize("eq", ["zf", "mf", "lmmse-no-whitening"])
@pytest.mark.parametrize("m,k,interf,bcast", list(_ofdm_cases()))
def test_ofdm_equalizer_envelope(cuda_device, eq, m, k, interf, bcast):
    from sionna_b200.phy.ofdm import ZFEqualizer, MFEqualizer, LMMSEEqualizer
    rg, sm, smr, y, h, ev, no = _ofdm_problem(m, k, interf, bcast, 6000 + 100 * m + 10 * k + interf + 2 * bcast)
    mask = rg.pilot_pattern.mask.astype(bool)
    x64, n64 = L.ofdm_equalize(y.astype(np.complex128), h.astype(np.complex128), ev.astype(np.float64),
                               np.asarray(no, np.float64), mask, smr, eq)
    x32, n32 = L.ofdm_equalize(y, h, ev, no, mask, smr, eq, np.complex64)
    blk = {"zf": lambda: ZFEqualizer(rg, sm), "mf": lambda: MFEqualizer(rg, sm),
           "lmmse-no-whitening": lambda: LMMSEEqualizer(rg, sm, whiten_interference=False)}[eq]()
    args = [torch.from_numpy(np.asarray(v)).to(cuda_device) for v in (y, h, ev, no)]
    xg, ng = blk(*args)
    assert xg.shape == x64.shape
    bar = _ofdm_bar(eq, m, k, interf)
    what = f"ofdm {eq} M={m} K={k} interf={interf} bcast={bcast}"
    bad = [envelope(f"{what} x_hat", xg.cpu().numpy(), x32, x64, bar, scale=np.abs(x64)),
           envelope(f"{what} no_eff", ng.cpu().numpy(), n32, n64, bar, scale=np.abs(n64))]
    x1, n1 = blk(*([a[:1] for a in args[:3]] + [args[3][:1] if args[3].dim() else args[3]]))
    assert torch.equal(x1, xg[:1]) and torch.equal(n1, ng[:1])
    if not bcast:
        x33, n33 = blk(*([a[:33] for a in args]))
        assert torch.equal(x33, xg[:33]) and torch.equal(n33, ng[:33])
    assert not any(bad), "\n".join(b for b in bad if b)


@pytest.mark.parametrize("eq", ["zf", "mf"])
def test_ofdm_unfused_route_matches_the_fused_kernel(cuda_device, eq):
    """OFDMEqualizer with this library's own zf_equalizer / mf_equalizer as a callable (the unfused route, explicit S)
    gives the fused kernel's results within the envelope."""
    from sionna_b200.phy.ofdm import ZFEqualizer, MFEqualizer, OFDMEqualizer
    from sionna_b200.phy.mimo import zf_equalizer, mf_equalizer
    rg, sm, smr, y, h, ev, no = _ofdm_problem(16, 2, True, False, 77)
    mask = rg.pilot_pattern.mask.astype(bool)
    x64, n64 = L.ofdm_equalize(y.astype(np.complex128), h.astype(np.complex128), ev.astype(np.float64),
                               no.astype(np.float64), mask, smr, eq)
    x32, n32 = L.ofdm_equalize(y, h, ev, no, mask, smr, eq, np.complex64)
    args = [torch.from_numpy(v).to(cuda_device) for v in (y, h, ev, no)]
    fused = (ZFEqualizer if eq == "zf" else MFEqualizer)(rg, sm)(*args)
    unfused = OFDMEqualizer(zf_equalizer if eq == "zf" else mf_equalizer, rg, sm)(*args)
    bad = []
    bar = _ofdm_bar(eq, 16, 2, True)
    for name, (xg, ng) in (("fused", fused), ("unfused", unfused)):
        bad += [envelope(f"{eq} {name} x_hat", xg.cpu().numpy(), x32, x64, bar, scale=np.abs(x64)),
                envelope(f"{eq} {name} no_eff", ng.cpu().numpy(), n32, n64, bar, scale=np.abs(n64))]
    assert not any(bad), "\n".join(b for b in bad if b)


@pytest.mark.parametrize("eq", ["zf", "mf", "lmmse-no-whitening"])
def test_ofdm_shapes_beyond_the_limits_are_refused(cuda_device, eq):
    """A receiver with interferers whose per-element scratch exceeds 200 KB, and more streams than antennas, raise
    ValueError with the library's message."""
    from sionna_b200.phy.ofdm import ZFEqualizer, MFEqualizer, LMMSEEqualizer
    cls = {"zf": ZFEqualizer, "mf": MFEqualizer,
           "lmmse-no-whitening": lambda r, s: LMMSEEqualizer(r, s, whiten_interference=False)}[eq]
    rg, sm, _, y, h, ev, no = _ofdm_problem(160, 1, True, False, 1)
    args = [torch.from_numpy(v).to(cuda_device) for v in (y[:1], h[:1], ev[:1], no[:1])]
    with pytest.raises(ValueError, match="the limit is 204800"):
        cls(rg, sm)(*args)
    rg, sm, _, y, h, ev, no = _ofdm_problem(4, 4, False, False, 2)
    args = [torch.from_numpy(v).to(cuda_device) for v in (y[:1, :, :3], h[:1, :, :3], ev[:1, :, :3], no[:1, :, :3])]
    with pytest.raises(ValueError, match="4 streams per receiver with 3 receive antennas"):
        cls(rg, sm)(*args)


def test_dense_shapes_beyond_the_scratch_limit_are_refused(cuda_device):
    """zf_equalizer, mf_equalizer and matrix_pinv with more per-matrix scratch than the device offers raise a
    ValueError (the library's SbUnsupportedError) with the library's message."""
    from sionna_b200.phy.mimo import zf_equalizer, mf_equalizer
    from sionna_b200.phy.utils import matrix_pinv
    m, k = 170, 1                                 # 8 (M^2 + 2 M K) bytes > 227 KB
    y = torch.zeros((1, m), dtype=torch.complex64, device=cuda_device)
    h = torch.ones((1, m, k), dtype=torch.complex64, device=cuda_device)
    s = torch.eye(m, dtype=torch.complex64, device=cuda_device)[None]
    for call in (lambda: zf_equalizer(y, h, s), lambda: mf_equalizer(y, h, s), lambda: matrix_pinv(h)):
        with pytest.raises(ValueError, match="shared-memory scratch per matrix"):
            call()


# ---- SymbolDemapper ---------------------------------------------------------------------------------------------------
SYM_CASES = [("qam", m) for m in (2, 4, 6, 8, 10)] + [("pam", 3), ("custom", 4)]
# hard decisions are compared where the float64 top-two gap exceeds this many fp32 ulps of the largest |exponent|
TIE_ULPS = 64


def _sym_inputs(kind, m, rng, window):
    pts = constellation(kind, m)
    p = pts().cpu().numpy()
    y, no = (demap_window if window else demap_noisy)(rng, p, 257)
    return pts, p, y, no


@pytest.mark.parametrize("prior_kind", [None, "points", "per_symbol"])
@pytest.mark.parametrize("window", [False, True])
@pytest.mark.parametrize("kind,m", SYM_CASES)
def test_symbol_demapper_envelope(cuda_device, kind, m, window, prior_kind):
    from sionna_b200.phy.mapping import SymbolDemapper
    rng = np.random.default_rng(7000 + 10 * m + window + 3 * (prior_kind is not None))
    pts, p, y, no = _sym_inputs(kind, m, rng, window)
    npts = len(p)
    prior = None
    if prior_kind == "points":
        prior = rng.normal(size=npts).astype(np.float32)
    elif prior_kind == "per_symbol":
        prior = rng.normal(size=y.shape + (npts,)).astype(np.float32)
    bad = []
    for no_arg in (no[:, None], np.float32(no[len(no) // 2])):            # per row of symbols, scalar
        ref = L.symbol_demap(y, no_arg, p, prior)
        f32 = L.symbol_demap(y, no_arg, p, prior, dtype=np.float32)
        yd = torch.from_numpy(y).to(cuda_device)
        nod = torch.as_tensor(no_arg).to(cuda_device)
        pd = None if prior is None else torch.from_numpy(prior).to(cuda_device)
        got = SymbolDemapper(constellation=pts)(yd, nod, pd)
        assert got.shape == y.shape + (npts,) and got.dtype == torch.float32
        bad.append(envelope(f"symbol logits {kind}{m} window={window} prior={prior_kind} no={np.ndim(no_arg)}",
                            got.cpu().numpy(), f32, ref, DEFAULT_BAR, axis=-1))
        hard = SymbolDemapper(constellation=pts, hard_out=True)(yd, nod, pd).cpu().numpy()
        assert hard.dtype == np.int32 and hard.shape == y.shape
        e = ref                                                            # log_softmax keeps the order of e
        srt = np.sort(e, axis=-1)
        gap = srt[..., -1] - srt[..., -2]
        lead = np.max(np.abs(e), axis=-1)
        clear = gap > TIE_ULPS * np.spacing(np.maximum(lead, 1.0).astype(np.float32))
        assert clear.mean() > 0.5
        np.testing.assert_array_equal(hard[clear], np.argmax(e, axis=-1)[clear])
    assert not any(bad), "\n".join(b for b in bad if b)


def test_symbol_demapper_tails_and_ties(cuda_device):
    """Symbol counts around the warp and grid tails return the first rows of the larger batch exactly; exact ties
    (y on the axis between two points) resolve to the first maximum."""
    from sionna_b200.phy.mapping import SymbolDemapper
    rng = np.random.default_rng(3)
    for kind, m in (("qam", 2), ("qam", 4), ("qam", 8)):
        pts = constellation(kind, m)
        y = torch.from_numpy(cnormal(rng, (300001,))).to(cuda_device)
        full = SymbolDemapper(constellation=pts)(y, 0.5)
        for n in (1, 31, 33, 129, 4097):
            assert torch.equal(SymbolDemapper(constellation=pts)(y[:n], 0.5), full[:n])
    pts = constellation("qam", 2)
    yt = torch.zeros(5, dtype=torch.complex64, device=cuda_device)     # equidistant from all four QPSK points
    hard = SymbolDemapper(constellation=pts, hard_out=True)(yt, 1.0)
    assert torch.equal(hard.cpu(), torch.zeros(5, dtype=torch.int32))


# ---- LinearDetector = equaliser + (Symbol)Demapper --------------------------------------------------------------------
COMBOS = [(eq, out, hard) for eq in ("lmmse", "zf", "mf") for out in ("bit", "symbol") for hard in (False, True)]


@pytest.mark.parametrize("eq,output,hard_out", COMBOS)
def test_dense_linear_detector_is_the_composition(cuda_device, eq, output, hard_out):
    from sionna_b200.phy.mimo import LinearDetector, lmmse_equalizer, zf_equalizer, mf_equalizer
    from sionna_b200.phy.mapping import Demapper, SymbolDemapper
    rng = np.random.default_rng(11)
    y, h, s = (torch.from_numpy(v).to(cuda_device) for v in mimo_problem(rng, 513, 8, 4, MAP.qam(4), 0.1))
    det = LinearDetector(eq, output, "maxlog", "qam", 4, hard_out=hard_out)
    got = det(y, h, s)
    x_hat, no_eff = {"lmmse": lmmse_equalizer, "zf": zf_equalizer, "mf": mf_equalizer}[eq](y, h, s)
    if output == "bit":
        ref = Demapper("maxlog", "qam", 4, hard_out=hard_out)(x_hat, no_eff).reshape(513, 4, 4)
    else:
        ref = SymbolDemapper("qam", 4, hard_out=hard_out)(x_hat, no_eff)
        assert got.shape == ((513, 4) if hard_out else (513, 4, 16))
    assert torch.equal(got, ref)


@pytest.mark.parametrize("eq,output,hard_out", COMBOS)
def test_ofdm_linear_detector_is_the_composition(cuda_device, eq, output, hard_out):
    from sionna_b200.phy.ofdm import LinearDetector, LMMSEEqualizer, ZFEqualizer, MFEqualizer
    from sionna_b200.phy.mapping import Demapper, SymbolDemapper
    rg, sm, _, y, h, ev, no = _ofdm_problem(8, 2, True, False, 12)
    args = [torch.from_numpy(v).to(cuda_device) for v in (y, h, ev, no)]
    got = LinearDetector(eq, output, "app", rg, sm, "qam", 4, hard_out=hard_out)(*args)
    x_hat, no_eff = {"lmmse": LMMSEEqualizer, "zf": ZFEqualizer, "mf": MFEqualizer}[eq](rg, sm)(*args)
    if output == "bit":
        ref = Demapper("app", "qam", 4, hard_out=hard_out)(x_hat, no_eff)
    else:
        ref = SymbolDemapper("qam", 4, hard_out=hard_out)(x_hat, no_eff)
        assert got.shape == tuple(x_hat.shape) + (() if hard_out else (16,))
    assert torch.equal(got, ref)


def test_linear_detector_accepts_every_pair_and_a_callable(cuda_device):
    from sionna_b200.phy.ofdm import LinearDetector
    from sionna_b200.phy.mimo import zf_equalizer
    rg, sm, _, y, h, ev, no = _ofdm_problem(4, 2, False, False, 13)
    args = [torch.from_numpy(v).to(cuda_device) for v in (y, h, ev, no)]
    for eq in ("lmmse", "zf", "mf", zf_equalizer):
        for out in ("bit", "symbol"):
            z = LinearDetector(eq, out, "maxlog", rg, sm, "qam", 4, hard_out=True)(*args)
            assert z.shape[:3] == (8, 1, 2)
    with pytest.raises(AssertionError, match="Unknown equalizer"):
        LinearDetector("zz", "bit", "maxlog", rg, sm, "qam", 4)


# ---- error statistics (test/unit/mimo/test_mimo_equalizers.py) --------------------------------------------------------
STAT_BATCH = 200_000
STAT_SIGMAS = 5.0                                # tolerance in standard errors of the estimate


@pytest.mark.parametrize("colored", [False, True])
@pytest.mark.parametrize("no", [0.01, 0.1, 1, 3, 10])
@pytest.mark.parametrize("eq", ["zf", "mf"])
def test_error_statistics(cuda_device, eq, no, colored):
    """4 streams, 8 antennas, 16-QAM, AWGN or coloured noise S = no I + R (R_ij = 0.95^|i-j|): the error x - x_hat has
    zero mean and its mean power equals the mean of no_eff, each within STAT_SIGMAS standard errors."""
    from sionna_b200.phy.mimo import zf_equalizer, mf_equalizer
    g = torch.Generator(device=cuda_device).manual_seed(int(no * 100) + 7 * colored)
    n, m, k = STAT_BATCH, 8, 4
    pts = torch.from_numpy(MAP.qam(4).astype(np.complex64)).to(cuda_device)
    x = pts[torch.randint(0, 16, (n, k), device=cuda_device, generator=g)]

    def cn(*shape):
        return torch.complex(torch.randn(*shape, device=cuda_device, generator=g),
                             torch.randn(*shape, device=cuda_device, generator=g)) / np.sqrt(2)
    h = cn(n, m, k)
    s = no * torch.eye(m, dtype=torch.complex64, device=cuda_device)
    if colored:
        idx = torch.arange(m, device=cuda_device)
        s = s + (0.95 ** (idx[:, None] - idx[None, :]).abs().double()).to(torch.complex64)
    w = (torch.linalg.cholesky(s.to(torch.complex128)) @ cn(n, m, 1).to(torch.complex128))[..., 0]
    y = (h @ x[..., None])[..., 0] + w.to(torch.complex64)
    x_hat, no_eff = (zf_equalizer if eq == "zf" else mf_equalizer)(y, h, s.expand(n, m, m))
    err = (x - x_hat).to(torch.complex128).flatten()
    se_mean = float(torch.sqrt(torch.mean(err.abs() ** 2) / err.numel()))
    assert abs(complex(err.mean())) <= STAT_SIGMAS * se_mean
    d = (err.abs() ** 2 - no_eff.double().flatten())
    assert abs(float(d.mean())) <= STAT_SIGMAS * float(d.std()) / np.sqrt(d.numel())
