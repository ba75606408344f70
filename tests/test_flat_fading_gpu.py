"""Flat-fading MIMO channels on the GPU (sb_flat_fading, sb_chol_lower and the blocks on them):
  1. draws: h equals the Philox stream of oracle/rng.awgn within 5 ulp (the bound of test_rng_streams_gpu.py), and the
     randomness contract holds bit for bit (complex_normal, the models on a given h, AWGN, generate then apply);
  2. correlation (Kronecker, per column) and the Cholesky factors against the float64 oracle, within 2x (rms) / 4x (max)
     of the complex64 oracle's error; a non-positive-definite matrix yields NaN in its own outputs only;
  3. y = h x within the envelope of a complex64 matmul, h shared or per row, every form of `no`;
  4. FlatFadingChannel equals generate then apply bit for bit;
  5. the reference's statistical unit tests (covariances, noise and output variance, per-example matrices, setters);
  6. links: the reference's test_mimo_flat_fading model and its MMSE-PIC / LMMSE comparison;
  7. precision="double".
Measured ratios and BERs are printed (pytest -s)."""
import numpy as np
import pytest
import torch

from oracle import flat_fading as O
from oracle.parity import envelope

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -23
SEEDS = [(0xFEDC_BA98_7654_3210, (0xABCD << 32) | 0x1234), (0x7FFF_FFFF_FFFF_FFFF, (1 << 63) + 5)]
BAR = (2.0, 4.0)
FLOOR = (2.0 ** -23, 2.0 ** -22)


@pytest.fixture(autouse=True)
def _restore_precision_warnings():
    """PrecisionWarning is issued once per class and process (phy/block.py keeps the record). The double-precision
    cases here must not use up the warnings that other test files expect, so the record is restored after each test."""
    from sionna_b200.phy import block
    saved = set(block._warned_double)
    yield
    block._warned_double.clear()
    block._warned_double.update(saved)


def _bits(t):
    return torch.view_as_real(t.contiguous()).contiguous().view(torch.int32).cpu().numpy()


def _same(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype
    assert np.array_equal(_bits(a), _bits(b))


def _dev(a, dtype=torch.complex64):
    return torch.as_tensor(np.asarray(a)).to(device="cuda", dtype=dtype).contiguous()


def _ff(num, M, K, seed=0, off=0, h_in=None, h_stride=0, l_tx=None, tx_stride=0, l_rx=None, rx_stride=0,
        per_column=0, want_h=True, x=None, x_stride=0, no=None, no_inner=1, seed_n=0, off_n=0):
    from sionna_b200._lib import lib, check, ptr, current_stream
    h = torch.empty(num, M, K, dtype=torch.complex64, device="cuda") if want_h else None
    y = torch.empty(num, M, dtype=torch.complex64, device="cuda") if x is not None else None
    check(lib().sb_flat_fading(ptr(h_in), h_stride, seed, off, ptr(l_tx), tx_stride, ptr(l_rx), rx_stride, per_column,
                               ptr(h), ptr(x), x_stride, ptr(no), no_inner, seed_n, off_n, ptr(y), num, M, K,
                               current_stream()), "sb_flat_fading")
    torch.cuda.synchronize()
    return h, y


# ---- 1. draws and the randomness contract ----------------------------------------------------------------------------
@pytest.mark.parametrize("num,M,K", [(1, 1, 1), (1, 1, 3), (95_239, 7, 3)])
def test_draw_values(cuda_device, num, M, K):
    for seed, off in SEEDS[: 1 if num > 1000 else 2]:
        h, _ = _ff(num, M, K, seed, off)
        ref = O.draw(seed, off, num, M, K)
        err = np.abs(h.cpu().numpy().astype(np.complex128) - ref) / (ULP * np.maximum(np.abs(ref), 1e-30))
        print(f"draw {num}x{M}x{K}: worst {err.max():.2f} ulp")
        assert err.max() <= 5.0


def _models(M, K):
    from sionna_b200.phy.channel import KroneckerModel, PerColumnModel, exp_corr_mat, one_ring_corr_mat
    return {"none": None,
            "kronecker": KroneckerModel(exp_corr_mat(0.4, K), exp_corr_mat(0.7 + 0.1j, M)),
            "per_column": PerColumnModel(one_ring_corr_mat(np.linspace(-40, 40, K), M, 1.0, 10))}


@pytest.mark.parametrize("model", ["none", "kronecker", "per_column"])
def test_generate_equals_draw_then_model(cuda_device, model):
    from sionna_b200.phy import config
    from sionna_b200.phy.channel import GenerateFlatFadingChannel
    from sionna_b200.phy.utils import complex_normal
    B, M, K = 1001, 7, 3
    sc = _models(M, K)[model]
    config.seed = 5
    h1 = GenerateFlatFadingChannel(K, M, spatial_corr=sc)(B)
    config.seed = 5
    h2 = complex_normal([B, M, K])
    if sc is not None:
        h2 = sc(h2)
    _same(h1, h2)


@pytest.mark.parametrize("no_shape", ["scalar", "batch", "full"])
def test_apply_noise_equals_awgn(cuda_device, no_shape):
    from sionna_b200.phy import config
    from sionna_b200.phy.channel import ApplyFlatFadingChannel, AWGN
    from sionna_b200.phy.utils import complex_normal
    B, M, K = 333, 5, 3
    h, x = complex_normal([B, M, K]), complex_normal([B, K])
    no = {"scalar": 0.3, "batch": torch.rand(B, device="cuda") + 0.1,
          "full": torch.rand(B, M, device="cuda") + 0.1}[no_shape]
    config.seed = 9
    y1 = ApplyFlatFadingChannel()(x, h, no)
    config.seed = 9
    y2 = AWGN()(ApplyFlatFadingChannel()(x, h), no)
    _same(y1, y2)


@pytest.mark.parametrize("model", ["none", "kronecker", "per_column"])
@pytest.mark.parametrize("return_channel", [False, True])
@pytest.mark.parametrize("noise", [False, True])
def test_flat_fading_equals_generate_then_apply(cuda_device, model, return_channel, noise):
    from sionna_b200.phy import config
    from sionna_b200.phy.channel import FlatFadingChannel
    from sionna_b200.phy.utils import complex_normal
    B, M, K = 517, 16, 4
    chn = FlatFadingChannel(K, M, spatial_corr=_models(M, K)[model], return_channel=return_channel)
    x = complex_normal([B, K])
    no = 0.2 if noise else None
    config.seed = 3
    out = chn(x, no)
    off1 = config._philox_offset
    config.seed = 3
    h = chn.generate(B)
    y = chn.apply(x, h, no)
    assert config._philox_offset == off1
    if return_channel:
        _same(out[0], y)
        _same(out[1], h)
    else:
        _same(out, y)


# ---- 2. correlation and factors against the float64 oracle -----------------------------------------------------------
def _corr(kind, n, count, rng):
    """count n x n correlation matrices (complex64 values, condition number <= 1e6)"""
    if kind == "exp":
        a = rng.uniform(0.1, 0.95, count) * np.exp(1j * rng.uniform(-np.pi, np.pi, count))
        return O.exp_corr(a, n).astype(np.complex64)
    out = []
    while len(out) < count:
        r = O.one_ring(rng.uniform(-60, 60), n, rng.choice([0.5, 1.0, 2.0]), rng.uniform(5, 15))
        r = r.astype(np.complex64)
        if np.linalg.cond(r.astype(np.complex128)) <= 1e6:
            out.append(r)
        elif n > 8 and rng.uniform() < 0.2:                       # large one-ring arrays: regularise toward cond 1e6
            w = np.linalg.eigvalsh(r.astype(np.complex128))
            out.append((r + np.float32(max(w[-1] / 1e6 - w[0], 0)) * np.eye(n)).astype(np.complex64))
    return np.stack(out)


def _f64(r):
    return np.asarray(r).astype(np.complex128)


@pytest.mark.parametrize("n", [1, 2, 4, 7, 16, 64, 128])
@pytest.mark.parametrize("kind", ["exp", "one_ring"])
def test_chol_lower_envelope(cuda_device, n, kind):
    from sionna_b200.phy.channel.spatial_correlation import cholesky
    rng = np.random.default_rng(n)
    r = _corr(kind, n, 6, rng)
    got = cholesky(_dev(r)).cpu().numpy()
    ref = O.chol(_f64(r))
    f32 = O.chol(r, np.complex64)
    assert np.all(np.triu(got, 1) == 0)
    bad = envelope(f"chol {kind} n={n}", got, f32, ref, BAR, FLOOR, axis=(-2, -1))
    assert not bad, bad


def test_non_positive_definite_stays_local(cuda_device):
    from sionna_b200.phy.channel import KroneckerModel
    from sionna_b200.phy.channel.spatial_correlation import cholesky
    r = O.exp_corr([0.3, 0.5, 0.7], 8).astype(np.complex64)
    r[1, 5, 5] = -1.0                                            # pivot 5 of matrix 1 goes negative
    l = cholesky(_dev(r)).cpu().numpy()
    assert np.isfinite(l[[0, 2]]).all() and np.isnan(l[1]).any() and np.isfinite(l[1, :5]).all()
    h = _dev(O.draw(1, 2, 3, 8, 2))
    out = KroneckerModel(None, _dev(r))(h).cpu().numpy()
    assert np.isfinite(out[[0, 2]]).all() and np.isnan(out[1]).any()


# (M, K) pairs: both small, tall, wide, square, the largest
SHAPES = [(1, 1), (2, 4), (4, 2), (7, 7), (16, 4), (4, 16), (64, 8), (8, 64), (16, 128), (128, 16), (64, 64),
          (128, 128)]


def _check(what, got, h64, h32):
    bad = envelope(what, got.cpu().numpy(), h32, h64, BAR, FLOOR, axis=(-2, -1))
    assert not bad, bad


@pytest.mark.parametrize("M,K", SHAPES)
@pytest.mark.parametrize("kind", ["exp", "one_ring"])
def test_kronecker_envelope(cuda_device, M, K, kind):
    from sionna_b200.phy.channel import KroneckerModel
    rng = np.random.default_rng(M * 1000 + K)
    B = 3 if M * K >= 4096 else 24
    h0 = (O.draw(11, 12, B, M, K)).astype(np.complex64)
    for per_example in (False, True):
        r_tx = _corr(kind, K, B if per_example else 1, rng)
        r_rx = _corr(kind, M, B if per_example else 1, rng)
        if not per_example:
            r_tx, r_rx = r_tx[0], r_rx[0]
        for use_tx, use_rx in ((True, False), (False, True), (True, True)):
            tx, rx = (r_tx if use_tx else None), (r_rx if use_rx else None)
            got = KroneckerModel(None if tx is None else _dev(tx), None if rx is None else _dev(rx))(_dev(h0))
            l64 = [None if r is None else O.chol(_f64(r)) for r in (tx, rx)]
            l32 = [None if r is None else O.chol(r, np.complex64) for r in (tx, rx)]
            _check(f"kron {kind} {M}x{K} tx={use_tx} rx={use_rx} per_example={per_example}", got,
                   O.kronecker(_f64(h0), *l64), O.kronecker(h0, *l32, dtype=np.complex64))


@pytest.mark.parametrize("M,K", [(1, 1), (4, 2), (7, 7), (16, 4), (64, 8), (128, 16), (128, 128)])
def test_per_column_envelope(cuda_device, M, K):
    from sionna_b200.phy.channel import PerColumnModel
    rng = np.random.default_rng(M * 1000 + K + 7)
    B = 3 if M * K >= 4096 else 12
    h0 = O.draw(13, 14, B, M, K).astype(np.complex64)
    for lead in [(), (K,), (B, K)]:
        kind = "one_ring" if len(lead) else "exp"
        r = _corr(kind, M, int(np.prod(lead)) if lead else 1, rng).reshape(lead + (M, M))
        got = PerColumnModel(_dev(r))(_dev(h0))
        full = np.broadcast_to(r, (B, K, M, M))
        _check(f"per-column {M}x{K} r_rx {lead + (M, M)}", got, O.per_column(_f64(h0), O.chol(_f64(full))),
               O.per_column(h0, O.chol(full, np.complex64), np.complex64))


# ---- 3. apply --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,K", [(1, 1), (16, 4), (7, 33), (128, 128), (300, 2)])
@pytest.mark.parametrize("h_per_row", [False, True])
def test_apply_envelope(cuda_device, M, K, h_per_row):
    from sionna_b200.phy import config
    from sionna_b200.phy.channel import ApplyFlatFadingChannel
    B = 257
    h = O.draw(21, 22, B if h_per_row else 1, M, K).astype(np.complex64)
    if not h_per_row:
        h = h[0]
    x = O.draw(23, 24, B, 1, K)[:, 0].astype(np.complex64)
    off = config._philox_offset
    y = ApplyFlatFadingChannel()(_dev(x), _dev(h))
    assert config._philox_offset == off                         # no=None draws nothing
    bad = envelope(f"apply {M}x{K} per_row={h_per_row}", y.cpu().numpy(), O.apply(h, x, np.complex64),
                   O.apply(_f64(h), _f64(x)), BAR, FLOOR)
    assert not bad, bad


# ---- 5. statistics (the reference's unit tests) ----------------------------------------------------------------------
def _covariances(h):
    h = h.to(torch.complex128)
    return torch.einsum("bmk,bml->kl", h.conj(), h), torch.einsum("bmk,bnk->mn", h, h.conj())


def _kron_cov(make_h, M, K, iters, batch):
    r_tx_hat = torch.zeros(K, K, dtype=torch.complex128, device="cuda")
    r_rx_hat = torch.zeros(M, M, dtype=torch.complex128, device="cuda")
    for _ in range(iters):
        t, r = _covariances(make_h(batch))
        r_tx_hat += t / (iters * batch * M)
        r_rx_hat += r / (iters * batch * K)
    return r_tx_hat.cpu().numpy(), r_rx_hat.cpu().numpy()


@pytest.mark.parametrize("a_rx", [0.4, 0.99])
def test_kronecker_covariance(cuda_device, a_rx):
    from sionna_b200.phy.channel import GenerateFlatFadingChannel, KroneckerModel, exp_corr_mat
    M, K = 16, 4
    r_tx, r_rx = exp_corr_mat(0.4, K), exp_corr_mat(a_rx, M)
    gen = GenerateFlatFadingChannel(K, M, KroneckerModel(r_tx, r_rx))
    t, r = _kron_cov(gen, M, K, 10, 1_000_000)
    print(f"kronecker covariance a_rx={a_rx}: max err tx {np.abs(t - r_tx.cpu().numpy()).max():.2e} "
          f"rx {np.abs(r - r_rx.cpu().numpy()).max():.2e}")
    assert np.allclose(t, r_tx.cpu().numpy(), atol=1e-3) and np.allclose(r, r_rx.cpu().numpy(), atol=1e-3)


def test_tutorial_covariance(cuda_device):
    """The Simple MIMO tutorial's check: FlatFadingChannel with return_channel, Kronecker 0.4 / 0.9."""
    from sionna_b200.phy.channel import FlatFadingChannel, KroneckerModel, exp_corr_mat
    from sionna_b200.phy.mapping import QAMSource
    M, K = 16, 4
    r_tx, r_rx = exp_corr_mat(0.4, K), exp_corr_mat(0.9, M)
    chn = FlatFadingChannel(K, M, add_awgn=True, return_channel=True)
    chn.spatial_corr = KroneckerModel(r_tx, r_rx)
    x = QAMSource(4)([1_000_000, K])
    y, h = chn(x, 0.1)
    t, r = _covariances(h)
    t, r = t.cpu().numpy() / (1e6 * M), r.cpu().numpy() / (1e6 * K)
    assert np.allclose(t, r_tx.cpu().numpy(), atol=1e-2) and np.allclose(r, r_rx.cpu().numpy(), atol=1e-2)


def test_per_column_covariance(cuda_device):
    from sionna_b200.phy.channel import GenerateFlatFadingChannel, PerColumnModel, one_ring_corr_mat
    M, K = 16, 4
    r_rx = one_ring_corr_mat([-45, -15, 0, 30], M)
    gen = GenerateFlatFadingChannel(K, M, PerColumnModel(r_rx))
    acc = torch.zeros(K, M, M, dtype=torch.complex128, device="cuda")
    iters, batch = 40, 1_000_000                                 # 4e7 draws: the largest of 1024 entries' errors < 1e-3
    for _ in range(iters):
        h = gen(batch).to(torch.complex128)
        acc += torch.einsum("bmk,bnk->kmn", h, h.conj()) / (iters * batch)
    err = np.abs(acc.cpu().numpy() - r_rx.cpu().numpy()).max()
    print(f"per-column covariance: max err {err:.2e}")
    assert err < 1e-3


def test_noise_and_output_variance(cuda_device):
    from sionna_b200.phy.channel import ApplyFlatFadingChannel, FlatFadingChannel, GenerateFlatFadingChannel
    from sionna_b200.phy.channel import KroneckerModel, exp_corr_mat
    from sionna_b200.phy.mapping import QAMSource
    M, K, B = 16, 4, 1_000_000
    h = GenerateFlatFadingChannel(K, M, KroneckerModel(exp_corr_mat(0.4, K), exp_corr_mat(0.99, M)))(B)
    x = QAMSource(4)([B, K])
    app = ApplyFlatFadingChannel()
    n = (app(x, h, 0.1) - app(x, h)).to(torch.complex128)
    assert abs(float(torch.mean(torch.abs(n) ** 2)) - 0.1) < 5e-4
    y = FlatFadingChannel(K, M)(x, 0.2).to(torch.complex128)
    var = float(torch.mean(torch.abs(y - y.mean()) ** 2))
    print(f"noise variance ok; y variance {var:.4f} (K + no = {K + 0.2})")
    assert abs(var - (K + 0.2)) < 5e-3


def test_per_example_matrices(cuda_device):
    from sionna_b200.phy.channel import KroneckerModel, PerColumnModel, exp_corr_mat, one_ring_corr_mat
    from sionna_b200.phy.utils import complex_normal
    rng = np.random.default_rng(4)
    M, K, B = 16, 4, 24
    cases = [(exp_corr_mat(rng.uniform(size=B), K), exp_corr_mat(0.99, M)),
             (exp_corr_mat(0.4, K), exp_corr_mat(rng.uniform(size=B), M)),
             (exp_corr_mat(rng.uniform(size=B), K), exp_corr_mat(rng.uniform(size=B), M))]
    h = complex_normal([B, M, K])
    hn = _f64(h.cpu().numpy())
    for r_tx, r_rx in cases:
        out = KroneckerModel(r_tx, r_rx)(h).cpu().numpy()
        lt = np.broadcast_to(O.chol(_f64(r_tx.cpu().numpy())), (B, K, K))
        lr = np.broadcast_to(O.chol(_f64(r_rx.cpu().numpy())), (B, M, M))
        for i in range(B):
            assert np.allclose(out[i], lr[i] @ hn[i] @ np.conj(lt[i].T), atol=2e-5)
    # one channel, a different correlation per example: the output gains the examples' dimension
    r_tx, r_rx = cases[2]
    out = KroneckerModel(r_tx, r_rx)(h[0]).cpu().numpy()
    assert out.shape == (B, M, K)
    for i in range(B):
        ref = O.chol(_f64(r_rx[i].cpu().numpy())) @ hn[0] @ np.conj(O.chol(_f64(r_tx[i].cpu().numpy())).T)
        assert np.allclose(out[i], ref, atol=2e-5)
    r = one_ring_corr_mat(rng.uniform(size=(B, K)), M)           # the reference's angles: condition number ~500
    out = PerColumnModel(r)(h).cpu().numpy()
    for i in range(B):
        for k in range(K):
            assert np.allclose(out[i, :, k], O.chol(_f64(r[i, k].cpu().numpy())) @ hn[i, :, k], atol=1e-4)


def test_property_setters(cuda_device):
    from sionna_b200.phy.channel import FlatFadingChannel, KroneckerModel, PerColumnModel, exp_corr_mat
    from sionna_b200.phy.utils import complex_normal
    M, K = 16, 4
    h = complex_normal([8, M, K])
    kron = KroneckerModel(None, None)
    _same(kron(h), h)
    r_tx = exp_corr_mat(0.4, K)
    kron.r_tx = r_tx
    assert kron.r_tx is r_tx and kron.r_rx is None
    a = kron(h)
    kron.r_rx = exp_corr_mat(0.9, M)
    b = kron(h)
    assert not torch.equal(a, b)
    r_tx.copy_(exp_corr_mat(0.8, K))                             # in place: the next call sees it
    c = kron(h)
    _same(c, KroneckerModel(exp_corr_mat(0.8, K), exp_corr_mat(0.9, M))(h))
    pc = PerColumnModel(exp_corr_mat(0.3, M))
    d = pc(h)
    pc.r_rx = exp_corr_mat(0.6, M)
    assert not torch.equal(d, pc(h))
    chn = FlatFadingChannel(K, M, return_channel=True)
    assert chn.spatial_corr is None and chn.generate.spatial_corr is None
    chn.spatial_corr = kron
    assert chn.spatial_corr is kron and chn.generate.spatial_corr is kron
    x = complex_normal([8, K])
    from sionna_b200.phy import config
    config.seed = 1
    _, h1 = chn(x)
    config.seed = 1
    _same(h1, kron(complex_normal([8, M, K])))


# ---- 6. links --------------------------------------------------------------------------------------------------------
class _MimoModel:
    """The reference's test_mimo_flat_fading.py model: 4 -> 16, 16-QAM, LDPC 512 / 1024, lmmse_equalizer."""

    def __init__(self, spatial_corr=None):
        from sionna_b200.phy.channel import FlatFadingChannel
        from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
        from sionna_b200.phy.mapping import Mapper, Demapper, BinarySource
        self.n, self.k, self.m, self.K, self.M = 1024, 512, 4, 4, 16
        self.source = BinarySource()
        self.encoder = LDPC5GEncoder(self.k, self.n)
        self.mapper = Mapper("qam", self.m)
        self.demapper = Demapper("app", "qam", self.m)
        self.decoder = LDPC5GDecoder(self.encoder, hard_out=True)
        self.channel = FlatFadingChannel(self.K, self.M, spatial_corr=spatial_corr, add_awgn=True,
                                         return_channel=True)

    def __call__(self, batch_size, ebno_db):
        from sionna_b200.phy.mimo import lmmse_equalizer
        from sionna_b200.phy.utils import ebnodb2no
        b = self.source([batch_size, self.K, self.k])
        x = self.mapper(self.encoder(b))
        shape = x.shape
        x = x.reshape(-1, self.K)
        no = float(ebnodb2no(ebno_db, self.m, self.k / self.n)) * np.sqrt(self.M)
        y, h = self.channel(x, no)
        s = (no * torch.eye(self.M, device=y.device)).to(torch.complex64)
        x_hat, no_eff = lmmse_equalizer(y, h, s)
        llr = self.demapper(x_hat.reshape(shape), no_eff.reshape(shape))
        return b, self.decoder(llr)


def test_mimo_flat_fading_link(cuda_device):
    from sionna_b200.phy import config
    from sionna_b200.phy.channel import KroneckerModel, exp_corr_mat
    from sionna_b200.phy.utils import sim_ber
    ebno = [-6.0, -4.0, -2.0]
    out = {}
    for name, sc in (("uncorrelated", None), ("correlated", KroneckerModel(exp_corr_mat(0.4, 4), exp_corr_mat(0.7, 16)))):
        config.seed = 7
        ber, bler = sim_ber(_MimoModel(sc), ebno, batch_size=64, max_mc_iter=10, early_stop=False, verbose=False)
        ber, bler = np.asarray(torch.as_tensor(ber).cpu()), np.asarray(torch.as_tensor(bler).cpu())
        print(f"{name}: Eb/N0 {ebno} dB BER {ber} BLER {bler}")
        assert not np.isnan(ber).any() and not np.isnan(bler).any()
        assert np.all(np.diff(ber) <= 0) and ber[0] > ber[-1]
        out[name] = ber
    assert np.all(out["correlated"] >= out["uncorrelated"]) and out["correlated"][0] > out["uncorrelated"][0]


def _pic_vs_lmmse_ber(det, M, K, ebno_db, precision):
    from sionna_b200.phy.channel import FlatFadingChannel, PerColumnModel, exp_corr_mat
    from sionna_b200.phy.mapping import BinarySource, Mapper
    from sionna_b200.phy.mimo import LinearDetector, MMSEPICDetector
    from sionna_b200.phy.utils import ebnodb2no, sim_ber
    m = 4
    source, mapper = BinarySource(precision=precision), Mapper("qam", m, precision=precision)
    chn = FlatFadingChannel(K, M, spatial_corr=PerColumnModel(exp_corr_mat(0.8, M, precision=precision)),
                            return_channel=True, precision=precision)
    if det == "mmse-pic":
        detector = MMSEPICDetector("bit", demapping_method="maxlog", num_iter=1, constellation_type="qam",
                                   num_bits_per_symbol=m, precision=precision)
    else:
        detector = LinearDetector("lmmse", "bit", "maxlog", constellation_type="qam", num_bits_per_symbol=m,
                                  precision=precision)
    cdt = torch.complex128 if precision == "double" else torch.complex64
    rdt = torch.float64 if precision == "double" else torch.float32
    prior = torch.zeros(64, K, m, dtype=rdt, device="cuda")
    s = torch.eye(M, dtype=cdt, device="cuda")

    def run(batch_size, ebno_db):
        no = float(ebnodb2no(ebno_db, m, 1.0))
        bits = source([64, K, m])
        x = mapper(bits).squeeze(-1)
        y, h = chn(x, no)
        llr = detector(y, h, no * s, prior) if det == "mmse-pic" else detector(y, h, no * s)
        return bits, llr

    ber, _ = sim_ber(run, [ebno_db], 1, max_mc_iter=100, num_target_bit_errors=1000, soft_estimates=True,
                     early_stop=False, verbose=False, precision=precision)
    return float(np.asarray(torch.as_tensor(ber).cpu())[0])


@pytest.mark.parametrize("precision", ["single", "double"])
@pytest.mark.parametrize("M,K,ebno_db", [(1, 1, 20.0), (16, 1, -5.0), (16, 4, 0.0)])
def test_mmse_pic_matches_lmmse(cuda_device, M, K, ebno_db, precision):
    """The reference's test_mmse_pic_det.py comparison: one MMSE-PIC iteration with a zero prior is LMMSE detection,
    so on the same channels (same seed) the BERs agree within 5 %."""
    from sionna_b200.phy import config
    config.seed = 1234
    b_lmmse = _pic_vs_lmmse_ber("lmmse", M, K, ebno_db, precision)
    config.seed = 1234
    b_pic = _pic_vs_lmmse_ber("mmse-pic", M, K, ebno_db, precision)
    print(f"{M}x{K} {ebno_db} dB {precision}: BER lmmse {b_lmmse:.4e} mmse-pic {b_pic:.4e}")
    assert abs(b_lmmse - b_pic) / b_lmmse < 5e-2


# ---- 7. precision ----------------------------------------------------------------------------------------------------
def test_double_precision(cuda_device):
    import warnings
    from sionna_b200.phy import block
    from sionna_b200.phy.block import PrecisionWarning
    from sionna_b200.phy.channel import FlatFadingChannel, GenerateFlatFadingChannel, KroneckerModel, exp_corr_mat
    from sionna_b200.phy.utils import complex_normal
    for name in ("FlatFadingChannel", "GenerateFlatFadingChannel", "KroneckerModel"):
        block._warned_double.discard(name)
    kron = KroneckerModel(exp_corr_mat(0.4, 4, precision="double"), exp_corr_mat(0.7, 16, precision="double"))
    chn = FlatFadingChannel(4, 16, spatial_corr=kron, return_channel=True, precision="double")
    x = complex_normal([32, 4], precision="double")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        y, h = chn(x, 0.1)
        chn(x, 0.1)
    assert y.dtype == torch.complex128 and h.dtype == torch.complex128
    assert sum(issubclass(v.category, PrecisionWarning) for v in w) == 1
    assert GenerateFlatFadingChannel(4, 16, precision="double")(8).dtype == torch.complex128
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        assert kron(h).dtype == torch.complex128
    assert sum(issubclass(v.category, PrecisionWarning) for v in w) == 1
