"""The signal oracle (oracle/signal.py) against NumPy and the reference's own formulas (tests/golden/
signal_golden.npz, made by tests/golden/make_signal_golden.py), and the pulse shapes' defining properties. CPU only."""
import numpy as np
import pytest

from oracle import signal as O

GOLDEN = np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "signal_golden.npz"))


@pytest.mark.parametrize("k", [1, 2, 5, 8, 33, 100])
@pytest.mark.parametrize("n", [1, 7, 64, 100])
@pytest.mark.parametrize("padding", ["full", "same", "valid"])
def test_convolve_equals_numpy(k, n, padding):
    rng = np.random.default_rng(k * 1000 + n)
    x = rng.normal(size=(3, n)) + 1j * rng.normal(size=(3, n))
    h = rng.normal(size=k)
    if padding == "valid" and k > n:
        return
    got = O.convolve(x, h, padding)
    if padding == "same" and k > n:                 # NumPy returns max(n, k) samples; this form keeps n
        full = np.stack([np.convolve(r, h, "full") for r in x])
        ref = full[:, (k - 1) // 2:(k - 1) // 2 + n]
    else:
        ref = np.stack([np.convolve(r, h, padding) for r in x])
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12)


def test_convolve_single_is_single():
    x = np.ones((2, 10), np.complex64)
    assert O.convolve(x, np.ones(3), single=True).dtype == np.complex64
    assert O.convolve(x.real, np.ones(3), single=True).dtype == np.float32
    assert O.convolve(x.real, np.ones(3)).dtype == np.float64


def _ulp_of_peak(h):
    return np.spacing(np.float32(np.abs(h).max()))


def test_pulses_match_reference_golden():
    """The float64 formulas against the reference's float32 evaluation: within 2 float32 ulps of the peak tap. (The
    reference evaluates in float32; near the pulses' zeros its values carry that absolute error, so ulps of each
    element are not a meaningful measure there; the largest gap measured is 1.8 ulps of the peak.)"""
    for key in GOLDEN.files:
        parts = key.split("_")
        if parts[0] not in ("rc", "rrc", "sinc"):
            continue
        sps, span = int(parts[-2][1:]), int(parts[-1][1:])
        t = O.sampling_times(span, sps)
        if parts[0] == "sinc":
            h = O.sinc(t)
        else:
            beta = float(parts[1][1:])
            h = (O.raised_cosine if parts[0] == "rc" else O.root_raised_cosine)(t, beta)
        g = GOLDEN[key].astype(np.float64)
        assert h.shape == g.shape, key
        assert np.abs(h - g).max() <= 2 * _ulp_of_peak(h), key


def test_package_pulses_equal_reference_golden():
    """The package's float32 host formulas reproduce the reference's coefficients bit for bit."""
    from sionna_b200.phy.signal import filter as F
    for key in GOLDEN.files:
        parts = key.split("_")
        if parts[0] not in ("rc", "rrc", "sinc"):
            continue
        sps, span = int(parts[-2][1:]), int(parts[-1][1:])
        t = O.sampling_times(span, sps).astype(np.float32)
        if parts[0] == "sinc":
            h = np.sinc(t)
        else:
            beta = float(parts[1][1:])
            h = (F.raised_cosine if parts[0] == "rc" else F.root_raised_cosine)(t, 1.0, beta)
        assert np.array_equal(np.asarray(h, np.float32), GOLDEN[key]), key


def test_windows_match_reference_golden():
    for key in GOLDEN.files:
        kind, n = key.rsplit("_", 1)
        if kind in ("hann", "hamming", "blackman"):
            np.testing.assert_allclose(O.window(kind, int(n)), GOLDEN[key], rtol=0, atol=1e-15)


@pytest.mark.parametrize("beta", [0.0, 0.22, 0.5, 1.0])
@pytest.mark.parametrize("sps", [2, 4, 8])
def test_raised_cosine_zero_isi(beta, sps):
    t = O.sampling_times(16, sps)
    h = O.raised_cosine(t, beta)
    assert h[len(t) // 2] == 1.0
    integer = np.isclose(t, np.round(t), atol=1e-12) & (t != 0)
    assert np.abs(h[integer]).max() < 1e-15


@pytest.mark.parametrize("beta", [0.1, 0.22, 0.5, 1.0])
def test_rrc_cascade_is_rc(beta):
    """RRC * RRC sampled densely approximates RC: the cascade at sample spacing 1 / sps, scaled by 1 / sps."""
    sps, span = 16, 64
    t = O.sampling_times(span, sps)
    g = O.root_raised_cosine(t, beta)
    rc = np.convolve(g, g)[len(t) // 2:len(t) // 2 + len(t)] / sps
    ref = O.raised_cosine(t, beta)
    mid = np.abs(t) <= 8
    assert np.abs(rc[mid] - ref[mid]).max() < 2e-2 * (1 + (beta < 0.2))


def test_prepare_taps_order():
    h = np.array([1.0, 2.0, 3.0 + 1j])
    w = np.array([0.5, 1.0, 0.5])
    p = O.prepare_taps(h, w, window_normalize=True, normalize=True, conjugate=True)
    ww = w / np.sqrt(np.mean(w ** 2))
    ref = np.conj(h * ww / np.linalg.norm(h * ww))
    np.testing.assert_allclose(p, ref, rtol=1e-15)
    assert np.isclose(np.sum(np.abs(p) ** 2), 1.0)


def test_linspace_f32():
    f = O.linspace_f32(-2.0, 2.0, 1024)
    assert f.dtype == np.float32 and f[0] == -2 and f[-1] == 2
    assert O.linspace_f32(-0.5, 0.5, 1)[0] == np.float32(-0.5)


def test_psd_of_white_noise_and_tone():
    rng = np.random.default_rng(0)
    x = (rng.normal(size=(4000, 64)) + 1j * rng.normal(size=(4000, 64))) / np.sqrt(2)
    _, p = O.psd(x)
    assert abs(p.mean() - 1) < 0.01
    tone = np.exp(2j * np.pi * 5 * np.arange(64) / 64)[None]
    f, p = O.psd(tone)
    assert np.argmax(p) == 32 + 5 and np.isclose(p.max(), 64)


@pytest.mark.parametrize("span, sps, beta, win, expect_db", [(32, 4, 0.22, None, -13.8057), (32, 4, 0.1, None, -17.3421),
                                                             (8, 8, 0.22, None, -13.9830),
                                                             (8, 8, 0.22, "blackman", -12.6241)])
def test_filter_aclr_tutorial(span, sps, beta, win, expect_db):
    """The Pulse_Shaping_Basics tutorial's filter ACLRs, from the float64 oracle."""
    t = O.sampling_times(span, sps)
    w = None if win is None else O.window(win, len(t))
    h = O.prepare_taps(O.root_raised_cosine(t, beta), w)
    c = np.zeros(1024, np.complex128)
    c[:len(h)] = h
    f, p = O.psd(c.astype(np.complex64), oversampling=sps)
    assert abs(10 * np.log10(O.aclr(f, p)) - expect_db) < 0.01
