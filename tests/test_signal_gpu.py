"""The signal module on the GPU (csrc/signal.cu, phy/signal/): convolve and the filters against np.convolve / the
float64 oracle (oracle/signal.py) -- the reference's unit tests (test/unit/signal/test_signal_utils.py, test_filter.py,
test_window.py) restated, and the fp32 envelope over the kernel's tile and tap-chunk boundaries -- windows, up- and
downsampling, the empirical PSD / ACLR, and the Pulse_Shaping_Basics tutorial's chain and printed numbers."""
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import signal as O
from oracle.parity import envelope

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "signal_golden.npz"))
DTYPES = [torch.float32, torch.float64, torch.complex64, torch.complex128]


@pytest.fixture(autouse=True)
def _restore_precision_warnings():
    """PrecisionWarning is issued once per name and process (phy/block.py keeps the record); the double-precision
    cases here must not use up the warnings that other test files expect, so the record is restored after each test."""
    from sionna_b200.phy import block
    saved = set(block._warned_double)
    yield
    block._warned_double.clear()
    block._warned_double.update(saved)


def _rand(rng, shape, cplx, dtype=None):
    v = rng.normal(size=shape) + (1j * rng.normal(size=shape) if cplx else 0)
    return v if dtype is None else v.astype(dtype)


def _np(t):
    return t.cpu().numpy()


# ---- convolve: dtype rules, shapes, double precision ------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["single", "double"])
@pytest.mark.parametrize("padding", ["full", "same", "valid"])
def test_convolve_dtypes(cuda_device, padding, precision):
    from sionna_b200.phy.signal import convolve
    rng = np.random.default_rng(1)
    for xd in DTYPES:
        for hd in DTYPES:
            x = torch.from_numpy(_rand(rng, (3, 40), xd.is_complex)).to(cuda_device, xd)
            h = torch.from_numpy(_rand(rng, 8, hd.is_complex)).to(cuda_device, hd)
            y = convolve(x, h, padding.upper() if padding == "same" else padding, precision=precision)
            cplx = xd.is_complex or hd.is_complex
            want = {("single", False): torch.float32, ("single", True): torch.complex64,
                    ("double", False): torch.float64, ("double", True): torch.complex128}[(precision, cplx)]
            assert y.dtype == want
            assert y.shape == (3, {"full": 47, "same": 40, "valid": 33}[padding])
            ref = O.convolve(_np(x).astype(np.complex128 if xd.is_complex else np.float64), _np(h), padding)
            np.testing.assert_allclose(_np(y), ref, rtol=0, atol=1e-4 if precision == "single" else 1e-10)


def test_convolve_shapes_and_axes(cuda_device):
    from sionna_b200.phy.signal import convolve
    rng = np.random.default_rng(2)
    x = torch.from_numpy(_rand(rng, (2, 3, 4, 50), True)).to(cuda_device, torch.complex64)
    h = torch.from_numpy(_rand(rng, 7, False)).to(cuda_device, torch.float32)
    for padding, m in (("full", 56), ("same", 50), ("valid", 44)):
        assert convolve(x, h, padding).shape == (2, 3, 4, m)
    y = convolve(x.movedim(-1, 1), h, "full", axis=1)
    assert y.shape == (2, 56, 3, 4)
    np.testing.assert_array_equal(_np(y.movedim(1, -1)), _np(convolve(x, h, "full")))


def test_convolve_errors(cuda_device):
    from sionna_b200.phy.signal import convolve
    x = torch.ones(2, 10, device=cuda_device)
    h = torch.ones(3, device=cuda_device)
    with pytest.raises(AssertionError):
        convolve(x, h, "circular")
    with pytest.raises(ValueError):
        convolve(x, torch.ones(11, device=cuda_device), "valid")
    with pytest.raises(TypeError):
        convolve(torch.ones(2, 10, dtype=torch.int32), h)
    with pytest.raises(TypeError):
        convolve(x, torch.ones(3, dtype=torch.int64))
    with pytest.raises(NotImplementedError):
        convolve(x, torch.ones(3, device=cuda_device, requires_grad=True))


@pytest.mark.parametrize("k", [1, 2, 5, 8, 100])
@pytest.mark.parametrize("padding", ["full", "same", "valid"])
def test_convolve_double_equals_numpy(cuda_device, k, padding):
    from sionna_b200.phy.signal import convolve
    rng = np.random.default_rng(k)
    x = _rand(rng, (4, 200), True)
    h = _rand(rng, k, True)
    y = _np(convolve(torch.from_numpy(x), torch.from_numpy(h), padding, precision="double"))
    ref = np.stack([np.convolve(r, h, padding) for r in x])
    assert y.shape == ref.shape
    assert np.abs(y - ref).max() < 1e-10


@pytest.mark.parametrize("span", [7, 8])
@pytest.mark.parametrize("sps", [1, 3, 4])
@pytest.mark.parametrize("window", [None, "hann"])
@pytest.mark.parametrize("conjugate", [False, True])
def test_filter_double_equals_numpy(cuda_device, span, sps, window, conjugate):
    from sionna_b200.phy.signal import CustomFilter, RootRaisedCosineFilter
    rng = np.random.default_rng(span * 10 + sps)
    x = _rand(rng, (3, 100), True)
    length = 2 * (span * sps // 2) + 1
    coef = _rand(rng, length, True)
    w = None if window is None else GOLDEN[f"hann_{length}"]
    for filt in (CustomFilter(sps, coef, window=window, precision="double"),
                 RootRaisedCosineFilter(span, sps, 0.3, window=window, precision="double")):
        taps = O.prepare_taps(_np(filt.coefficients), w, conjugate=conjugate)
        for padding in ("full", "same", "valid"):
            y = _np(filt(torch.from_numpy(x), padding=padding, conjugate=conjugate))
            if padding == "valid" and length > x.shape[-1]:
                continue
            ref = np.stack([np.convolve(r, taps, padding) for r in x])
            assert np.abs(y - ref).max() < 1e-10, (padding, type(filt).__name__)


def test_filter_normalization_and_conjugation(cuda_device):
    from sionna_b200.phy.signal import CustomFilter, RaisedCosineFilter, SincFilter, RootRaisedCosineFilter
    for filt in (RaisedCosineFilter(8, 4, 0.3), SincFilter(8, 4), RootRaisedCosineFilter(8, 4, 0.3, window="blackman")):
        h = filt(torch.ones(1, device=cuda_device), padding="full")       # a length-1 input through a 33-tap filter
        assert h.shape == (33,)
        assert abs(float((h.abs() ** 2).sum()) - 1) < 1e-5
    rng = np.random.default_rng(3)
    coef = _rand(rng, 9, True)
    filt = CustomFilter(2, coef, normalize=False)
    x = torch.from_numpy(_rand(rng, (2, 30), True)).to(cuda_device, torch.complex64)
    from sionna_b200.phy.signal import convolve
    ref = convolve(x, torch.from_numpy(np.conj(coef)).to(cuda_device))
    np.testing.assert_allclose(_np(filt(x, conjugate=True)), _np(ref), rtol=0, atol=1e-6)
    assert RaisedCosineFilter(8, 4, 0.3, precision="double").coefficients.dtype == torch.float64
    assert filt.length == 9 and filt.sampling_times.dtype == np.float32


def test_filter_properties_and_errors(cuda_device):
    from sionna_b200.phy.signal import RootRaisedCosineFilter, CustomFilter, HannWindow, CustomWindow
    f = RootRaisedCosineFilter(32, 4, 0.22)
    assert (f.length, f.span_in_symbols, f.samples_per_symbol, f.beta, f.normalize) == (129, 32, 4, 0.22, True)
    np.testing.assert_array_equal(f.sampling_times, (np.arange(-64, 65, dtype=np.float32) / np.float32(4)))
    with pytest.raises(AssertionError):
        f.window = "kaiser"
    with pytest.raises(AssertionError):
        f.window = HannWindow(precision="double")
    with pytest.raises(ValueError):
        f.window = CustomWindow(np.ones(5, np.float32))
    with pytest.raises(AssertionError):
        RootRaisedCosineFilter(8, 4, 1.5)
    with pytest.raises(AssertionError):
        CustomFilter(2, np.ones(8, np.float32))
    with pytest.raises(NotImplementedError):
        f.show()
    with pytest.raises(NotImplementedError):
        HannWindow().show(4)
    f.coefficients = torch.ones(129, device=cuda_device, requires_grad=True)
    with pytest.raises(NotImplementedError):
        f(torch.ones(4, 200, device=cuda_device))
    f.window = "hamming"
    assert f.window.length == 129


def test_filter_state_follows_coefficients(cuda_device):
    from sionna_b200.phy.signal import CustomFilter
    rng = np.random.default_rng(4)
    x = torch.from_numpy(_rand(rng, (2, 64), False)).to(cuda_device, torch.float32)
    filt = CustomFilter(2, _rand(rng, 9, False).astype(np.float32), normalize=False)
    y0 = _np(filt(x))
    new = torch.from_numpy(_rand(rng, 9, False)).to(cuda_device, torch.float32)
    filt.coefficients = new
    y1 = _np(filt(x))
    np.testing.assert_allclose(y1, O.convolve(_np(x), _np(new)), rtol=0, atol=1e-5)
    assert not np.allclose(y0, y1)
    filt.coefficients.mul_(2)                                  # in place: the next call sees it
    np.testing.assert_allclose(_np(filt(x)), 2 * y1, rtol=1e-6, atol=1e-6)


def test_non_floating_inputs_are_refused(cuda_device):
    """Integer and bool inputs never reach the kernels: they would be read and written with another element size."""
    from sionna_b200.phy.signal import (convolve, HannWindow, CustomWindow, RootRaisedCosineFilter, CustomFilter,
                                        Upsampling, Downsampling)
    filt = RootRaisedCosineFilter(8, 4, 0.22)
    win = HannWindow()
    for dtype in (torch.int32, torch.bool, torch.int64, torch.uint8):
        x = torch.ones(4, 33, dtype=dtype, device=cuda_device)
        with pytest.raises(TypeError):
            win(x)
        with pytest.raises(TypeError):
            filt(x)
        with pytest.raises(TypeError):
            filt(x, padding="same")
        with pytest.raises(TypeError):
            convolve(x, torch.ones(3, device=cuda_device))
    for precision in ("single", "double"):
        with pytest.raises(TypeError):
            HannWindow(precision=precision)(torch.ones(2, 16, dtype=torch.int32, device=cuda_device))
    f = CustomFilter(2, np.ones(9, np.float32))
    with pytest.raises(TypeError):
        f.window = CustomWindow(np.ones(9, np.complex64))             # kept complex by the precision cast
    f.window = CustomWindow(np.ones(9, np.float32))
    f.window.coefficients = np.ones(9, np.complex64)
    with pytest.raises(TypeError):
        f(torch.ones(2, 20, device=cuda_device))
    for block in (Upsampling(2), Downsampling(2)):
        with pytest.raises(NotImplementedError):
            block(torch.ones(2, 10, dtype=torch.bool, device=cuda_device))
        with pytest.raises(NotImplementedError):
            block(torch.ones(2, 10, dtype=torch.int16, device=cuda_device))


# ---- fp32 envelope over the kernel's boundaries -----------------------------------------------------------------------
# Tiles hold 9 * threads-per-row outputs (2304 for long rows); with complex64 x a chunk holds up to 2808 taps for long
# rows and 27 when 64 short rows share a CTA; rows of <= 9 * tpr outputs are packed tpr = 4 ... 128 threads per row.
CASES = [  # rows, n, k, padding, x complex, h complex
    (3, 2304, 129, "same", True, False), (3, 2305, 129, "same", True, True), (2, 2303, 128, "same", False, True),
    (2, 4609, 9, "full", True, False), (2, 2175, 129, "full", False, False), (2, 2176, 129, "full", True, True),
    (2, 3000, 2808, "full", True, False), (2, 3000, 2809, "same", True, False), (2, 3000, 7930, "same", False, False), (1, 5000, 4097, "full", True, True),
    (1, 100, 4097, "full", True, False), (3, 50, 4097, "same", False, True), (5, 10, 33, "full", True, False),
    (5, 10, 33, "same", True, True), (4, 64, 64, "valid", True, False), (4, 65, 64, "same", True, False),
    (1, 1, 1, "full", False, False), (7, 1, 33, "full", True, True), (700, 20, 129, "full", True, False),
    (700, 20, 27, "same", True, False), (700, 20, 28, "same", True, True), (300, 36, 9, "full", False, False),
    (300, 37, 9, "same", True, False), (70000, 20, 9, "full", True, False), (0, 30, 5, "full", True, False),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(map(str, c)))
def test_convolve_fp32_envelope(cuda_device, case):
    from sionna_b200.phy.signal import convolve
    rows, n, k, padding, xc, hc = case
    rng = np.random.default_rng(rows * 7 + n * 3 + k)
    x = _rand(rng, (rows, n), xc, np.complex64 if xc else np.float32)
    h = _rand(rng, k, hc, np.complex64 if hc else np.float32)
    y = _np(convolve(torch.from_numpy(x).to(cuda_device), torch.from_numpy(h).to(cuda_device), padding))
    ref = O.convolve(x, h, padding)
    assert y.shape == ref.shape
    if rows == 0:
        return
    f32 = O.convolve(x, h, padding, single=True)
    assert not envelope(f"convolve {case}", y, f32, ref, (2, 4), floor=(1e-8, 1e-7))


def test_convolve_strided_input_and_middle_axis(cuda_device):
    from sionna_b200.phy.signal import convolve
    rng = np.random.default_rng(5)
    x = _rand(rng, (6, 300, 4), True, np.complex64)
    h = _rand(rng, 31, False, np.float32)
    xt = torch.from_numpy(x).to(cuda_device)[::2]                       # non-contiguous
    y = _np(convolve(xt, torch.from_numpy(h).to(cuda_device), "same", axis=1))
    xs = np.moveaxis(x[::2], 1, -1)
    ref, f32 = O.convolve(xs, h, "same"), O.convolve(xs, h, "same", single=True)
    assert not envelope("convolve axis 1", np.moveaxis(y, 1, -1), f32, ref, (2, 4))


def test_filter_fp32_envelope_window_conjugate(cuda_device):
    from sionna_b200.phy.signal import CustomFilter, BlackmanWindow
    rng = np.random.default_rng(6)
    coef = _rand(rng, 129, True, np.complex64)
    filt = CustomFilter(4, coef, window=BlackmanWindow(normalize=True))
    x = _rand(rng, (40, 1000), True, np.complex64)
    y = _np(filt(torch.from_numpy(x).to(cuda_device), padding="same", conjugate=True))
    w = GOLDEN["blackman_129"]
    ref = O.convolve(x, O.prepare_taps(coef, w, window_normalize=True, conjugate=True), "same")
    f32 = O.convolve(x, O.prepare_taps(coef, w.astype(np.float32), window_normalize=True, conjugate=True, single=True),
                     "same", single=True)
    assert not envelope("filter window conj", y, f32, ref, (2, 4), floor=(1e-8, 1e-7))


# ---- windows ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["Hann", "Hamming", "Blackman"])
@pytest.mark.parametrize("n", [16, 33, 129])
def test_window_coefficients_and_call(cuda_device, name, n):
    import sionna_b200.phy.signal as S
    rng = np.random.default_rng(n)
    for precision, normalize in (("single", False), ("double", True)):
        win = getattr(S, f"{name}Window")(normalize=normalize, precision=precision)
        for xc in (False, True):
            x = _rand(rng, (3, n), xc)
            y = win(torch.from_numpy(x))
            want = {(False, "single"): torch.float32, (True, "single"): torch.complex64,
                    (False, "double"): torch.float64, (True, "double"): torch.complex128}[(xc, precision)]
            assert y.dtype == want and y.shape == (3, n)
            w = GOLDEN[f"{name.lower()}_{n}"]
            np.testing.assert_array_equal(_np(win.coefficients), w.astype(np.float32 if precision == "single" else
                                                                         np.float64))
            if normalize:
                w = w / np.sqrt(np.mean(w ** 2))
            np.testing.assert_allclose(_np(y), w * x, rtol=0, atol=1e-6 if precision == "single" else 1e-13)
        with pytest.raises(ValueError):
            win(torch.ones(2, n + 1))


# ---- up- and downsampling ---------------------------------------------------------------------------------------------
def _up_ref(x, sps, axis):
    x = x.movedim(axis, -1)
    y = torch.zeros(x.shape[:-1] + (x.shape[-1] * sps,), dtype=x.dtype, device=x.device)
    y[..., ::sps] = x
    return y.movedim(-1, axis)


@pytest.mark.parametrize("dtype", DTYPES + [torch.int32, torch.int64])
@pytest.mark.parametrize("axis", [-1, 1, -2])
def test_up_and_downsampling_bit_exact(cuda_device, dtype, axis):
    from sionna_b200.phy.signal import Upsampling, Downsampling
    prec = "double" if dtype in (torch.float64, torch.complex128) else "single"
    rng = np.random.default_rng(7)
    if dtype.is_floating_point or dtype.is_complex:
        x = torch.from_numpy(_rand(rng, (2, 11, 5, 13), dtype.is_complex)).to(cuda_device, dtype)
    else:
        x = torch.from_numpy(rng.integers(-2 ** 31, 2 ** 31, (2, 11, 5, 13))).to(cuda_device, dtype)
    for sps in (1, 3, 4):
        y = Upsampling(sps, axis=axis, precision=prec)(x)
        assert y.dtype == dtype
        assert torch.equal(y, _up_ref(x, sps, axis))
        n = x.shape[axis]
        for offset in (0, 2, -3, -20, n - 1, n, n + 5):
            for num in (None, 2, 0):
                z = Downsampling(sps, offset=offset, num_symbols=num, axis=axis, precision=prec)(x)
                ref = x.movedim(axis, -1)[..., offset::sps]
                if num is not None:
                    ref = ref[..., :num]
                ref = ref.movedim(-1, axis)
                assert z.dtype == dtype and z.shape == ref.shape and torch.equal(z, ref), (sps, offset, num)
                assert z.shape[axis] == min(len(range(n)[offset::sps]), n if num is None else num)


# ---- PSD and ACLR -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(128, 4128 // 2), (3000, 64), (1, 1), (7, 8192), (2, 3, 1000)])
def test_empirical_psd(cuda_device, shape):
    from sionna_b200.phy.signal import empirical_psd
    rng = np.random.default_rng(8)
    x = _rand(rng, shape, True, np.complex64)
    freqs, psd = empirical_psd(torch.from_numpy(x).to(cuda_device), show=False, oversampling=4.0)
    f_ref, p_ref = O.psd(x, oversampling=4.0)
    _, p32 = O.psd(x, oversampling=4.0, single=True)
    assert freqs.dtype == torch.float32 and psd.dtype == torch.float32
    np.testing.assert_array_equal(_np(freqs), f_ref)
    # the PSD carries the FFT kernel's error, whose own envelope against complex64 pocketfft reaches 2.94x (rms) at
    # some sizes (tests/test_fft_envelope_gpu.py); averaging few rows does not shrink it
    assert not envelope(f"psd {shape}", _np(psd)[None], p32[None], p_ref[None], (3, 4), floor=(1e-8, 1e-7))


def test_power_mean_is_deterministic(cuda_device):
    from sionna_b200.phy.signal import utils as U
    for shape in ((10 ** 6, 64), (128, 4128)):
        x = torch.randn(shape, dtype=torch.complex64, device=cuda_device)
        a, b = U._power_mean(x), U._power_mean(x)
        assert torch.equal(a, b)
        ref = (x.abs() ** 2).double().mean(0).float()
        assert torch.allclose(a, ref, rtol=1e-4)


def test_empirical_aclr_and_psd_errors(cuda_device):
    from sionna_b200.phy.signal import empirical_aclr, empirical_psd
    rng = np.random.default_rng(9)
    x = _rand(rng, (64, 256), True, np.complex64)
    a = empirical_aclr(torch.from_numpy(x).to(cuda_device), oversampling=2.0, f_min=-0.3, f_max=0.4)
    f, p = O.psd(x, oversampling=2.0)
    assert isinstance(a, float) and abs(a / O.aclr(f, p, -0.3, 0.4) - 1) < 1e-4
    with pytest.raises(ValueError):
        empirical_psd(torch.ones(2, 8193, dtype=torch.complex64), show=False)


# ---- the Pulse_Shaping_Basics tutorial --------------------------------------------------------------------------------
@pytest.mark.parametrize("span, sps, beta, window, expect_db", [(32, 4, 0.22, None, -13.8057),
                                                                (32, 4, 0.1, None, -17.3421),
                                                                (8, 8, 0.22, None, -13.9830),
                                                                (8, 8, 0.22, "blackman", -12.6241)])
def test_tutorial_filter_aclr(cuda_device, span, sps, beta, window, expect_db):
    from sionna_b200.phy.signal import RootRaisedCosineFilter
    f = RootRaisedCosineFilter(span, sps, beta, window=window)
    aclr = f.aclr
    assert isinstance(aclr, float)
    assert abs(10 * np.log10(aclr) - expect_db) < 0.01


def test_tutorial_chain(cuda_device):
    from sionna_b200.phy import config
    from sionna_b200.phy.mapping import BinarySource, Mapper
    from sionna_b200.phy.signal import Upsampling, Downsampling, RootRaisedCosineFilter, empirical_aclr, empirical_psd
    config.seed = 42
    batch, num_symbols, sps = 128, 1000, 4
    x = Mapper("qam", 4)(BinarySource()([batch, num_symbols * 4]))
    rrcf = RootRaisedCosineFilter(32, sps, 0.22)
    assert rrcf.length == 129
    x_rrcf = rrcf(Upsampling(sps)(x))
    assert x_rrcf.shape == (batch, num_symbols * sps + 128)
    x_hat = Downsampling(sps, rrcf.length - 1, num_symbols)(rrcf(x_rrcf))
    assert x_hat.shape == x.shape
    mse_db = 10 * np.log10(float(((x - x_hat).abs() ** 2).mean()))
    assert abs(mse_db - (-53.49)) < 0.5, mse_db
    aclr_db = 10 * np.log10(empirical_aclr(x_rrcf, oversampling=sps))
    assert abs(aclr_db - (-13.78)) < 0.1, aclr_db
    with warnings.catch_warnings(record=True) as w:                 # show=True: values, and one warning, ever
        warnings.simplefilter("always")
        from sionna_b200.phy.signal import utils as U
        U._warned_show = False
        freqs, psd = empirical_psd(x_rrcf, oversampling=sps)
        empirical_psd(x_rrcf, oversampling=sps)
    assert sum("no plot" in str(v.message) for v in w) == 1
    assert freqs.shape == psd.shape == (num_symbols * sps + 128,)


def test_precision_warnings(cuda_device):
    from sionna_b200.phy import block
    from sionna_b200.phy.block import PrecisionWarning
    from sionna_b200.phy.signal import convolve, RootRaisedCosineFilter, empirical_psd, Upsampling, HannWindow
    block._warned_double.discard("empirical_psd")
    x = torch.randn(4, 100, dtype=torch.complex128, device=cuda_device)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        assert convolve(x, torch.ones(5, dtype=torch.float64), precision="double").dtype == torch.complex128
        f = RootRaisedCosineFilter(8, 4, 0.22, window="hann", precision="double")
        assert f(x).dtype == torch.complex128
        f.aclr
        Upsampling(2, precision="double")(x)
        HannWindow(precision="double")(x)
    assert not any(issubclass(v.category, PrecisionWarning) for v in w)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        freqs, psd = empirical_psd(x, show=False, precision="double")
        empirical_psd(x, show=False, precision="double")
    assert freqs.dtype == psd.dtype == torch.float64
    assert sum(issubclass(v.category, PrecisionWarning) for v in w) == 1
