"""The parity toolkit (oracle/parity.py) on the host: the envelope criterion and the shared input generators."""
import numpy as np
import pytest

from oracle import ldpc as O
from oracle.parity import (assert_mixed_convergence, bpsk_llr, cnormal, envelope, lifted_pcm, noise_covariance,
                           rel_err)

BAR = (2.0, 4.0)
UP = 1.0 + 2.0 ** -20


def _env(got, f32, bar=BAR):
    """envelope against a zero reference with unit scale: the errors are got and f32 themselves."""
    return envelope("t", np.asarray(got), np.asarray(f32), np.zeros(len(f32)), bar, scale=1.0)


def test_envelope_holds_at_the_bar_and_fails_just_above_it():
    f32 = np.ones(16)                                      # rms 1, max 1
    assert _env(2.0 * f32, f32) == ""                      # rms exactly at 2, max 2 <= 4
    assert _env(2.0 * UP * f32, f32) != ""                 # rms above, max still within
    spike = np.r_[4.0, np.zeros(15)]                       # rms 1 <= 2, max exactly at 4
    assert _env(spike, f32) == ""
    assert _env(UP * spike, f32) != ""                     # max above, rms still within


def test_envelope_requires_matching_finiteness():
    ref = np.array([1.0, np.inf, 2.0])
    ok = np.array([1.0, np.inf, 2.0])
    assert envelope("t", ok, ok, ref, BAR) == ""
    with pytest.raises(AssertionError, match="kernel finite"):
        envelope("t", np.array([1.0, 5.0, 2.0]), ok, ref, BAR)
    with pytest.raises(AssertionError, match="complex64 evaluation finite"):
        envelope("t", ok, np.array([np.nan, np.inf, 2.0]), ref, BAR)


def test_envelope_with_exact_complex64_does_not_divide_by_zero():
    ref = np.arange(1.0, 5.0)
    assert envelope("t", ref.copy(), ref.copy(), ref, BAR) == ""
    line = envelope("t", ref + 1e-3, ref.copy(), ref, BAR)
    assert "complex64 rms 0.00e+00" in line
    assert envelope("t", ref + 1e-3, ref.copy(), ref, BAR, floor=(1.0, 1.0)) == ""


def test_rel_err_forms_and_mask():
    ref = np.array([[3.0, 4.0], [np.inf, 2.0]])
    got = ref + np.array([[0.5, 1.0], [7.0, 0.25]])
    e = rel_err(got, ref)                                  # rms of each row, the non-finite entry counted as 0
    assert np.all(np.isfinite(e)) and e[1, 0] == 0
    np.testing.assert_allclose(e[0], [0.5, 1.0] / np.sqrt(12.5))
    np.testing.assert_allclose(e[1], [0.0, 0.25 / np.sqrt(2.0)])
    np.testing.assert_allclose(rel_err(got[:1], ref[:1], axis=None), [[0.5, 1.0]] / np.sqrt(12.5))
    np.testing.assert_allclose(rel_err(got[:1], ref[:1], scale=np.abs(ref[:1])), [[0.5 / 3, 0.25]])


def test_cnormal_has_unit_variance():
    z = cnormal(np.random.default_rng(1), (200, 1000))
    assert z.dtype == np.complex64
    assert abs(np.mean(np.abs(z) ** 2) - 1.0) < 0.01
    assert abs(np.var(z.real) - 0.5) < 0.01 and abs(np.var(z.imag) - 0.5) < 0.01
    assert cnormal(np.random.default_rng(1), 3, dtype=np.complex128).dtype == np.complex128


def test_noise_covariance_is_hermitian_positive_definite():
    s = noise_covariance(np.random.default_rng(2), 64, 8, 0.1).astype(np.complex128)
    np.testing.assert_allclose(s, np.conj(np.swapaxes(s, -1, -2)), atol=1e-7)
    assert np.linalg.eigvalsh(s).min() >= 0.1 * (1 - 1e-5)   # no (I + PSD)


def test_lifted_pcm_has_the_degrees_of_its_base_graph():
    rng = np.random.default_rng(3)
    z, rows, cols = 7, 5, 9
    base = rng.random((rows, cols)) < 0.5
    base[:, 0] = True                                      # every row and column non-empty
    base[0, :] = True
    br, bc = np.nonzero(base)
    sh = rng.integers(0, z, len(br))
    pcm = lifted_pcm(z, rows, cols, z, br, bc, sh)
    assert pcm.shape == (rows * z, cols * z)
    assert np.array_equal(pcm.sum(1), np.repeat(base.sum(1), z))
    assert np.array_equal(pcm.sum(0), np.repeat(base.sum(0), z))
    cut = lifted_pcm(z, rows, cols, 3, br, bc, sh)         # last block row cut to 3 checks
    assert cut.shape == ((rows - 1) * z + 3, cols * z) and np.array_equal(cut, pcm[:(rows - 1) * z + 3])


def test_bpsk_llr_batch_converges_at_its_high_snr_end():
    k, n, bs = 1024, 2048, 40
    rng = np.random.default_rng(4)
    enc = O.LDPC5GEncoderRef(k, n)
    c = enc(rng.integers(0, 2, (bs, k)))
    llr = bpsk_llr(c, np.repeat([-1.0, 5.0], bs // 2), k / n, rng)
    assert llr.dtype == np.float32 and llr.shape == c.shape
    x = O.LDPC5GDecoderRef(enc, hard_out=False, return_infobits=False, num_iter=20)(llr)
    assert np.array_equal(x[bs // 2:] > 0, c[bs // 2:] > 0)   # 5 dB: every codeword error-free
    assert_mixed_convergence(x, c, 2)
