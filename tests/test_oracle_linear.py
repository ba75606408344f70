"""The ZF / MF / pseudo-inverse / symbol-demapper oracle (oracle/linear.py) against independent formulas: numpy's SVD
pseudo-inverse, the closed-form MF error variance, scipy's log_softmax, and a per-element loop for the OFDM wrapper."""
import numpy as np
import pytest
from scipy.special import log_softmax

from oracle import linear as L
from oracle import mapping as MAP
from oracle import ofdm as F
from oracle.parity import cnormal, mimo_problem


@pytest.mark.parametrize("m,k", [(1, 1), (4, 2), (8, 8), (16, 4)])
def test_zf_and_pinv_match_the_svd_pseudo_inverse(m, k):
    rng = np.random.default_rng(m * 10 + k)
    y, h, s = (v.astype(np.complex128) for v in mimo_problem(rng, 50, m, k, MAP.qam(4), 0.1))
    p = np.linalg.pinv(h)
    np.testing.assert_allclose(L.matrix_pinv(h), p, atol=1e-9)
    x, ne = L.zf_equalizer(y, h, s)
    np.testing.assert_allclose(x, (p @ y[..., None])[..., 0], atol=1e-9)
    ref = np.real(np.einsum("nkm,nma,nka->nk", p, s, np.conj(p)))
    np.testing.assert_allclose(ne, ref, rtol=1e-9)


@pytest.mark.parametrize("m,k", [(1, 1), (4, 2), (8, 8), (16, 4)])
def test_mf_matches_the_closed_form_error(m, k):
    rng = np.random.default_rng(100 + m * 10 + k)
    y, h, s = (v.astype(np.complex128) for v in mimo_problem(rng, 50, m, k, MAP.qam(4), 0.1))
    x, ne = L.mf_equalizer(y, h, s)
    b = np.conj(np.swapaxes(h, -1, -2)) @ h
    bkk = np.real(np.diagonal(b, axis1=-2, axis2=-1))
    off = np.sum(np.abs(b) ** 2, axis=-1) - bkk ** 2
    q = np.real(np.einsum("nmk,nma,nak->nk", np.conj(h), s, h))
    np.testing.assert_allclose(ne, (off + q) / bkk ** 2, rtol=1e-9)
    np.testing.assert_allclose(x, np.einsum("nmk,nm->nk", np.conj(h), y) / bkk, rtol=1e-9)


def test_symbol_demap_matches_scipy_log_softmax():
    rng = np.random.default_rng(7)
    pts = MAP.qam(4)
    y = cnormal(rng, (3, 50)).astype(np.complex128)
    no = rng.uniform(0.05, 1.0, (3,))
    prior = rng.normal(size=(50, 16))
    e = -np.abs(y[..., None] - pts) ** 2 / no[:, None, None] + prior
    np.testing.assert_allclose(L.symbol_demap(y, no, pts, prior), log_softmax(e, axis=-1), atol=1e-12)
    np.testing.assert_array_equal(L.symbol_demap(y, no, pts, prior, hard_out=True), np.argmax(e, axis=-1))
    f32 = L.symbol_demap(y, no, pts, prior, dtype=np.float32)
    assert f32.dtype == np.float32
    np.testing.assert_allclose(f32, log_softmax(e, axis=-1), atol=1e-4)


@pytest.mark.parametrize("eq", ["zf", "mf", "lmmse-no-whitening"])
def test_ofdm_wrapper_equals_a_per_element_loop(eq):
    """One receiver, no interference: every data element of the OFDM wrapper equals the dense equaliser on that
    element's y, H and S = diag(no + sum err_var)."""
    rng = np.random.default_rng(5)
    b, ant, k, s_, f_ = 2, 3, 2, 3, 4
    mask = F.kronecker_mask(1, k, s_, f_, [1])
    smr = F.stream_management(np.ones((1, 1), int), k)
    h = cnormal(rng, (b, 1, ant, 1, k, s_, f_)).astype(np.complex128)
    y = cnormal(rng, (b, 1, ant, s_, f_)).astype(np.complex128)
    ev = 0.01 * rng.uniform(size=h.shape)
    no = rng.uniform(0.05, 0.1, (b, 1, ant))
    x, ne = L.ofdm_equalize(y, h, ev, no, mask, smr, eq)
    data = np.flatnonzero(~mask[0, 0].reshape(-1).astype(bool))
    for bi in range(b):
        for j, re in enumerate(data):
            si, fi = divmod(re, f_)
            hh = h[bi, 0, :, 0, :, si, fi]
            ss = np.diag(no[bi, 0] + ev[bi, 0, :, 0, :, si, fi].sum(-1)).astype(np.complex128)
            xr, nr = L.OFDM_EQUALIZERS[eq](y[bi, 0, :, si, fi], hh, ss)
            np.testing.assert_allclose(x[bi, 0, :, j], xr, rtol=1e-10)
            np.testing.assert_allclose(ne[bi, 0, :, j], nr, rtol=1e-10)
