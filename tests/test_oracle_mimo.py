"""The ML-detection oracle (oracle/mimo.py) against an independent formula: the quadratic form
-(y - H x)^H S^-1 (y - H x) per candidate and explicit per-(stream, point) loops, as the reference's own
test/unit/mimo/test_mimo_ml_det.py::test_logits_calc_eager computes them. CPU only."""
import numpy as np
import pytest
from scipy.stats import unitary_group

from oracle.mapping import qam as qam_points
from oracle.mimo import build_vecs, ml_detect


def _eager_vecs(points, k):
    """Candidate list of test_logits_calc_eager: stream k's point repeats in blocks of |C|^(K-k-1)."""
    n = len(points)
    vecs = np.zeros((n ** k, k), complex)
    ind = np.zeros((n ** k, k), int)
    for j in range(k):
        tile_point, tile_const = n ** (k - j - 1), n ** j
        for t in range(tile_const):
            for i, p in enumerate(points):
                lo = t * n * tile_point + i * tile_point
                vecs[lo:lo + tile_point, j] = p
                ind[lo:lo + tile_point, j] = i
    return vecs, ind


def _problem(rng, batch, m_ant, k, npts, with_prior):
    y = rng.normal(size=(batch, m_ant)) + 1j * rng.normal(size=(batch, m_ant))
    h = rng.normal(size=(batch, m_ant, k)) + 1j * rng.normal(size=(batch, m_ant, k))
    e = rng.uniform(0.5, 2.0, size=(batch, m_ant))
    u = unitary_group.rvs(dim=m_ant, random_state=rng) if m_ant > 1 else np.ones((1, 1))
    s = u[None] @ (np.eye(m_ant)[None] * e[:, None, :]) @ np.conj(u.T)[None]
    prior = rng.normal(size=(batch, k, npts)) if with_prior else None
    return y, h, s, prior


def _eager_logits(y, h, s, prior, points, k, method):
    vecs, ind = _eager_vecs(points, k)
    diff = y[:, None, :] - np.einsum("nmk,vk->nvm", h, vecs)
    s_inv = np.linalg.inv(s)
    ex = -np.einsum("nvm,nml,nvl->nv", np.conj(diff), s_inv, diff).real
    if prior is not None:
        ex = ex + sum(prior[:, j, ind[:, j]] for j in range(k))
    n = len(points)
    out = np.zeros((y.shape[0], k, n))
    for j in range(k):
        for i in range(n):
            sel = ex[:, ind[:, j] == i]
            if method == "app":
                mx = sel.max(-1, keepdims=True)
                out[:, j, i] = np.log(np.exp(sel - mx).sum(-1)) + mx[:, 0]
            else:
                out[:, j, i] = sel.max(-1)
    return out


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_candidate_order_matches_build_vecs(k):
    pts = qam_points(2)
    vecs, ind, c = build_vecs(pts, k)
    ev, ei = _eager_vecs(pts, k)
    np.testing.assert_array_equal(ind, ei)
    np.testing.assert_array_equal(vecs, ev)
    for j in range(k):
        for i in range(4):
            assert np.all(ind[c[:, j, i], j] == i)


@pytest.mark.parametrize("method", ["app", "maxlog"])
@pytest.mark.parametrize("with_prior", [False, True])
@pytest.mark.parametrize("m,k", [(2, 1), (2, 2), (2, 3), (2, 4), (4, 1), (4, 2), (4, 3), (4, 4)])
def test_oracle_logits_against_quadratic_form(method, with_prior, m, k):
    rng = np.random.default_rng(1000 * m + 10 * k + with_prior)
    pts = qam_points(m)
    batch = 3 if m ** k < 4 ** 4 else 2
    y, h, s, prior = _problem(rng, batch, 4, k, 2 ** m, with_prior)
    want = _eager_logits(y, h, s, prior, pts, k, method)
    got = ml_detect(y, h, s, pts, method, "symbol", prior=prior)
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-9)
    hard = ml_detect(y, h, s, pts, method, "symbol", prior=prior, hard_out=True)
    np.testing.assert_array_equal(hard, np.argmax(want, -1))


@pytest.mark.parametrize("method", ["app", "maxlog"])
def test_oracle_bits_follow_symbol_logits(method):
    """Bit LLRs are SymbolLogits2LLRs of the symbol logits; bit priors enter as LLRs2SymbolLogits."""
    rng = np.random.default_rng(7)
    pts = qam_points(4)
    y, h, s, _ = _problem(rng, 3, 3, 2, 16, False)
    bit_prior = rng.normal(size=(3, 2, 4))
    lab = (np.arange(16)[:, None] >> np.arange(3, -1, -1)) & 1
    sym_prior = np.sum(-np.log1p(np.exp(-(2 * lab - 1) * bit_prior[:, :, None, :])), -1)
    logits = _eager_logits(y, h, s, sym_prior, pts, 2, method)
    red = (lambda x: np.log(np.exp(x).sum(-1))) if method == "app" else (lambda x: x.max(-1))
    want = np.stack([red(logits[..., lab[:, i] == 1]) - red(logits[..., lab[:, i] == 0]) for i in range(4)], -1)
    got = ml_detect(y, h, s, pts, method, "bit", prior=bit_prior)
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-9)
    hard = ml_detect(y, h, s, pts, method, "bit", prior=bit_prior, hard_out=True)
    np.testing.assert_array_equal(hard, (want > 0).astype(float))
