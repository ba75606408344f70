"""Pin the mapping / demapping oracle against the reference's closed forms and test recipes:
38.211 5.1 QAM formulas (test/unit/mapping/test_constellation.py:11-62), mapper index identity
(test_mapping.py:37-45), demapper app / maxlog vs scipy.special.logsumexp / np.max with atol 1e-5
(test_mapping.py:175-225), with priors (:398-478). The float64 reference `demapper_f64` against the same recipe, and the
kernel-math mode held to the single-precision envelope against it."""
import numpy as np
import pytest
from scipy.special import logsumexp

from oracle import mapping as M
from oracle import parity as P


def _bpsk(b):
    return (1 - 2 * b[0] + 1j * (1 - 2 * b[0])) / np.sqrt(2)


def _qpsk(b):
    return (1 - 2 * b[0] + 1j * (1 - 2 * b[1])) / np.sqrt(2)


def _qam16(b):
    return ((1 - 2 * b[0]) * (2 - (1 - 2 * b[2])) + 1j * (1 - 2 * b[1]) * (2 - (1 - 2 * b[3]))) / np.sqrt(10)


def _qam64(b):
    return ((1 - 2 * b[0]) * (4 - (1 - 2 * b[2]) * (2 - (1 - 2 * b[4])))
            + 1j * (1 - 2 * b[1]) * (4 - (1 - 2 * b[3]) * (2 - (1 - 2 * b[5])))) / np.sqrt(42)


@pytest.mark.parametrize("m,f", [(2, _qpsk), (4, _qam16), (6, _qam64)])
def test_qam_38211(m, f):
    c = M.qam(m)
    for i in range(2 ** m):
        b = np.array(list(np.binary_repr(i, m)), dtype=np.int32)
        assert np.allclose(c[i], f(b), atol=1e-6)
    assert np.isclose(np.mean(np.abs(c) ** 2), 1.0, atol=1e-6)


def test_pam_energy_and_gray():
    for m in (1, 2, 3, 4):
        c = M.pam(m)
        assert np.isclose(np.mean(np.abs(c) ** 2), 1.0, atol=1e-6)
        order = np.argsort(c.real)
        labels = [np.binary_repr(i, m) for i in order]
        assert all(sum(a != b for a, b in zip(x, y)) == 1 for x, y in zip(labels[:-1], labels[1:]))


def test_mapper_index_identity():
    for m in (2, 4, 6, 8):
        pts = M.qam(m)
        idx = np.arange(2 ** m)
        bits = ((idx[:, None] >> np.arange(m - 1, -1, -1)) & 1).reshape(-1)
        x, ind = M.mapper(bits, pts)
        assert np.array_equal(ind, idx) and np.array_equal(x, pts)


def _ref_llr(y, no, pts, method, prior=None):
    m = int(np.log2(len(pts)))
    e = -np.abs(y[..., None].astype(np.complex128) - pts.astype(np.complex128)) ** 2 / np.asarray(no, np.float64)[..., None]
    if prior is not None:
        lab = 2.0 * ((np.arange(2 ** m)[:, None] >> np.arange(m - 1, -1, -1)) & 1) - 1.0
        lp = np.sum(-np.log1p(np.exp(-lab * np.asarray(prior, np.float64)[..., None, :])), axis=-1)
        e = e + lp
    out = np.zeros(y.shape + (m,))
    for i in range(m):
        s1 = [j for j in range(2 ** m) if (j >> (m - 1 - i)) & 1]
        s0 = [j for j in range(2 ** m) if not (j >> (m - 1 - i)) & 1]
        if method == "app":
            out[..., i] = logsumexp(e[..., s1], axis=-1) - logsumexp(e[..., s0], axis=-1)
        else:
            out[..., i] = np.max(e[..., s1], axis=-1) - np.max(e[..., s0], axis=-1)
    return out.reshape(y.shape[:-1] + (-1,))


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("method", ["app", "maxlog"])
@pytest.mark.parametrize("m", [2, 4, 6])
def test_demapper_vs_scipy(m, method, mode):
    rng = np.random.default_rng(m)
    pts = M.qam(m)
    b = rng.integers(0, 2, (7, 20 * m))
    x, _ = M.mapper(b, pts)
    no_scalar = 0.25
    y = (x + (rng.normal(size=x.shape) + 1j * rng.normal(size=x.shape)) * np.sqrt(no_scalar / 2)).astype(np.complex64)
    llr = M.demapper(y, no_scalar, pts, method, math_mode=mode)
    assert np.allclose(llr, _ref_llr(y, np.full(y.shape, no_scalar), pts, method), atol=1e-5 * max(1, np.abs(llr).max()) , rtol=1e-5)
    no_sym = rng.uniform(0.05, 1.0, size=y.shape).astype(np.float32)          # per-symbol noise variance
    llr = M.demapper(y, no_sym, pts, method, math_mode=mode)
    assert np.allclose(llr, _ref_llr(y, no_sym, pts, method), atol=1e-4, rtol=1e-5)
    prior = rng.normal(size=y.shape + (m,)).astype(np.float32)
    llr = M.demapper(y, no_scalar, pts, method, prior=prior, math_mode=mode)
    assert np.allclose(llr, _ref_llr(y, np.full(y.shape, no_scalar), pts, method, prior), atol=1e-4, rtol=1e-5)


@pytest.mark.parametrize("prior_shape", [None, "bits", "full"])
@pytest.mark.parametrize("method", ["app", "maxlog"])
def test_demapper_f64_vs_scipy(method, prior_shape):
    """The float64 reference equals the reference's test recipe (scipy logsumexp / max over the two index sets) on the
    2-D formula, with per-symbol no, for 64-QAM and a 5-bit custom constellation."""
    rng = np.random.default_rng(5)
    for pts in (M.qam(6), (rng.normal(size=32) + 1j * rng.normal(size=32)).astype(np.complex64)):
        m = int(np.log2(len(pts)))
        y = (rng.normal(size=(3, 40)) + 1j * rng.normal(size=(3, 40))).astype(np.complex64)
        no = rng.uniform(0.05, 1.0, y.shape).astype(np.float32)
        prior = {None: None, "bits": rng.normal(size=m), "full": rng.normal(size=y.shape + (m,))}[prior_shape]
        prior = None if prior is None else prior.astype(np.float32)
        ref = _ref_llr(y, no, pts, method, None if prior is None else np.broadcast_to(prior, y.shape + (m,)))
        np.testing.assert_allclose(M.demapper_f64(y, no, pts, method, prior), ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("inputs", ["noisy", "window"])
@pytest.mark.parametrize("method", ["app", "maxlog"])
@pytest.mark.parametrize("m", [2, 4, 6, 8, 10])
def test_kernel_math_demapper_envelope(m, method, inputs):
    """What the separable square-QAM kernel computes (the oracle's kernel-math mode, which the GPU kernel equals bit for
    bit) stays within 2x (rms) / 3x (max) of the libm 2-D formula's error against the float64 reference, errors relative
    to the rms of each row's reference LLRs. "noisy": constellation points plus noise at 40 noise variances from 1e-4 to 3;
    "window": y uniform over the constellation, no swept so that |LLR| crosses 60 ... 100, where a bit group's members
    fall below exp's underflow relative to the dimension's largest exponent while still comparable to the group's own."""
    rng = np.random.default_rng(100 + m)
    pts = M.qam(m)
    y, no = (P.demap_noisy if inputs == "noisy" else P.demap_window)(rng, pts, 256)
    no = no[:, None]
    ref = M.demapper_f64(y, no, pts, method)
    if inputs == "window":
        assert np.mean((np.abs(ref) > 60) & (np.abs(ref) < 100)) > 0.05
    bad = P.envelope(f"m={m} {method} {inputs}", M.demapper(y, no, pts, method, math_mode=1),
                     M.demapper(y, no, pts, method, math_mode=0), ref, (2.0, 3.0))
    assert not bad, bad


def test_ebnodb2no_and_hard_decisions():
    assert np.isclose(M.ebnodb2no(4.0, 2, 1.0), 1 / (10 ** 0.4 * 2), rtol=1e-6)
    assert np.array_equal(M.hard_decisions(np.array([-1.0, 0.0, 2.0])), [0, 0, 1])
