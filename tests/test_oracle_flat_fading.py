"""The flat-fading oracle against closed-form properties, and the host-side correlation helpers `exp_corr_mat` /
`one_ring_corr_mat` against the oracle in float64 over the reference's grids (no GPU: the helpers are host NumPy, so
the tests place their outputs on the CPU)."""
import numpy as np
import pytest
import torch

from oracle import flat_fading as O


@pytest.fixture
def on_cpu():
    from sionna_b200.phy import config
    old = config._device
    config.device = "cpu"
    yield
    config._device = old


def _hermitian_toeplitz(r):
    assert np.allclose(r, np.conj(np.swapaxes(r, -1, -2)), atol=0, rtol=0)
    n = r.shape[-1]
    for d in range(n):
        diag = np.diagonal(r, -d, -2, -1)
        assert np.all(diag == diag[..., :1])


@pytest.mark.parametrize("a", [0.0, 0.5, 0.9, 0.5 + 0.3j, -0.7j])
@pytest.mark.parametrize("n", [1, 2, 7, 32])
def test_exp_corr_closed_form(a, n):
    r = O.exp_corr(a, n)
    _hermitian_toeplitz(r)
    assert np.allclose(r[:, 0], a ** np.arange(n))
    assert np.linalg.eigvalsh(r).min() > 0                       # positive definite for |a| < 1
    l = O.chol(r)
    assert np.allclose(l @ np.conj(l.T), r, atol=1e-12)
    assert np.allclose(np.triu(l, 1), 0)
    # det R = (1 - |a|^2)^(n - 1)
    assert np.isclose(np.linalg.det(r).real, (1 - abs(a) ** 2) ** (n - 1), rtol=1e-9)


@pytest.mark.parametrize("phi", [-60, -15, 0, 30, 75])
@pytest.mark.parametrize("sigma", [2, 10, 15])
def test_one_ring_closed_form(phi, sigma):
    r = O.one_ring(phi, 16, 0.5, sigma)
    _hermitian_toeplitz(r)
    assert np.allclose(np.diagonal(r), 1)
    assert np.linalg.eigvalsh(r).min() > -1e-12                  # positive semi-definite
    if np.linalg.cond(r) < 1e10:
        l = O.chol(r)
        assert np.allclose(l @ np.conj(l.T), r, atol=1e-10)


def test_products_closed_form():
    rng = np.random.default_rng(0)
    h = rng.normal(size=(3, 5, 4)) + 1j * rng.normal(size=(3, 5, 4))
    l_tx, l_rx = O.chol(O.exp_corr(0.4, 4)), O.chol(O.exp_corr(0.7 - 0.2j, 5))
    ref = np.stack([l_rx @ h[i] @ np.conj(l_tx.T) for i in range(3)])
    assert np.allclose(O.kronecker(h, l_tx, l_rx), ref)
    lk = O.chol(O.one_ring([-30, 0, 20, 45], 5, 0.5, 10))
    pc = O.per_column(h, lk)
    for k in range(4):
        assert np.allclose(pc[:, :, k], (lk[k] @ h[:, :, k, None])[..., 0])
    x = rng.normal(size=(3, 4)) + 0j
    assert np.allclose(O.apply(h, x), np.einsum("bmk,bk->bm", h, x))
    # the draw has unit variance per complex entry
    w = O.draw(5, 2 ** 32 + 7, 20000, 4, 3)
    assert abs(np.mean(np.abs(w) ** 2) - 1) < 0.02


@pytest.mark.parametrize("a", [0.0, 0.9999, 0.5 + 0.3j])
@pytest.mark.parametrize("n", [1, 2, 4, 7, 64, 128])
def test_exp_corr_mat_grid(on_cpu, a, n):
    from sionna_b200.phy.channel import exp_corr_mat
    r = exp_corr_mat(a, n, precision="double")
    assert r.dtype == torch.complex128 and r.shape == (n, n)
    assert np.max(np.abs(r.numpy() - O.exp_corr(a, n))) < 1e-12
    r32 = exp_corr_mat(a, n)
    assert r32.dtype == torch.complex64
    assert np.max(np.abs(r32.numpy() - O.exp_corr(a, n))) < 1e-6
    if a == 0:
        assert np.array_equal(r.numpy(), np.eye(n))


def test_exp_corr_mat_multiple_dims(on_cpu):
    from sionna_b200.phy.channel import exp_corr_mat
    from sionna_b200.phy.channel.utils import exp_corr_mat as from_utils
    assert from_utils is exp_corr_mat
    a = np.random.default_rng(1).uniform(0, 1, [2, 4, 3])
    r = exp_corr_mat(a, 11, precision="double")
    assert r.shape == (2, 4, 3, 11, 11)
    for i, ai in enumerate(a.reshape(-1)):
        assert np.max(np.abs(r.reshape(-1, 11, 11)[i].numpy() - O.exp_corr(ai, 11))) < 1e-12


@pytest.mark.parametrize("a", [1.1 + 0.3j, 1.0, -1.0, [0.5, 1.0]])
def test_exp_corr_mat_rejects_abs_one(on_cpu, a):
    from sionna_b200.phy.channel import exp_corr_mat
    with pytest.raises(ValueError, match="smaller than one"):
        exp_corr_mat(a, 12)


@pytest.mark.parametrize("phi", [-180, -90, -45, -12, 0, 15, 45, 65, 90, 180, 360])
@pytest.mark.parametrize("num_ant", [1, 4, 16, 128])
def test_one_ring_corr_mat_grid(on_cpu, phi, num_ant):
    from sionna_b200.phy.channel import one_ring_corr_mat
    for d_h in [0, 0.2, 0.5, 1, 3]:
        for sigma in [0, 2, 5, 15]:
            r = one_ring_corr_mat(phi, num_ant, d_h, sigma, precision="double")
            assert r.shape == (num_ant, num_ant) and r.dtype == torch.complex128
            assert np.max(np.abs(r.numpy() - O.one_ring(phi, num_ant, d_h, sigma))) < 1e-12


def test_one_ring_corr_mat_multiple_dims(on_cpu):
    from sionna_b200.phy.channel import one_ring_corr_mat
    phi = np.random.default_rng(2).uniform(-np.pi, np.pi, [2, 4, 3])
    r = one_ring_corr_mat(phi, 32, 0.7, 10, precision="double")
    assert r.shape == (2, 4, 3, 32, 32)
    assert np.max(np.abs(r.numpy() - O.one_ring(phi, 32, 0.7, 10))) < 1e-12


def test_one_ring_corr_mat_warns_above_15_degrees(on_cpu):
    from sionna_b200.phy.channel import one_ring_corr_mat
    with pytest.warns(UserWarning, match="smaller than 15"):
        one_ring_corr_mat(35, 32, 0.7, 16)
