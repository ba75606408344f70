"""The float64 precoding oracle (oracle/precoding.py) against properties that need no TensorFlow: zero forcing
diagonalises the channel, every precoding column has unit norm, ZF equals the column-normalised pseudo-inverse, RZF
tends to CBF as alpha grows, and the OFDM gather and effective channel equal a literal per-(receiver, transmitter)
loop written as in the reference's test/unit/ofdm/test_precoded_channel.py:53-71."""
import numpy as np

from oracle import precoding as P
from oracle.parity import cnormal


def _h(rng, shape):
    return cnormal(rng, shape, dtype=np.complex128)


def test_zf_diagonalises_the_channel():
    rng = np.random.default_rng(1)
    h = _h(rng, (64, 10, 15))
    g = P.rzf_precoding_matrix(h, 0.)
    hg = h @ g
    off = hg - np.eye(10) * np.diagonal(hg, axis1=-2, axis2=-1)[..., None, :]
    assert np.linalg.norm(off) < 1e-10 * np.linalg.norm(hg)


def test_unit_norm_columns():
    rng = np.random.default_rng(2)
    h = _h(rng, (32, 4, 8))
    for g in (P.rzf_precoding_matrix(h, 0.3), P.cbf_precoding_matrix(h)):
        assert np.allclose(np.linalg.norm(g, axis=-2), 1.0)
        assert np.allclose(np.trace(g @ np.conj(np.swapaxes(g, -1, -2)), axis1=-2, axis2=-1), 4.0)


def test_zf_equals_normalised_pseudo_inverse():
    rng = np.random.default_rng(3)
    h = _h(rng, (16, 6, 9))
    p = np.linalg.pinv(h)
    p = p / np.linalg.norm(p, axis=-2, keepdims=True)
    assert np.allclose(P.rzf_precoding_matrix(h, 0.), p, atol=1e-10)


def test_large_alpha_tends_to_cbf():
    rng = np.random.default_rng(4)
    h = _h(rng, (16, 4, 8))
    assert np.allclose(P.rzf_precoding_matrix(h, 1e9), P.cbf_precoding_matrix(h), atol=1e-7)


def test_zero_channel_gives_zero_columns():
    g = P.cbf_precoding_matrix(np.zeros((2, 3, 5), np.complex128))
    assert np.all(g == 0)


def test_ofdm_gather_and_effective_channel_equal_literal_loop():
    """2 transmitters, each serving 2 of 4 two-antenna receivers: h_eff also holds the off-association entries."""
    from oracle.ofdm import eff_sc_ind
    rng = np.random.default_rng(5)
    b, rx, ra, tx, m, s_, f_ = 3, 4, 2, 2, 6, 2, 12
    assoc = np.zeros((rx, tx), np.int32)
    for j in range(tx):
        assoc[2 * j:2 * j + 2, j] = 1
    pind = np.stack([np.where(assoc[:, j])[0] for j in range(tx)])
    k = 2 * ra
    h = _h(rng, (b, rx, ra, tx, m, s_, f_))
    x = _h(rng, (b, tx, k, s_, f_))
    pw = rng.uniform(size=(b, tx, k, s_, f_))
    alpha = rng.uniform(size=(b, tx, 1, 1))
    eff = eff_sc_ind(f_, (1, 2), True)
    xp, h_eff = P.ofdm_precode("rzf", h, pind, eff, x=x, alpha=alpha, alpha_left=True, tx_power=pw)
    for j in range(tx):
        rx_ind = np.where(assoc[:, j])[0]
        h_des = h[:, rx_ind][:, :, :, j]                                    # [b, 2, ra, m, s, f]
        h_des = np.transpose(h_des.reshape(b, -1, m, s_, f_), (0, 3, 4, 1, 2))
        g = P.rzf_precoding_matrix(h_des, alpha[:, j])                     # [b, s, f, m, k]
        assert np.allclose(np.transpose(xp[:, j], (0, 2, 3, 1)), (g @ np.transpose(x[:, j], (0, 2, 3, 1))[..., None])[..., 0])
        g = np.sqrt(np.transpose(pw[:, j], (0, 2, 3, 1)))[..., None, :] * g
        for i in range(rx):
            h_ij = np.transpose(h[:, i, :, j], (0, 3, 4, 1, 2))             # [b, s, f, ra, m]
            q = np.transpose(h_eff[:, i, :, j], (0, 3, 4, 1, 2))            # [b, s, ne, ra, k]
            assert np.allclose(q, (h_ij @ g)[:, :, eff])
    assert h_eff.shape == (b, rx, ra, tx, k, s_, len(eff))
    # the interference toward the other transmitter's receivers is not zero
    assert np.abs(h_eff[:, 2:, :, 0]).max() > 0.1


def test_eye_and_single_precision_sequence():
    from oracle.ofdm import eff_sc_ind
    rng = np.random.default_rng(6)
    h = _h(rng, (2, 1, 2, 1, 3, 1, 8))
    eff = eff_sc_ind(8, (0, 0), False)
    _, h_eff = P.ofdm_precode("eye", h, None, eff, tx_power=np.full((2, 1), 4.0))
    assert np.allclose(h_eff, 2 * h)
    g64 = P.rzf_precoding_matrix(h[0, 0, :, 0, :, 0, :2].transpose(2, 0, 1), 0.1)
    g32 = P.rzf_precoding_matrix(h[0, 0, :, 0, :, 0, :2].transpose(2, 0, 1), 0.1, dtype=np.complex64)
    assert g32.dtype == np.complex64 and np.allclose(g32, g64, atol=1e-5)
