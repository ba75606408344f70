"""The EP and MMSE-PIC oracle (oracle/iterative.py) against the reference's own checks, on the CPU: EP makes no symbol
or bit errors on noise-free channels (test_ep_det.py), MMSE-PIC produces the reference's output shapes
(test_mmse_pic_det.py), and MMSE-PIC with a zero prior and one iteration is soft-output LMMSE with the same demapping
(maxlog: the identity the IDD tutorial starts from)."""
import numpy as np
import pytest

from oracle import mapping as MAP
from oracle.iterative import ep_detect, mmse_pic_detect
from oracle.mimo import logits_to_llrs
from oracle.ofdm import lmmse_equalizer


def _c(rng, shape):
    return (rng.normal(size=shape) + 1j * rng.normal(size=shape)) / np.sqrt(2)


@pytest.mark.parametrize("m", [2, 4, 6, 8])
def test_ep_noise_free_has_no_errors(m):
    rng = np.random.default_rng(m)
    pts = MAP.qam(m).astype(np.complex128)
    h = _c(rng, (100, 7, 3))
    ind = rng.integers(0, 2 ** m, (100, 3))
    y = (h @ pts[ind][..., None])[..., 0]
    s = 1e-4 * np.eye(7)
    sym, _ = ep_detect(y, h, s, m, "symbol", hard_out=True)
    bits, _ = ep_detect(y, h, s, m, "bit", hard_out=True)
    assert np.array_equal(sym, ind)
    assert np.array_equal(bits, (ind[..., None] >> np.arange(m - 1, -1, -1)) & 1)


@pytest.mark.parametrize("output,hard_out", [("bit", False), ("bit", True), ("symbol", False), ("symbol", True)])
def test_mmse_pic_shapes(output, hard_out):
    rng = np.random.default_rng(1)
    m, batch, mm, kk = 4, (3, 2), 6, 3
    pts = MAP.qam(m)
    y, h = _c(rng, batch + (mm,)), _c(rng, batch + (mm, kk))
    s = np.eye(mm) * 0.1
    prior = rng.normal(size=batch + (kk, m if output == "bit" else 2 ** m))
    out, margin = mmse_pic_detect(y, h, s, prior, pts, output, "app", 2, hard_out)
    want = batch + (kk,) if (output == "symbol" and hard_out) else batch + (kk, m if output == "bit" else 2 ** m)
    assert out.shape == want and margin.shape == batch
    out, _ = ep_detect(y, h, s, m, output, hard_out)
    assert out.shape == want


@pytest.mark.parametrize("method", ["maxlog", "app"])
def test_zero_prior_single_iteration_is_lmmse(method):
    rng = np.random.default_rng(2)
    m = 4
    pts = MAP.qam(m).astype(np.complex128)
    pts = pts / np.sqrt(np.mean(np.abs(pts) ** 2))          # unit energy in float64: the prior variance is exactly 1
    h = _c(rng, (500, 8, 4))
    ind = rng.integers(0, 16, (500, 4))
    s = 0.1 * np.eye(8) + 0j
    y = (h @ pts[ind][..., None])[..., 0] + np.sqrt(0.1) * _c(rng, (500, 8))
    out, _ = mmse_pic_detect(y, h, s, np.zeros((500, 4, m)), pts, "bit", method, 1)
    xh, ne = lmmse_equalizer(y, h, s)
    ref = logits_to_llrs(-np.abs(xh[..., None] - pts) ** 2 / ne[..., None], m, method)
    assert np.abs(out - ref).max() < 1e-10
