"""The K-Best oracle (oracle/kbest.py) reproduces the reference's own K-Best assertions (test_kbest_det.py): with
k = |C|^S and no clipping its LLRs are the maxlog ML LLRs, and noiseless problems are detected without errors."""
import numpy as np
import pytest

from oracle import mapping as MAP
from oracle.kbest import kbest_detect, qam_from_pam
from oracle.mimo import ml_detect


def _flat_fading(rng, num, m, k, points, no):
    """FlatFadingChannel: h ~ CN(0, 1) [num, m, k], y = h x + CN(0, no) noise; returns y, h, indices."""
    h = (rng.normal(size=(num, m, k)) + 1j * rng.normal(size=(num, m, k))) / np.sqrt(2)
    ind = rng.integers(0, len(points), (num, k))
    n = (rng.normal(size=(num, m)) + 1j * rng.normal(size=(num, m))) * np.sqrt(no / 2)
    return (h @ points[ind][..., None])[..., 0] + n, h, ind


@pytest.mark.parametrize("ebno_db", [-20, -10, 0, 10, 20, 30, 50])
@pytest.mark.parametrize("kind,bits,real_rep", [("qam", 2, False), ("qam", 4, False), ("qam", 2, True),
                                                ("qam", 4, True), ("pam", 1, False), ("pam", 2, False),
                                                ("pam", 3, False), ("pam", 4, False)])
def test_full_k_llrs_equal_maxlog_ml(kind, bits, real_rep, ebno_db):
    rng = np.random.default_rng(1000 + 10 * bits + ebno_db + 7 * real_rep + (kind == "pam"))
    # QAM built from the real representation's PAM levels in float64, so both detectors see the same points
    pts = qam_from_pam(bits) if kind == "qam" else MAP.pam(bits).astype(np.complex128)
    no = MAP.ebnodb2no(ebno_db, bits, 1.0)
    y, h, _ = _flat_fading(rng, 100, 8, 3, pts, no)
    s = no * np.eye(8)
    llr, _ = kbest_detect(y, h, s, pts, len(pts) ** 3, "bit", real_rep=real_rep, llr_clip=np.inf)
    ml = ml_detect(y, h, s, pts, "maxlog", "bit")
    assert np.allclose(llr, ml, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("output", ["symbol", "bit"])
@pytest.mark.parametrize("kind,bits,real_rep", [("qam", b, r) for b in (2, 4, 6, 8) for r in (False, True)] +
                         [("pam", b, False) for b in (1, 2, 3, 4)])
def test_noiseless_problems_have_no_errors(kind, bits, real_rep, output):
    rng = np.random.default_rng(50 + bits + 3 * real_rep + (output == "bit"))
    pts = MAP.qam(bits) if kind == "qam" else MAP.pam(bits)
    k, streams, ant = (64, 3, 7) if kind == "qam" else (16, 4, 8 if output == "symbol" else 7)
    y, h, ind = _flat_fading(rng, 100, ant, streams, pts, 0.0)
    s = 1e-9 * np.eye(ant)
    got, _ = kbest_detect(y, h, s, pts, k, output, hard_out=True, real_rep=real_rep)
    if output == "symbol":
        assert np.array_equal(got, ind)
    else:
        assert np.array_equal(got, (ind[..., None] >> np.arange(bits - 1, -1, -1)) & 1)


def test_clip_and_real_rep_bit_order():
    """The real representation's LLRs interleave real (even) and imaginary (odd) bits; clipping bounds every LLR."""
    rng = np.random.default_rng(4)
    pts = qam_from_pam(4)
    y, h, _ = _flat_fading(rng, 64, 4, 2, pts, 0.01)
    s = 0.01 * np.eye(4)
    full_c, _ = kbest_detect(y, h, s, pts, 256, "bit", llr_clip=np.inf)
    full_r, _ = kbest_detect(y, h, s, pts, 256, "bit", real_rep=True, llr_clip=np.inf)
    assert np.allclose(full_c, full_r, rtol=1e-9, atol=1e-9)
    clipped, _ = kbest_detect(y, h, s, pts, 4, "bit", llr_clip=20.0)
    assert np.abs(clipped).max() <= 20.0 and np.isin(20.0, np.abs(clipped))
