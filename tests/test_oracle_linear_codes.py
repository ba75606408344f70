"""CPU tests of the linear-code utilities (sionna_b200.phy.fec.utils) and of oracle/linear_codes.py: the reference's
unit-test expectations for alist / make_systematic / pcm2gm / gm2pcm / verify_gm_pcm / int_mod_2, the three facts the
OSD kernel relies on (row-pivot MRB = greedy MRB, the discrepancy form decides as the softplus metric, OSD of order k =
ML), and that the package's conversions equal the oracle's loop forms."""
import os

import numpy as np
import pytest
import torch

from oracle import linear_codes as O
from sionna_b200.phy.fec.utils import (alist2mat, load_alist, make_systematic, gm2pcm, pcm2gm, verify_gm_pcm,
                                       int_mod_2, load_parity_check_examples)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _full_rank(rng, k, n):
    while True:
        g = rng.integers(0, 2, (k, n))
        if O.gf2_rank(g) == k:
            return g


def test_alist_explicit_example():
    alist = [[7, 3], [3, 4], [1, 1, 1, 2, 2, 2, 3], [4, 4, 4], [1, 0, 0], [2, 0, 0], [3, 0, 0], [1, 2, 0], [1, 3, 0],
             [2, 3, 0], [1, 2, 3], [1, 4, 5, 7], [2, 4, 6, 7], [3, 5, 6, 7]]
    pcm, k, n, r = alist2mat(alist, verbose=False)
    assert (k, n, r) == (4, 7, 4 / 7)
    assert np.array_equal(pcm, [[1, 0, 0, 1, 1, 0, 1], [0, 1, 0, 1, 0, 1, 1], [0, 0, 1, 0, 1, 1, 1]])
    assert np.array_equal(O.alist2mat(alist)[0], pcm)


def test_alist_wimax_file():
    alist = load_alist(os.path.join(GOLDEN, "wimax_576_0.5.alist"))
    pcm, k, n, r = alist2mat(alist, verbose=False)
    assert (k, n, r) == (288, 576, 0.5) and pcm.shape == (288, 576)
    assert np.array_equal(O.alist2mat(alist)[0], pcm)
    gm = pcm2gm(pcm)
    assert verify_gm_pcm(gm, pcm)


@pytest.mark.parametrize("pcm_id", range(5))
def test_example_codes_match_oracle(pcm_id):
    pcm, k, n, _ = load_parity_check_examples(pcm_id)
    gm = pcm2gm(pcm)
    assert gm.shape == (k, n) and verify_gm_pcm(gm, pcm)
    assert np.array_equal(gm, O.pcm2gm(pcm))
    s, sw = make_systematic(pcm, is_pcm=True)
    s2, sw2 = O.make_systematic(pcm, is_pcm=True)
    assert np.array_equal(s, s2) and sw == sw2
    p2 = gm2pcm(pcm)                                        # the pcm read as a generator
    assert verify_gm_pcm(pcm, p2) and np.array_equal(p2, O.gm2pcm(pcm))


def test_verify_gm_pcm_rejects():
    with pytest.raises(AssertionError):
        verify_gm_pcm(np.zeros((20, 12)), np.zeros((20, 12)))
    with pytest.raises(AssertionError):
        verify_gm_pcm(np.zeros((20, 8)), np.zeros((20, 12)))
    pcm, _, _, _ = load_parity_check_examples(3)
    gm = pcm2gm(pcm)
    assert verify_gm_pcm(gm, pcm)
    assert not verify_gm_pcm(make_systematic(gm)[0], pcm)
    pcm, _, _, _ = load_parity_check_examples(0)
    gm = pcm2gm(pcm)
    g2, p2 = gm.copy(), pcm.copy()
    g2[0, 0] = 2
    p2[0, 0] = 2
    with pytest.raises(AssertionError):
        verify_gm_pcm(g2, pcm)
    with pytest.raises(AssertionError):
        verify_gm_pcm(gm, p2)
    manual = np.array([[1, 0, 0, 0, 0, 1, 1], [0, 1, 0, 0, 1, 0, 1], [0, 0, 1, 0, 1, 0, 0], [0, 0, 0, 1, 0, 1, 0]])
    assert verify_gm_pcm(pcm2gm(manual, verify_results=False), manual)


def test_random_full_rank_matrices():
    rng = np.random.default_rng(1)
    for _ in range(200):
        k = int(rng.integers(1, 12))
        n = int(rng.integers(k + 1, 24))
        g = _full_rank(rng, k, n)
        s, sw = make_systematic(g)
        s2, sw2 = O.make_systematic(g)
        assert np.array_equal(s, s2) and sw == sw2 and np.array_equal(s[:, :k], np.eye(k))
        pcm = gm2pcm(g)
        assert verify_gm_pcm(g, pcm) and np.array_equal(pcm, O.gm2pcm(g))
        g2 = pcm2gm(pcm)
        assert verify_gm_pcm(g2, pcm) and np.array_equal(g2, O.pcm2gm(pcm))
        assert O.gf2_rank(np.concatenate([g, g2])) == k           # same code


def test_rank_deficient_raises():
    g = np.array([[1, 0, 1, 1], [0, 1, 1, 0], [1, 1, 0, 1]])
    with pytest.raises(ValueError):
        make_systematic(g)
    with pytest.raises(ValueError):
        pcm2gm(g)
    with pytest.raises(ValueError):
        gm2pcm(g)


def test_int_mod_2():
    x = torch.tensor([-3, -2, 0, 1, 4, 7])
    assert int_mod_2(x).tolist() == [1, 0, 0, 1, 0, 1]
    xf = torch.tensor([-3.2, -1.6, 0.4, 1.0, 2.6, 7.0], dtype=torch.float64)
    assert int_mod_2(xf).tolist() == [1.0, 0.0, 0.0, 1.0, 1.0, 1.0]
    assert int_mod_2(np.array([3, 4, -5])).tolist() == [1, 0, 1]


def test_row_pivot_mrb_equals_greedy_mrb():
    rng = np.random.default_rng(2)
    tested = 0
    while tested < 3000:
        k = int(rng.integers(1, 7))
        n = int(rng.integers(k, 12))
        g = rng.integers(0, 2, (k, n))
        if O.gf2_rank(g) < k:
            continue
        tested += 1
        piv, _ = O.mrb_row_pivot(g)
        assert sorted(piv) == O.mrb_greedy(g), g


def _llrs(rng, gm, ebno_db, num):
    k, n = gm.shape
    u = rng.integers(0, 2, (num, k))
    c = O.encode(u, gm)
    no = 1 / (10 ** (ebno_db / 10) * k / n)
    y = (2.0 * c - 1) + rng.normal(size=c.shape) * np.sqrt(no / 2)
    return (4 * y / no).astype(np.float32)


@pytest.mark.parametrize("pcm_id,t", [(0, 1), (0, 2), (0, 4), (1, 1), (1, 2)])
def test_literal_and_discrepancy_osd_agree(pcm_id, t):
    pcm, k, n, _ = load_parity_check_examples(pcm_id)
    gm = pcm2gm(pcm)
    rng = np.random.default_rng(3)
    for l in _llrs(rng, gm, 1.0, 40):
        a, d, d2 = O.osd_discrepancy(l, gm, t, return_gap=True)
        if d2 - d <= 1e-5 * np.abs(l).sum():
            continue
        assert np.array_equal(a, O.osd_literal(l, gm, t))


def test_discrepancy_form_stays_finite_where_softplus_overflows():
    gm = pcm2gm(load_parity_check_examples(0)[0])
    l = np.array([95, -95, 99, 98, -97, 96, 94], np.float32)   # not a codeword's signs; every flip costs > 88.7
    c = O.osd_discrepancy(l, gm, 4)
    assert np.array_equal(c, O.ml_bruteforce(l, gm))


def test_osd_order_k_is_ml():
    rng = np.random.default_rng(4)
    for _ in range(30):
        k = int(rng.integers(1, 9))
        n = int(rng.integers(k + 1, 16))
        gm = _full_rank(rng, k, n)
        for l in _llrs(rng, gm, 0.0, 10):
            c, d, d2 = O.ml_bruteforce(l, gm, return_gap=True)
            if d2 - d <= 1e-5 * np.abs(l).sum():
                continue
            assert np.array_equal(O.osd_discrepancy(l, gm, k), c)
            assert np.array_equal(O.osd_discrepancy(l, gm, k + 3), c)


def test_pcm2gm_equals_reference_golden():
    """Example code 3's generator and column swaps as the reference's own make_systematic / pcm2gm produced them
    (tests/golden/make_linear_golden.py)."""
    with np.load(os.path.join(GOLDEN, "linear_golden.npz")) as d:
        gm = np.unpackbits(d["gm3"], axis=-1)[:, :int(d["n3"])]
        swaps = d["swaps3"].tolist()
    pcm = load_parity_check_examples(3)[0]
    assert np.array_equal(pcm2gm(pcm), gm)
    assert make_systematic(pcm, is_pcm=True)[1] == swaps
    assert np.array_equal(O.pcm2gm(pcm), gm)
