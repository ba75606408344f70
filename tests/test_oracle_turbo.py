"""The turbo oracle (oracle/turbo.py) and the QPP table on the CPU: the table has the structure of TS 36.212 Table
5.1.3-3, the oracle reproduces the reference's goldens (encoder exactly, the float64 decoder's decisions exactly, errors
included) and decodes noise-free codewords of every supported code."""
import itertools
import os

import numpy as np
import pytest

from oracle import conv as C
from oracle import turbo as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "turbo_golden.npz")
LTE = ("1011", "1101")
POLYS = {3: ("111", "101"), 4: ("1011", "1101"), 5: ("10011", "11011"), 6: ("111101", "101011")}


def qpp():
    from sionna_b200.phy.fec.interleaving import qpp_table
    return qpp_table()


def golden(k):
    with np.load(GOLDEN) as d:
        unpack = lambda name: np.unpackbits(d[f"{name}_{k}"], axis=-1)[:, :int(d[f"len_{name}_{k}"])]
        return unpack("u"), unpack("x"), d[f"y_{k}"], unpack("uhat")


def test_qpp_table_structure():
    tab = qpp()
    sizes = list(range(40, 513, 8)) + list(range(528, 1025, 16)) + list(range(1056, 2049, 32)) + \
        list(range(2112, 6145, 64))
    assert len(sizes) == 188 and sorted(tab) == sizes
    for K, (f1, f2) in tab.items():
        i = np.arange(K, dtype=np.int64)
        assert np.array_equal(np.sort((f1 * i + f2 * i * i) % K), i), K


def test_turbo3gpp_perm_shortened():
    from sionna_b200.phy.fec.interleaving import turbo3gpp_perm
    for k in (1, 41, 100, 1000, 6143):
        p = turbo3gpp_perm(k)
        assert np.array_equal(np.sort(p), np.arange(k))
        assert np.array_equal(p, O.qpp_perm(k, qpp()))
    with pytest.raises(ValueError):
        turbo3gpp_perm(6145)


@pytest.mark.parametrize("k", (40, 112, 168, 432))
def test_oracle_encoder_goldens(k):
    u, x, _, _ = golden(k)
    assert np.array_equal(O.encode(u, LTE, O.qpp_perm(k, qpp()), 1 / 3, True), x)


@pytest.mark.parametrize("k", (40, 112, 168))
def test_oracle_decoder_goldens(k):
    u, _, y, uhat = golden(k)
    no = 1 / ((1 / 3) * 10 ** 0)
    llr = (-4.0 * y / no).astype(np.float32).astype(np.float64)
    out = O.decode(llr, LTE, O.qpp_perm(k, qpp()), 1 / 3, True, num_iter=10, algorithm="map")
    assert np.array_equal((out > 0).astype(np.uint8), uhat)
    assert (uhat != u).sum() > 0                       # the goldens include decoding errors


@pytest.mark.parametrize("K,rate,terminate", list(itertools.product((3, 4, 5, 6), (1 / 3, 1 / 2), (False, True))))
def test_oracle_roundtrip(K, rate, terminate):
    rng = np.random.default_rng(K)
    k = 57
    perm = rng.permutation(k)
    u = rng.integers(0, 2, (4, k))
    x = O.encode(u, POLYS[K], perm, rate, terminate)
    out = O.decode(20.0 * (2 * x - 1), POLYS[K], perm, rate, terminate, num_iter=2, algorithm="maxlog")
    assert np.array_equal(out > 0, u == 1)


def test_layout_matches_oracle():
    """The encoder's and decoder's index tables (turbo_layout) equal the oracle's multiplexing and depuncturing."""
    from sionna_b200.phy.fec.turbo.encoding import turbo_layout
    rng = np.random.default_rng(1)
    for (K, rate, terminate), k in itertools.product(itertools.product((3, 4, 5, 6), (1 / 3, 1 / 2), (False, True)),
                                                     (40, 41)):
        mu, perm = K - 1, rng.permutation(k)
        T = k + (mu if terminate else 0)
        u = rng.integers(0, 2, (3, k))
        comp = np.concatenate([C.encode(u, POLYS[K], True, terminate), C.encode(u[:, perm], POLYS[K], True, terminate)], 1)
        mux, demux, rank = turbo_layout(k, mu, rate, terminate)
        ext = np.concatenate([comp, np.zeros((3, 1))], 1)            # index -1 reads 0
        assert np.array_equal(ext[:, mux], O.encode(u, POLYS[K], perm, rate, terminate))
        y = rng.normal(size=(3, len(mux)))
        demux[2 * T + 2 * np.arange(k)] = rank[3 * perm]
        y1, y2 = O.depuncture(y, k, mu, perm, rate, terminate)
        yext = np.concatenate([y, np.zeros((3, 1))], 1)
        assert np.array_equal(yext[:, demux], np.concatenate([y1, y2], 1))
