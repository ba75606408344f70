"""The convolutional-code oracle (oracle/conv.py) against the reference's goldens (tests/golden/conv_golden.npz),
noise-free round trips, the reference's trellis construction rules and the host-side Trellis / polynomial table."""
import itertools
import os

import numpy as np
import pytest

from oracle import conv as O
from sionna_b200.phy.fec.conv import Trellis, polynomial_selector
from sionna_b200.phy.fec.utils import int2bin, bin2int

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "conv_golden.npz")
KEYS = ("57", "6474", "577", "5777")


def golden(key):
    with np.load(GOLDEN) as d:
        k, n = d[f"shape_{key}"]
        return (tuple(str(p) for p in d[f"poly_{key}"]), np.unpackbits(d[f"u_{key}"], axis=1)[:, :k],
                np.unpackbits(d[f"x_{key}"], axis=1)[:, :n], d[f"y_{key}"],
                np.unpackbits(d[f"uhat_{key}"], axis=1)[:, :k])


def golden_no():
    return 1.0 / (10 ** (4.95 / 10) * 2)          # ebnodb2no(4.95, num_bits_per_symbol=2, coderate=1)


@pytest.mark.parametrize("key", KEYS)
def test_goldens(key):
    g, u, x, y, uhat = golden(key)
    assert np.array_equal(O.encode(u, g), x)
    assert np.array_equal(O.viterbi(np.float32(2 * y / golden_no()), g, dtype=np.float32), uhat)
    for alg in ("map", "log", "maxlog"):
        llr = np.float32(0.5 * (y + 1))
        assert np.array_equal(O.bcjr(llr, g, algorithm=alg, dtype=np.float32)[:, :u.shape[1]] > 0, uhat)
        assert np.array_equal(O.bcjr(llr.astype(np.float64), g, algorithm=alg)[:, :u.shape[1]] > 0, uhat)


def test_polynomial_table():
    with np.load(GOLDEN) as d:
        table = [str(s) for s in d["selector"]]
    for row in table:
        rate, K, polys = row.split(":")
        assert polynomial_selector({"1/2": 1 / 2, "1/3": 1 / 3}[rate], int(K)) == tuple(polys.split(","))
    with pytest.raises(ValueError):
        polynomial_selector(1 / 2, 9)
    with pytest.raises(ValueError):
        polynomial_selector(1 / 4, 5)
    with pytest.raises(TypeError):
        polynomial_selector(1 / 2, 5.0)


def test_int2bin_bin2int():
    assert int2bin(5, 4) == [0, 1, 0, 1] and int2bin(12, 3) == [1, 0, 0] and int2bin(3, 0) == []
    assert bin2int([1, 0, 1]) == 5 and bin2int([]) is None
    assert all(bin2int(int2bin(v, 9)) == v for v in range(512))


@pytest.mark.parametrize("rsc", [False, True])
@pytest.mark.parametrize("gen_poly", [("101", "111"), ("10011", "11011"), ("11100101", "10011111"),
                                      ("1011", "1101", "1111"), ("110101001", "101110111")])
def test_trellis_construction(gen_poly, rsc):
    """The host Trellis equals the oracle's, and both follow the reference's rules: the newest bit is the state's MSB,
    predecessors are listed input-major (input 0 pass first), an RSC code's new bit is input + feedback parity."""
    tr, ref = Trellis(gen_poly, rsc=rsc), O.trellis(gen_poly, rsc)
    for name in ("to_nodes", "from_nodes", "op_by_tonode", "ip_by_tonode", "op_by_fromnode"):
        assert np.array_equal(getattr(tr, name), ref[name]), name
    ns, K = tr.ns, len(gen_poly[0])
    for s in range(ns):
        assert sorted(tr.from_nodes[s]) == [(s << 1) & (ns - 1), ((s << 1) & (ns - 1)) | 1]
        for b in range(2):
            new = b ^ (bin(s & int(gen_poly[0][1:], 2)).count("1") & 1) if rsc else b
            assert tr.to_nodes[s, b] == (new << (K - 2)) | (s >> 1)
            assert tr.op_mat[s, tr.to_nodes[s, b]] == tr.op_by_fromnode[s, b]
    # the reference's loop order: the transitions with input 0 are listed before those with input 1
    for s in range(ns):
        assert tr.ip_by_tonode[s, 0] <= tr.ip_by_tonode[s, 1] or rsc


@pytest.mark.parametrize("rate,K,rsc,terminate", list(itertools.product((1 / 2, 1 / 3), range(3, 9), (False, True),
                                                                         (False, True))))
def test_noise_free_round_trip(rate, K, rsc, terminate):
    g = polynomial_selector(rate, K)
    rng = np.random.default_rng(K)
    u = rng.integers(0, 2, (4, 40))
    x = O.encode(u, g, rsc, terminate)
    assert x.shape == (4, (40 + (K - 1) * terminate) * len(g))
    llr = 10.0 * (2 * x - 1)
    for method, inp in (("soft_llr", llr), ("hard", x)):
        assert np.array_equal(O.viterbi(inp, g, rsc, terminate, method), u)
        assert np.array_equal(O.viterbi(inp, g, rsc, terminate, method, return_info_bits=False), x)
    for alg in ("map", "log", "maxlog"):
        for dt in (np.float64, np.float32):
            out = O.bcjr(llr, g, rsc, terminate, alg, dtype=dt)
            assert np.array_equal(out[:, :40] > 0, u == 1)
    if terminate:        # termination drives the register to the all-zero state
        tr = O.trellis(g, rsc)
        assert np.array_equal(O.viterbi(llr, g, rsc, False, return_info_bits=False), x)
        assert tr["to_nodes"].shape[0] == 2 ** (K - 1)


def test_map_equals_log_in_float64():
    """The reference's probability-domain "map" and the log-domain "log" are the same function."""
    g = ("10011", "11011")
    rng = np.random.default_rng(3)
    u = rng.integers(0, 2, (8, 60))
    x = O.encode(u, g, False, True)
    llr = 4.0 * (2 * x - 1) + rng.normal(size=x.shape) * 3
    la = rng.normal(size=(8, 64))
    a = O.bcjr(llr, g, False, True, "map", llr_a=la)
    b = O.bcjr(llr, g, False, True, "log", llr_a=la)
    assert np.allclose(a, b, rtol=1e-9, atol=1e-9)
