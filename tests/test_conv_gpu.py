"""Convolutional codes on the GPU (csrc/conv.cu) against oracle/conv.py and the reference's goldens.

Encoder and Viterbi decoder: bit-identical to the oracle (the Viterbi decoder to its float32 path-metric arithmetic).
BCJR decoder: the goldens exactly; soft outputs within 2x (rms) / 4x (max) of the float32 evaluation's error against
float64 (parity.envelope), hard outputs equal float64's wherever |LLR| exceeds that error. Then the reference's unit
tests restated and two links of the coding tutorials."""
import itertools
import os

import numpy as np
import pytest
import torch

from oracle import conv as O
from oracle.parity import envelope

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "conv_golden.npz")
KEYS = ("57", "6474", "577", "5777")
# one code per state count 2 ... 256 (the last two beyond the reference's selector), plus rate 1/4
CODES = [("11", "10"), ("101", "111"), ("1101", "1011"), ("10011", "11011"), ("110101", "101111"),
         ("1011011", "1111001"), ("11100101", "10011111"), ("110101001", "101110111"),
         ("10101", "11011", "11111"), ("1011011", "1111001", "1100101", "1110111")]


@pytest.fixture(autouse=True)
def _restore_precision_warnings():
    """PrecisionWarning is issued once per class and process; the double-precision cases restore the record."""
    from sionna_b200.phy import block
    saved = set(block._warned_double)
    yield
    block._warned_double.clear()
    block._warned_double.update(saved)


def _conv():
    from sionna_b200.phy.fec import conv
    return conv


def golden(key):
    with np.load(GOLDEN) as d:
        k, n = d[f"shape_{key}"]
        return (tuple(str(p) for p in d[f"poly_{key}"]), np.unpackbits(d[f"u_{key}"], axis=1)[:, :k],
                np.unpackbits(d[f"x_{key}"], axis=1)[:, :n], d[f"y_{key}"],
                np.unpackbits(d[f"uhat_{key}"], axis=1)[:, :k])


def gpu(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def host(t):
    return t.cpu().numpy()


def noisy_llr(x, snr_db, rng):
    no = 10 ** (-snr_db / 10)
    return (2 / no * ((2 * x - 1) + rng.normal(size=x.shape) * np.sqrt(no))).astype(np.float32)


# ---- goldens ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", KEYS)
def test_goldens(cuda_device, key):
    conv = _conv()
    g, u, x, y, uhat = golden(key)
    assert np.array_equal(host(conv.ConvEncoder(gen_poly=g)(gpu(u))), x)
    no = 1.0 / (10 ** (4.95 / 10) * 2)
    assert np.array_equal(host(conv.ViterbiDecoder(gen_poly=g, method="soft_llr")(gpu(2 * y / no))), uhat)
    for alg in ("map", "log", "maxlog"):
        assert np.array_equal(host(conv.BCJRDecoder(gen_poly=g, algorithm=alg)(gpu(0.5 * (y + 1)))), uhat)
    if key in ("57", "577"):
        enc = conv.ConvEncoder(rate={"57": 1 / 2, "577": 1 / 3}[key], constraint_length=3)
        assert np.array_equal(host(enc(gpu(u))), x)


# ---- encoder ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", CODES)
@pytest.mark.parametrize("rsc,terminate", list(itertools.product((False, True), (False, True))))
def test_encoder(cuda_device, g, rsc, terminate):
    conv = _conv()
    rng = np.random.default_rng(len(g[0]))
    for k, b in ((1, 3), (37, 5), (10000, 2)):
        u = rng.integers(0, 2, (b, k))
        x = host(conv.ConvEncoder(gen_poly=g, rsc=rsc, terminate=terminate)(gpu(u)))
        assert np.array_equal(x, O.encode(u, g, rsc, terminate)), (k, b)


# ---- Viterbi ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", CODES)
@pytest.mark.parametrize("rsc,terminate", list(itertools.product((False, True), (False, True))))
def test_viterbi_bit_exact(cuda_device, g, rsc, terminate):
    """Soft and hard methods, both outputs, random LLRs at several SNRs and batch tails of the packed warps."""
    conv = _conv()
    rng = np.random.default_rng(7 * len(g[0]) + len(g))
    k, b = 97, 67
    u = rng.integers(0, 2, (b, k))
    x = O.encode(u, g, rsc, terminate)
    llr = np.concatenate([noisy_llr(x[i::4], snr, rng) for i, snr in enumerate((-3.0, 0.0, 3.0, 8.0))])
    for method in ("soft_llr", "hard"):
        for info in (True, False):
            dec = conv.ViterbiDecoder(gen_poly=g, rsc=rsc, terminate=terminate, method=method, return_info_bits=info)
            got = host(dec(gpu(llr)))
            ref = O.viterbi(llr, g, rsc, terminate, method, info, dtype=np.float32)
            assert np.array_equal(got, ref), (method, info, np.sum(got != ref))


def test_viterbi_hard_ties(cuda_device):
    """Integer hard metrics tie often: the first predecessor must win, as in the oracle (and tf.argmin)."""
    conv = _conv()
    rng = np.random.default_rng(11)
    for g in CODES[:5]:
        y = rng.integers(-3, 4, (200, 60 * len(g))).astype(np.float32) + rng.choice([0.0, 0.5, 0.49], (200, 60 * len(g)))
        got = host(conv.ViterbiDecoder(gen_poly=g, method="hard")(gpu(y)))
        assert np.array_equal(got, O.viterbi(y, g, method="hard", dtype=np.float32))


@pytest.mark.parametrize("g", [CODES[1], CODES[3], CODES[6], CODES[7]])
def test_viterbi_long_codeword(cuda_device, g):
    """k = 5000: the decisions no longer fit in shared memory and go through the workspace."""
    conv = _conv()
    from sionna_b200._lib import lib
    rng = np.random.default_rng(5)
    u = rng.integers(0, 2, (9, 5000))
    x = O.encode(u, g, False, True)
    ns = 2 ** (len(g[0]) - 1)
    if ns >= 32:
        assert lib().sb_viterbi_workspace_bytes(9, x.shape[1] // len(g), ns) > 0
    llr = noisy_llr(x, 1.0, rng)
    for info in (True, False):
        got = host(conv.ViterbiDecoder(gen_poly=g, terminate=True, return_info_bits=info)(gpu(llr)))
        assert np.array_equal(got, O.viterbi(llr, g, False, True, "soft_llr", info, dtype=np.float32))


# ---- BCJR -------------------------------------------------------------------------------------------------------------
def _bcjr_case(g, rsc, terminate, alg, prior, rng, k=83, b=48, snr=(-2.0, 1.0, 4.0)):
    conv = _conv()
    u = rng.integers(0, 2, (b, k))
    x = O.encode(u, g, rsc, terminate)
    llr = np.concatenate([noisy_llr(x[i::len(snr)], s, rng) for i, s in enumerate(snr)])
    T = x.shape[1] // len(g)
    la = (rng.normal(size=(b, T)) * 2).astype(np.float32) if prior else None
    dec = conv.BCJRDecoder(gen_poly=g, rsc=rsc, terminate=terminate, algorithm=alg, hard_out=False)
    got = host(dec(gpu(llr), llr_a=None if la is None else gpu(la)))
    hard = host(conv.BCJRDecoder(gen_poly=g, rsc=rsc, terminate=terminate, algorithm=alg, hard_out=True)(
        gpu(llr), llr_a=None if la is None else gpu(la)))
    ref = O.bcjr(llr.astype(np.float64), g, rsc, terminate, "log" if alg == "map" else alg,
                 None if la is None else la.astype(np.float64))[:, :k]
    f32 = O.bcjr(llr, g, rsc, terminate, alg, la, dtype=np.float32)[:, :k]
    return got, hard, ref, f32


def _check_bcjr(what, got, hard, ref, f32):
    assert np.all(np.isfinite(got))
    bad = envelope(what, got, f32, ref, (2.0, 4.0), floor=(1e-6, 1e-5), axis=None)
    assert not bad, bad
    err = np.abs(f32 - ref)
    sure = np.abs(ref) > 4 * max(float(err.max()), 1e-5 * float(np.sqrt(np.mean(ref ** 2))))
    assert np.array_equal(hard[sure], (ref[sure] > 0).astype(np.float32)), what


@pytest.mark.parametrize("alg", ["map", "log", "maxlog"])
@pytest.mark.parametrize("g", [CODES[1], CODES[3], CODES[5], CODES[6], CODES[7], CODES[9]])
@pytest.mark.parametrize("rsc,terminate,prior", [(False, False, False), (False, True, True), (True, True, False),
                                                 (True, False, True)])
def test_bcjr_envelope(cuda_device, alg, g, rsc, terminate, prior):
    rng = np.random.default_rng(len(g[0]) * 13 + len(g))
    got, hard, ref, f32 = _bcjr_case(g, rsc, terminate, alg, prior, rng)
    _check_bcjr(f"{alg} {g} rsc={rsc} term={terminate} prior={prior}", got, hard, ref, f32)


@pytest.mark.parametrize("alg", ["map", "maxlog"])
@pytest.mark.parametrize("g", [CODES[3], CODES[6]])
def test_bcjr_long_codeword(cuda_device, alg, g):
    """k = 3000: alpha goes through the workspace (K = 8) or fills shared memory (K = 5)."""
    rng = np.random.default_rng(17)
    got, hard, ref, f32 = _bcjr_case(g, False, True, alg, True, rng, k=3000, b=6, snr=(0.0, 2.0))
    _check_bcjr(f"long {alg} {g}", got, hard, ref, f32)


def test_bcjr_full_length_output(cuda_device):
    """sb_bcjr_decode returns the APP LLRs of all num_syms steps when asked (the turbo decoder's use)."""
    from sionna_b200._lib import lib, check, ptr, current_stream
    conv = _conv()
    g = CODES[3]
    rng = np.random.default_rng(2)
    got, _, ref, f32 = _bcjr_case(g, False, True, "log", True, rng, k=50, b=8)
    tr = conv.Trellis(g, rsc=False)
    tabs = [np.ascontiguousarray(t, np.int32) for t in (tr.from_nodes, tr.op_by_tonode, tr.ip_by_tonode)]
    u = rng.integers(0, 2, (8, 50))
    x = O.encode(u, g, False, True)
    llr = noisy_llr(x, 1.0, rng)
    la = (rng.normal(size=(8, 54))).astype(np.float32)
    y, a = gpu(llr), gpu(la)
    out = torch.empty((8, 54), device="cuda")
    check(lib().sb_bcjr_decode(ptr(y), ptr(a), ptr(out), 8, 54, 54, 1, 1, 0, *[ptr(t) for t in tabs], 16, 2, None, 0,
                               current_stream()), "sb_bcjr_decode")
    ref = O.bcjr(llr.astype(np.float64), g, False, True, "log", la.astype(np.float64))
    f32 = O.bcjr(llr, g, False, True, "log", la, dtype=np.float32)
    assert not envelope("full length", host(out), f32, ref, (2.0, 4.0), floor=(1e-6, 1e-5), axis=None)


@pytest.mark.parametrize("hard_out", [True, False])
def test_bcjr_numerical_stability(cuda_device, hard_out):
    """The reference's test_numerical_stab (|LLR| ~ 1e4 and all-zero input), extended to soft outputs: no NaN, no inf."""
    conv = _conv()
    from sionna_b200.phy.fec.utils import GaussianPriorSource
    src = GaussianPriorSource()
    for k, rate, alg in itertools.product((22, 55), (1 / 2, 1 / 3), ("map", "log", "maxlog")):
        n = int(k / rate)
        dec = conv.BCJRDecoder(rate=rate, constraint_length=5, algorithm=alg, hard_out=hard_out)
        for c in (src([10, n], 0.0001), torch.zeros((10, n), device="cuda")):
            u = host(dec(c))
            assert np.all(np.isfinite(u)), (k, rate, alg)
        vit = conv.ViterbiDecoder(rate=rate, constraint_length=5)
        assert np.all(np.isfinite(host(vit(src([10, n], 0.0001)))))


# ---- the reference's unit tests ---------------------------------------------------------------------------------------
def test_output_dim(cuda_device):
    conv = _conv()
    for k, rate in itertools.product((10, 22, 40), (1 / 2, 1 / 3)):
        for make in (lambda **kw: conv.ViterbiDecoder(**kw), lambda **kw: conv.BCJRDecoder(**kw)):
            for dec in (make(rate=rate, constraint_length=5), make(rate=rate, constraint_length=3, rsc=True),
                        make(rate=rate, constraint_length=4, terminate=True)):
                n = int(k / rate) + (int(3 / rate) if dec.terminate else 0)
                u = host(dec(-10.0 * torch.ones((10, n), device="cuda")))
                assert u.shape == (10, k) and not u.any()
    enc = conv.ConvEncoder(rate=1 / 2, constraint_length=5, terminate=True)
    assert tuple(enc(torch.zeros((3, 4, 20), device="cuda")).shape) == (3, 4, 48)
    assert enc.k == 20 and enc.n == 48 and abs(enc.coderate - 20 / 48) < 1e-12


def test_errors_and_notes(cuda_device, capsys):
    conv = _conv()
    dec = conv.ViterbiDecoder(rate=1 / 2, constraint_length=3)
    assert dec.k is None and dec.n is None
    assert "cannot be computed before the first call()" in capsys.readouterr().out
    with pytest.raises(ValueError):
        dec(torch.zeros((2, 11), device="cuda"))
    with pytest.raises(ValueError):
        conv.BCJRDecoder(rate=1 / 3, constraint_length=5)(torch.zeros((2, 10), device="cuda"))
    with pytest.raises(ValueError):
        conv.BCJRDecoder(algorithm="exact")
    with pytest.raises(ValueError):
        conv.ViterbiDecoder(method="soft")
    with pytest.raises(ValueError):
        conv.ConvEncoder(constraint_length=9)
    with pytest.raises(ValueError):
        conv.ConvEncoder(gen_poly=("101", "11"))
    with pytest.raises(TypeError):
        conv.ConvEncoder(gen_poly=(101, 111))
    from sionna_b200._lib import SbUnsupportedError
    with pytest.raises(SbUnsupportedError, match="512 states"):
        conv.ViterbiDecoder(gen_poly=("1101011011", "1011101111"))(torch.zeros((1, 40), device="cuda"))


def test_multi_dimensional_and_batch(cuda_device):
    conv = _conv()
    rng = np.random.default_rng(3)
    enc = conv.ConvEncoder(rate=1 / 2, constraint_length=5, terminate=True)
    u = rng.integers(0, 2, (6, 5, 40)).astype(np.float32)
    x = enc(gpu(u))
    assert np.array_equal(host(x).reshape(30, -1), host(enc(gpu(u.reshape(30, 40)))))
    llr = gpu(noisy_llr(host(x), 2.0, rng))
    for dec in (conv.ViterbiDecoder(encoder=enc), conv.BCJRDecoder(encoder=enc, hard_out=False)):
        out = host(dec(llr))
        assert out.shape == (6, 5, 40)
        assert np.array_equal(out.reshape(30, 40), host(dec(llr.reshape(30, -1))))
        one = host(dec(llr[2:3, 1:2]))
        assert np.array_equal(one[0, 0], out[2, 1])
    # k follows the input on every call
    dec = conv.ViterbiDecoder(encoder=enc)
    assert host(dec(torch.zeros((2, 2 * (17 + 4)), device="cuda"))).shape == (2, 17) and dec.k == 17


@pytest.mark.parametrize("rate,K", [(1 / 2, 3), (1 / 2, 8), (1 / 3, 3), (1 / 3, 8)])
def test_init_and_identity(cuda_device, rate, K):
    """Decoders built from encoder= equal those built from gen_poly; noise-free and mildly noisy words are recovered."""
    conv = _conv()
    rng = np.random.default_rng(K)
    for rsc in (False, True):
        enc = conv.ConvEncoder(rate=rate, constraint_length=K, rsc=rsc)
        u = gpu(rng.integers(0, 2, (5, 40)))
        cw = enc(u)
        for syms in (20.0 * (2 * cw - 1), 6.0 * (2 * cw - 1) + gpu(rng.normal(size=tuple(cw.shape)))):
            for alg in ("map", "log", "maxlog"):
                a = conv.BCJRDecoder(encoder=enc, algorithm=alg)(syms)
                b = conv.BCJRDecoder(gen_poly=enc.gen_poly, rsc=rsc, algorithm=alg)(syms)
                assert torch.equal(a, b) and torch.equal(a, u)
            a = conv.ViterbiDecoder(encoder=enc)(syms)
            assert torch.equal(a, conv.ViterbiDecoder(gen_poly=enc.gen_poly, rsc=rsc)(syms)) and torch.equal(a, u)


def test_dtype_and_double_precision(cuda_device):
    conv = _conv()
    from sionna_b200.phy.block import PrecisionWarning
    enc = conv.ConvEncoder(rate=1 / 2, constraint_length=5, precision="double")
    u = torch.randint(0, 2, (4, 30), device="cuda").to(torch.float64)
    with pytest.warns(PrecisionWarning):
        x = enc(u)
    assert x.dtype == torch.float64
    llr = 8.0 * (2 * x - 1)
    with pytest.warns(PrecisionWarning):
        out = conv.ViterbiDecoder(encoder=enc, precision="double")(llr)
    assert out.dtype == torch.float64 and torch.equal(out, u)
    with pytest.warns(PrecisionWarning):
        out = conv.BCJRDecoder(encoder=enc, precision="double", hard_out=False)(llr)
    assert out.dtype == torch.float64 and torch.equal((out > 0).to(torch.float64), u)
    single = conv.ViterbiDecoder(encoder=enc)(llr.to(torch.float32))
    assert single.dtype == torch.float32


# ---- links of the coding tutorials ------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,k,batch,ebno", [(8, 64, 2000, 2.0), (5, 64, 2000, 3.0)])
def test_link(cuda_device, K, k, batch, ebno):
    """QPSK + AWGN + Demapper, decoded on the GPU and by the oracle from the same LLRs: identical bit errors."""
    conv = _conv()
    from sionna_b200.phy.mapping import Mapper, Demapper, BinarySource
    from sionna_b200.phy.channel import AWGN
    from sionna_b200.phy.utils import ebnodb2no, sim_ber
    enc = conv.ConvEncoder(rate=1 / 2, constraint_length=K)
    vit = conv.ViterbiDecoder(gen_poly=enc.gen_poly, method="soft_llr")
    bcjr = conv.BCJRDecoder(encoder=enc, algorithm="maxlog")
    mapper, demapper, awgn, src = Mapper("qam", 2), Demapper("app", "qam", 2), AWGN(), BinarySource()
    seen = []

    def run(batch_size, ebno_db):
        no = ebnodb2no(ebno_db, 2, 0.5)
        u = src([batch_size, k])
        llr = demapper(awgn(mapper(enc(u)), no), no)
        u_hat = vit(llr)
        seen.append((host(u), host(llr), host(u_hat), host(bcjr(llr))))
        return u, u_hat

    ber, _ = sim_ber(run, [ebno], batch, max_mc_iter=2, early_stop=False, verbose=False)
    errs = 0
    for u, llr, v, b in seen:
        g = enc.gen_poly
        assert np.array_equal(v, O.viterbi(llr, g, dtype=np.float32))
        ref = O.bcjr(llr, g, algorithm="maxlog", dtype=np.float32)
        assert np.mean(b != (ref > 0)) < 1e-3
        errs += int(np.sum(v != u))
    assert abs(float(ber[0]) - errs / (len(seen) * batch * k)) < 1e-9
    assert 0 < errs / (len(seen) * batch * k) < 0.05
