"""Turbo codes on the GPU against oracle/turbo.py, the composed component-decoder loop and the reference's goldens.

Encoder (sb_gather_rows + sb_conv_encode): bit-identical to the oracle. Decoder (sb_turbo_decode): bit-identical to
the reference's loop run on this library's BCJRDecoder with torch glue (same recursion code, same fp32 operations);
within 2x (rms) / 4x (max) of the float32 oracle's error against float64 (parity.envelope), hard outputs equal
float64's wherever |LLR| exceeds that error. Then the reference's unit tests restated and its BER test."""
import itertools
import os

import numpy as np
import pytest
import torch

from oracle import turbo as O
from oracle.parity import envelope

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "turbo_golden.npz")
POLYS = {3: ("111", "101"), 4: ("1011", "1101"), 5: ("10011", "11011"), 6: ("111101", "101011"),
         8: ("11100101", "10011111"), 9: ("110101001", "101110111")}
ALL_POLYS = {2: ("11", "10"), 7: ("1011011", "1111001"), **POLYS}      # ns = 2 ... 256


@pytest.fixture(autouse=True)
def _restore_precision_warnings():
    """PrecisionWarning is issued once per class and process; the double-precision cases restore the record."""
    from sionna_b200.phy import block
    saved = set(block._warned_double)
    yield
    block._warned_double.clear()
    block._warned_double.update(saved)


def _turbo():
    from sionna_b200.phy.fec import turbo
    return turbo


def gpu(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def host(t):
    return t.cpu().numpy()


def golden(k):
    with np.load(GOLDEN) as d:
        unpack = lambda name: np.unpackbits(d[f"{name}_{k}"], axis=-1)[:, :int(d[f"len_{name}_{k}"])]
        return unpack("u"), unpack("x"), d[f"y_{k}"], unpack("uhat")


def noisy(x, snr_db, rng):
    no = 10 ** (-snr_db / 10)
    return (2 / no * ((2 * x - 1) + rng.normal(size=x.shape) * np.sqrt(no))).astype(np.float32)


def perm_of(enc, k):
    from sionna_b200.phy.fec.turbo.encoding import interleaver_perm
    return interleaver_perm(enc.internal_interleaver, k)


def composed(dec, y):
    """The reference's decoding loop (decoding.py:357-435) on BCJRDecoder with torch glue, from the same component
    codewords the fused decoder reads."""
    from sionna_b200.phy.fec.conv import BCJRDecoder
    from sionna_b200.phy.fec.turbo.encoding import gather
    if dec._demux is None:
        dec._prepare()
    k, T = dec._k, dec._convenc_numsyms
    yc = gather(y.reshape(-1, dec._n).contiguous(), dec._demux, 1, 4 * T, dec._n).reshape(-1, 2, 2 * T)
    y1, y2 = yc[:, 0].contiguous(), yc[:, 1].contiguous()
    perm = torch.from_numpy(perm_of_dec(dec, k)).cuda()
    pinv = torch.argsort(perm)
    bcjr = BCJRDecoder(gen_poly=dec.gen_poly, rsc=True, terminate=dec._terminate, hard_out=False,
                       algorithm=dec._algorithm)
    B, tz = y1.shape[0], T - k
    lch, lch2 = y1[:, 0:2 * k:2], y2[:, 0:2 * k:2]
    zeros = torch.zeros((B, tz), device=y.device)
    l1e = torch.zeros((B, T), device=y.device)
    l2i = torch.zeros((B, k), device=y.device)
    for _ in range(dec.num_iter):
        l1i = bcjr(y1, llr_a=l1e)[:, :k]
        ex = l1i - lch - l1e[:, :k]
        l2e = torch.cat([ex[:, perm].clamp(-20, 20), zeros], 1)
        l2i = bcjr(y2, llr_a=l2e)[:, :k]
        ex = l2i - l2e[:, :k] - lch2
        l1e = torch.cat([ex[:, pinv].clamp(-20, 20), zeros], 1)
    return l2i[:, pinv]


def perm_of_dec(dec, k):
    from sionna_b200.phy.fec.turbo.encoding import interleaver_perm
    return interleaver_perm(dec.internal_interleaver, k)


# ---- goldens ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", (40, 112, 168, 432))
def test_goldens(cuda_device, k):
    turbo = _turbo()
    u, x, y, uhat = golden(k)
    enc = turbo.TurboEncoder(rate=1 / 3, terminate=True, constraint_length=4)
    assert np.array_equal(host(enc(gpu(u))), x)
    if k == 432:
        return
    dec = turbo.TurboDecoder(enc, num_iter=10)
    no = 1 / ((1 / 3) * 10 ** 0)
    assert np.array_equal(host(dec(gpu(-4.0 * y / no))), uhat)


# ---- encoder ----------------------------------------------------------------------------------------------------------
ENC_CASES = [(K, r, t, il, k) for K, r, t, il, k in itertools.product((3, 4, 5, 6, 8), (1 / 3, 1 / 2), (False, True),
                                                                      ("3GPP", "random"), (40, 41, 1000, 6144))]
ENC_CASES += [(K, r, t, "random", 10000) for K, r, t in itertools.product((4, 8), (1 / 3, 1 / 2), (False, True))]


@pytest.mark.parametrize("K,rate,terminate,il,k", ENC_CASES)
def test_encoder_vs_oracle(cuda_device, K, rate, terminate, il, k):
    turbo = _turbo()
    enc = turbo.TurboEncoder(gen_poly=POLYS[K], rate=rate, terminate=terminate, interleaver_type=il)
    u = np.random.default_rng(k + K).integers(0, 2, (3, k))
    x = host(enc(gpu(u)))
    assert np.array_equal(x, O.encode(u, POLYS[K], perm_of(enc, k), rate, terminate))
    if terminate:
        assert abs(enc.coderate - k / x.shape[-1]) < 1e-6 or rate == 1 / 2


# ---- decoder: bit-identical to the composed loop ----------------------------------------------------------------------
DEC_CASES = [(alg, K, it, rate, term) for (alg, K), it, rate, term in
             zip(itertools.product(("map", "log", "maxlog"), (2, 3, 4, 5, 6, 7, 8, 9)),
                 itertools.cycle((1, 2, 3, 4, 5, 6, 6)), itertools.cycle((1 / 3, 1 / 2, 1 / 3)),
                 itertools.cycle((True, False)))]


@pytest.mark.parametrize("alg,K,num_iter,rate,terminate", DEC_CASES)
def test_decoder_equals_composed(cuda_device, alg, K, num_iter, rate, terminate):
    turbo = _turbo()
    k = 96 if K < 9 else 40
    enc = turbo.TurboEncoder(gen_poly=ALL_POLYS[K], rate=rate, terminate=terminate)
    dec = turbo.TurboDecoder(enc, num_iter=num_iter, hard_out=False, algorithm=alg)
    rng = np.random.default_rng(K * 7 + num_iter)
    u = rng.integers(0, 2, (70, k))
    y = gpu(noisy(host(enc(gpu(u))), 0.5, rng))
    got = dec(y)
    ref = composed(dec, y)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("k,batch", [(40, 300), (6144, 3)])
def test_storage_paths(cuda_device, sb_lib, k, batch):
    """k = 40 keeps alpha and the extrinsic LLRs on chip, k = 6144 both in the workspace; both equal the composed
    loop and the float32 oracle's decisions."""
    turbo = _turbo()
    ws = sb_lib.sb_turbo_workspace_bytes(batch, k, 1, 8)
    assert (ws == 0) == (k == 40)
    enc = turbo.TurboEncoder(constraint_length=4, terminate=True)
    dec = turbo.TurboDecoder(enc, num_iter=3, hard_out=False, algorithm="maxlog")
    rng = np.random.default_rng(k)
    u = rng.integers(0, 2, (batch, k))
    y = noisy(host(enc(gpu(u))), 0.0, rng)
    got = dec(gpu(y))
    assert torch.equal(got, composed(dec, gpu(y)))
    ref = O.decode(y, enc.gen_poly, perm_of(enc, k), 1 / 3, True, 3, "maxlog", np.float32)
    assert np.mean((host(got) > 0) == (ref > 0)) > 0.999


# ---- decoder: the float32 envelope ------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg,rate,terminate", [("map", 1 / 3, True), ("log", 1 / 2, False), ("maxlog", 1 / 3, False),
                                                ("map", 1 / 2, True)])
def test_decoder_envelope(cuda_device, alg, rate, terminate):
    turbo = _turbo()
    k, it = 112, 4
    enc = turbo.TurboEncoder(constraint_length=4, rate=rate, terminate=terminate)
    dec = turbo.TurboDecoder(enc, num_iter=it, hard_out=False, algorithm=alg)
    rng = np.random.default_rng(3)
    u = rng.integers(0, 2, (40, k))
    y = noisy(host(enc(gpu(u))), 0.5, rng)
    got = host(dec(gpu(y))).astype(np.float64)
    perm = perm_of(enc, k)
    ref = O.decode(y.astype(np.float64), enc.gen_poly, perm, rate, terminate, it, alg, np.float64)
    f32 = O.decode(y, enc.gen_poly, perm, rate, terminate, it, alg, np.float32).astype(np.float64)
    assert not envelope(f"turbo {alg} rate {rate:.2f} term {terminate}", got, f32, ref, (2.0, 4.0), floor=(1e-7, 1e-6),
                        axis=None)
    err = np.abs(f32 - ref).max() * 4
    sure = np.abs(ref) > err
    assert np.array_equal((got > 0)[sure], (ref > 0)[sure])


# ---- the reference's unit tests ---------------------------------------------------------------------------------------
def test_output_dim_num_stab(cuda_device):
    """decoding.py test_output_dim_num_stab: shapes, and zeros -> hard 0 / finite soft values."""
    turbo = _turbo()
    for rate, k, term, il in itertools.product((1 / 2, 1 / 3), (40, 100, 1024), (True, False), ("3GPP", "random")):
        enc = turbo.TurboEncoder(constraint_length=4, rate=rate, terminate=term, interleaver_type=il)
        dec = turbo.TurboDecoder(enc, num_iter=2)
        c = enc(gpu(np.zeros((10, k))))
        u_hat = dec(gpu(-10.0 * np.ones(host(c).shape)))
        assert tuple(u_hat.shape) == (10, k) and torch.equal(u_hat, torch.zeros_like(u_hat))
        soft = turbo.TurboDecoder(enc, num_iter=2, hard_out=False)(gpu(np.zeros(host(c).shape)))
        assert torch.isfinite(soft).all()


@pytest.mark.parametrize("alg,terminate", list(itertools.product(("map", "log", "maxlog"), (False, True))))
def test_identity(cuda_device, alg, terminate):
    turbo = _turbo()
    for K, rate in itertools.product((3, 4, 5, 6), (1 / 3, 1 / 2)):
        enc = turbo.TurboEncoder(constraint_length=K, rate=rate, terminate=terminate)
        dec = turbo.TurboDecoder(enc, num_iter=2, algorithm=alg)
        u = np.random.default_rng(K).integers(0, 2, (10, 98))
        c = host(enc(gpu(u)))
        assert np.array_equal(host(dec(gpu(20.0 * (2 * c - 1)))), u)


def test_multi_dimensional_batch_and_dynamic_shapes(cuda_device):
    turbo = _turbo()
    enc = turbo.TurboEncoder(constraint_length=4, terminate=True)
    dec = turbo.TurboDecoder(enc, num_iter=3, hard_out=False)
    rng = np.random.default_rng(0)
    u = rng.integers(0, 2, (2, 3, 4, 64))
    c = enc(gpu(u))
    assert tuple(c.shape) == (2, 3, 4, 3 * 64 + 12)
    y = gpu(noisy(host(c), 1.0, rng))
    out = dec(y)
    flat = dec(y.reshape(-1, y.shape[-1]))
    assert torch.equal(out.reshape(-1, 64), flat)
    for i in range(3):                                     # each example decodes alone as in the batch
        assert torch.equal(dec(y[0, i]), out[0, i])
    for k in (40, 200, 65):                               # new lengths rebuild both blocks
        uk = rng.integers(0, 2, (5, k))
        assert np.array_equal(host(turbo.TurboDecoder(enc)(gpu(20.0 * (2 * host(enc(gpu(uk))) - 1)))), uk)
        assert dec.k is not None


def test_dtype_flexible(cuda_device):
    from sionna_b200.phy.block import PrecisionWarning
    turbo = _turbo()
    enc = turbo.TurboEncoder(constraint_length=4, precision="double")
    u = np.random.default_rng(0).integers(0, 2, (5, 40))
    with pytest.warns(PrecisionWarning):
        c = enc(torch.from_numpy(u.astype(np.float64)).cuda())
    assert c.dtype == torch.float64
    dec = turbo.TurboDecoder(enc, precision="double", hard_out=False)
    with pytest.warns(PrecisionWarning):
        out = dec(20.0 * (2 * c - 1))
    assert out.dtype == torch.float64
    assert np.array_equal(host(out) > 0, u == 1)
    enc32 = turbo.TurboEncoder(constraint_length=4)
    assert host(enc32(torch.from_numpy(u.astype(np.int32)).cuda())).dtype == np.float32


def test_num_iter_zero(cuda_device):
    turbo = _turbo()
    enc = turbo.TurboEncoder(constraint_length=4)
    c = enc(gpu(np.ones((4, 40))))
    for hard in (True, False):
        out = turbo.TurboDecoder(enc, num_iter=0, hard_out=hard)(20.0 * (2 * c - 1))
        assert torch.equal(out, torch.zeros_like(out))


def test_encoder_output_dim_and_invalid_inputs(cuda_device):
    turbo = _turbo()
    for rate, term, K, k in itertools.product((1 / 2, 1 / 3), (False, True), (3, 4, 5, 6), (40, 123)):
        enc = turbo.TurboEncoder(constraint_length=K, rate=rate, terminate=term)
        c = host(enc(gpu(np.zeros((3, k)))))
        mu = K - 1
        assert c.shape[-1] == int(k / rate) + (int(np.ceil(4 * mu / 3)) * (2 if rate == 1 / 2 else 3) if term else 0)
        assert not c.any()
        if term:
            assert enc.coderate - k / c.shape[-1] < 1e-6
    for r in (0.2, 0.45, 0.01):
        with pytest.raises(ValueError):
            turbo.TurboEncoder(rate=r, constraint_length=4)
    for K in (2, 7, 8):
        with pytest.raises(ValueError):
            turbo.TurboEncoder(rate=1 / 3, constraint_length=K)
    with pytest.raises(ValueError):
        turbo.TurboEncoder(constraint_length=4)(gpu(np.zeros((1, 6145))))
    with pytest.raises(TypeError):
        turbo.TurboEncoder(constraint_length=4, terminate=1)
    with pytest.raises(ValueError):
        turbo.TurboEncoder(constraint_length=4, interleaver_type="x")


def test_polynomial_input(cuda_device):
    turbo = _turbo()
    u = np.random.default_rng(0).integers(0, 2, (4, 60))
    for g in (("101", "111"), ("1101", "1011"), ("10011", "11011")):
        enc = turbo.TurboEncoder(gen_poly=g, rate=1 / 3)
        assert np.array_equal(host(enc(gpu(u))), O.encode(u, g, perm_of(enc, 60)))
    with pytest.raises(TypeError):
        turbo.TurboEncoder(gen_poly=(101, 111))
    with pytest.raises(ValueError):
        turbo.TurboEncoder(gen_poly=("101", "1111"))
    with pytest.raises(ValueError):
        turbo.TurboEncoder(gen_poly=("101", "111", "111"))
    with pytest.raises(ValueError):
        turbo.TurboDecoder(gen_poly=("102", "111"))
    with pytest.raises(NotImplementedError):
        turbo.TurboDecoder(gen_poly=("101", "111", "111"))


def test_decoder_invalid_lengths(cuda_device):
    turbo = _turbo()
    dec = turbo.TurboDecoder(constraint_length=4, rate=1 / 2, terminate=True)
    with pytest.raises(ValueError):
        dec(gpu(np.zeros((2, 91))))
    dec3 = turbo.TurboDecoder(constraint_length=4, rate=1 / 3, terminate=True)
    with pytest.raises(ValueError):
        dec3(gpu(np.zeros((2, 3 * 40 + 13))))


def test_random_interleaver_shared_with_decoder(cuda_device):
    turbo = _turbo()
    enc = turbo.TurboEncoder(constraint_length=4, interleaver_type="random")
    dec = turbo.TurboDecoder(enc, num_iter=2)
    assert dec.internal_interleaver is enc.internal_interleaver
    u = np.random.default_rng(1).integers(0, 2, (8, 200))
    assert np.array_equal(host(dec(20.0 * (2 * enc(gpu(u)) - 1))), u)


@pytest.mark.parametrize("num_iter", (3, 6))
def test_ber_match(cuda_device, num_iter):
    """decoding.py test_ber_match: k = 512, rate 1/3, terminated, QPSK over AWGN, within the reference's bounds."""
    turbo = _turbo()
    from sionna_b200.phy.mapping import Mapper, Demapper, BinarySource
    from sionna_b200.phy.channel import AWGN
    from sionna_b200.phy.utils import ebnodb2no, sim_ber
    k, r = 512, 1 / 3
    enc = turbo.TurboEncoder(gen_poly=("1101", "1011"), rate=r, terminate=True)
    dec = turbo.TurboDecoder(enc, num_iter=num_iter)
    mapper, demapper, awgn, src = Mapper("qam", 2), Demapper("app", "qam", 2), AWGN(), BinarySource()

    def run(batch_size, ebno_db):
        no = ebnodb2no(ebno_db, 2, r)
        u = src([batch_size, k])
        return u, dec(demapper(awgn(mapper(enc(u)), no), no))

    snrs = [0, 0.5, 1, 1.5, 2]
    ub = {3: [10.0e-02, 6.0e-02, 5.5e-03, 2.5e-4, 5.0e-06], 6: [10.0e-02, 4.0e-02, 6.5e-04, 4.5e-5]}[num_iter]
    lb = {3: [5.0e-02, 1.0e-02, 1.0e-03, 5.0e-5, 8.0e-07], 6: [5.0e-02, 8.0e-03, 1.0e-04, 2.0e-6]}[num_iter]
    snrs = snrs[:len(ub)]
    ber, _ = sim_ber(run, snrs, 10000, max_mc_iter=20, num_target_bit_errors=500, early_stop=True, verbose=False)
    ber = np.asarray(torch.as_tensor(ber).cpu())
    print(f"turbo BER {num_iter} iterations: {ber}")
    assert np.all(ber <= np.array(ub)) and np.all(ber >= np.array(lb)), ber
