"""LinearEncoder (sb_gf2_encode) and OSDecoder (sb_osd_decode) on the GPU against oracle/linear_codes.py, brute-force
ML, the reference's unit tests and its ML BLER tables.

Decisions are compared where the float64 gap between the best and the runner-up candidate exceeds 1e-5 sum |llr|
(the kernel ranks in float32); elsewhere the kernel's word must be within that tolerance of the oracle's best."""
import numpy as np
import pytest
import torch

from oracle import linear_codes as O

pytestmark = pytest.mark.gpu


def _mods():
    from sionna_b200.phy.fec import linear, utils
    return linear, utils


def _llrs(rng, gm, ebno_db, num):
    k, n = gm.shape
    u = rng.integers(0, 2, (num, k))
    c = O.encode(u, gm)
    no = 1 / (10 ** (ebno_db / 10) * k / n)
    y = (2.0 * c - 1) + rng.normal(size=c.shape) * np.sqrt(no / 2)
    return (4 * y / no).astype(np.float32), c


def _tutorial_gm():
    """The reference's 5G LDPC (64, 128) generator (1-based sparse (row, col) pairs in the golden file)."""
    import os
    sp = np.load(os.path.join(os.path.dirname(__file__), "golden", "ldpc_k64_n128_G.npy")).astype(int)
    gm = np.zeros((64, 128), np.int64)
    gm[sp[0] - 1, sp[1] - 1] = 1
    return gm


def _disc(l, c):
    l = np.clip(l.astype(np.float32), -100, 100).astype(np.float64)
    return float(((c != (l > 0)) * np.abs(l)).sum())


def _is_codeword(c, gm):
    from sionna_b200.phy.fec.utils import gm2pcm
    k, n = gm.shape
    if k == n:
        return True
    return not np.any(np.asarray(c, np.int64) @ gm2pcm(gm).astype(np.int64).T % 2)


# ---------------------------------------------------------------- encoder

@pytest.mark.parametrize("pcm_id", range(5))
def test_encoder_example_codes(cuda_device, pcm_id):
    linear, utils = _mods()
    pcm, k, n, _ = utils.load_parity_check_examples(pcm_id)
    enc = linear.LinearEncoder(pcm, is_pcm=True)
    gm = O.pcm2gm(pcm)
    assert np.array_equal(enc.gm.cpu().numpy(), gm) and (enc.k, enc.n, enc.coderate) == (k, n, k / n)
    u = np.random.default_rng(pcm_id).integers(0, 2, (333, k))
    c = enc(torch.tensor(u, dtype=torch.float32, device=cuda_device)).cpu().numpy()
    assert np.array_equal(c, O.encode(u, gm))
    assert not np.any(c @ pcm.T % 2)


def test_encoder_tutorial_generator(cuda_device):
    linear, _ = _mods()
    gm = _tutorial_gm()
    u = np.random.default_rng(0).integers(0, 2, (1000, 64))
    c = linear.LinearEncoder(gm)(torch.tensor(u, device=cuda_device, dtype=torch.float32)).cpu().numpy()
    assert np.array_equal(c, O.encode(u, gm))


def test_encoder_random_pcms(cuda_device):
    linear, _ = _mods()
    rng = np.random.default_rng(1)
    done = 0
    while done < 100:
        pcm = rng.integers(0, 2, (123 - 89, 123))
        try:
            enc = linear.LinearEncoder(pcm, is_pcm=True)
        except ValueError:
            continue
        done += 1
        u = rng.integers(0, 2, (100, 89))
        c = enc(torch.tensor(u, device=cuda_device, dtype=torch.float32)).cpu().numpy().astype(np.int64)
        assert not np.any(c @ pcm.T % 2)
        assert np.array_equal(c, O.encode(u, O.pcm2gm(pcm)))


@pytest.mark.parametrize("k,n,batch", [(40, 1100, 130), (1100, 1500, 70), (57, 57, 65), (1, 1, 3), (300, 301, 1)])
def test_encoder_random_generators(cuda_device, k, n, batch):
    linear, _ = _mods()
    rng = np.random.default_rng(k + n)
    gm = rng.integers(0, 2, (k, n))
    if k == n:
        gm = np.eye(k, dtype=np.int64)
    u = rng.integers(0, 2, (batch, k))
    c = linear.LinearEncoder(gm)(torch.tensor(u, device=cuda_device, dtype=torch.int64)).cpu().numpy()
    assert np.array_equal(c, O.encode(u, gm))


def test_encoder_largest_5g_shape(cuda_device):
    """k = 8448, n = 25344 (the largest 5G generator's shape): G = [I | R] with a random R; 25 column CTAs and 33 chunks
    of information bits, more than one tile of codewords."""
    linear, _ = _mods()
    rng = np.random.default_rng(8)
    k, n = 8448, 25344
    r = rng.integers(0, 2, (k, n - k), dtype=np.uint8)
    enc = linear.LinearEncoder(np.concatenate([np.eye(k, dtype=np.uint8), r], axis=1))
    u = rng.integers(0, 2, (70, k), dtype=np.uint8)
    c = enc(torch.tensor(u, device=cuda_device, dtype=torch.float32)).cpu().numpy()
    par = (u.astype(np.float32) @ r.astype(np.float32)) % 2                  # exact: sums < 2^24
    assert np.array_equal(c[:, :k], u) and np.array_equal(c[:, k:], par)


def test_encoder_dtypes(cuda_device):
    linear, utils = _mods()
    pcm, k, n, _ = utils.load_parity_check_examples(2)
    u = np.random.default_rng(2).integers(0, 2, (20, k))
    ref = O.encode(u, O.pcm2gm(pcm))
    for prec, fdt in (("single", torch.float32), ("double", torch.float64)):
        enc = linear.LinearEncoder(pcm, is_pcm=True, precision=prec)
        for dt in (torch.float16, torch.float32, torch.float64, torch.int32, torch.int64):
            c = enc(torch.tensor(u, device=cuda_device).to(dt))
            assert c.dtype == (fdt if dt.is_floating_point else dt)
            assert np.array_equal(c.cpu().to(torch.int64).numpy(), ref)


def test_encoder_shapes_and_errors(cuda_device):
    linear, utils = _mods()
    pcm, k, n, _ = utils.load_parity_check_examples(3)
    enc = linear.LinearEncoder(pcm, is_pcm=True)
    g = torch.Generator().manual_seed(0)
    for s in ([k], [10, 20, 30, k], [1, 40, k], [10, 2, 3, 4, 3, k], [0, k]):
        u = torch.randint(0, 2, s, generator=g).float().to(cuda_device)
        c = enc(u)
        assert list(c.shape) == s[:-1] + [n]
        assert torch.equal(c.reshape(-1, n), enc(u.reshape(-1, k)))
    with pytest.raises(ValueError):
        enc(torch.zeros(10, 2, k - 1, device=cuda_device))
    bad = pcm.copy()
    bad[0, 0] = 2
    with pytest.raises(ValueError):
        linear.LinearEncoder(bad)
    with pytest.raises(ValueError):
        linear.LinearEncoder(bad, is_pcm=True)
    with pytest.raises(ValueError):
        linear.LinearEncoder(np.zeros((2, 3, 4)))
    with pytest.raises(AttributeError):
        linear.LinearEncoder(np.ones((5, 4), int))


# ---------------------------------------------------------------- OSD

def _decode(dec, llr, dev):
    return dec(torch.tensor(llr, device=dev)).cpu().numpy().astype(np.int64)


def _check_against(llr, out, ref_fn, gm):
    """Identical decisions where the oracle's gap exceeds the tolerance, else D within it; always a codeword."""
    mism = 0
    for l, c in zip(llr, out):
        r, d, d2 = ref_fn(l)
        tol = 1e-5 * float(np.abs(np.clip(l, -100, 100)).sum())
        if d2 - d > tol:
            mism += not np.array_equal(c, r)
        else:
            assert _disc(l, c) <= d + tol
    assert mism == 0
    assert _is_codeword(out, gm)


def test_osd_is_ml_at_order_k(cuda_device):
    linear, utils = _mods()
    rng = np.random.default_rng(3)
    codes = [O.pcm2gm(utils.load_parity_check_examples(0)[0])]
    while len(codes) < 12:
        k = int(rng.integers(1, 11))
        n = int(rng.integers(k, 20))
        g = rng.integers(0, 2, (k, n))
        if O.gf2_rank(g) == k:
            codes.append(g)
    for gm in codes:
        k = gm.shape[0]
        llr, _ = _llrs(rng, gm, 0.0, 200)
        for t in (k, k + 2):
            out = _decode(linear.OSDecoder(gm, t=t), llr, cuda_device)
            _check_against(llr, out, lambda l: O.ml_bruteforce(l, gm, return_gap=True), gm)


@pytest.mark.parametrize("pcm_id,t,num", [(0, 1, 300), (0, 2, 300), (1, 1, 200), (1, 2, 100), (1, 3, 20),
                                          (2, 1, 100), (2, 2, 30), (3, 1, 100), (3, 2, 30), (4, 1, 40)])
def test_osd_matches_discrepancy_oracle(cuda_device, pcm_id, t, num):
    linear, utils = _mods()
    pcm = utils.load_parity_check_examples(pcm_id)[0]
    gm = O.pcm2gm(pcm)
    dec = linear.OSDecoder(pcm, t=t, is_pcm=True)
    rng = np.random.default_rng(10 * pcm_id + t)
    for ebno in (0.0, 2.0, 4.0):
        llr, _ = _llrs(rng, gm, ebno, num)
        out = _decode(dec, llr, cuda_device)
        _check_against(llr, out, lambda l: O.osd_discrepancy(l, gm, t, return_gap=True), gm)


@pytest.mark.parametrize("t,num", [(1, 200), (2, 100), (3, 20), (4, 6)])
def test_osd_tutorial_ldpc(cuda_device, t, num):
    linear, _ = _mods()
    gm = _tutorial_gm()
    dec = linear.OSDecoder(gm, t=t)
    rng = np.random.default_rng(t)
    for ebno in (1.0, 3.0):
        llr, _ = _llrs(rng, gm, ebno, num)
        out = _decode(dec, llr, cuda_device)
        _check_against(llr, out, lambda l: O.osd_discrepancy(l, gm, t, return_gap=True), gm)


def test_osd_order_zero_and_full_length(cuda_device):
    linear, utils = _mods()
    rng = np.random.default_rng(5)
    gm = O.pcm2gm(utils.load_parity_check_examples(1)[0])
    llr, _ = _llrs(rng, gm, 1.0, 50)
    out = _decode(linear.OSDecoder(gm, t=0), llr, cuda_device)
    ref = np.stack([O.osd_discrepancy(l, gm, 0) for l in llr])
    assert np.array_equal(out, ref)
    eye = np.eye(9, dtype=np.int64)
    llr = rng.normal(size=(20, 9)).astype(np.float32)
    assert np.array_equal(_decode(linear.OSDecoder(eye, t=3), llr, cuda_device), (llr > 0).astype(np.int64))
    assert linear.OSDecoder(eye, t=3)(torch.zeros(0, 9, device=cuda_device)).shape == (0, 9)


def test_osd_numerical_stability(cuda_device):
    linear, utils = _mods()
    pcm, k, _, _ = utils.load_parity_check_examples(1)
    enc = linear.LinearEncoder(pcm, is_pcm=True)
    dec = linear.OSDecoder(pcm, is_pcm=True)
    u = torch.randint(0, 2, (100, k), device=cuda_device).float()
    c = enc(u)
    for s in (1000., 1e-4):
        assert torch.equal(dec(s * (2 * c - 1)), c)


def test_osd_saturated_llrs_choose_the_better_word(cuda_device):
    """Every flip costs |llr| > 88.7: the reference's float32 metric is inf for all candidates and keeps the order-0
    word; the discrepancy is finite and the kernel returns the ML word."""
    linear, utils = _mods()
    gm = O.pcm2gm(utils.load_parity_check_examples(0)[0])
    l = np.array([[95, -95, 99, 98, -97, 96, 94]], np.float32)
    out = _decode(linear.OSDecoder(gm, t=4), l, cuda_device)
    assert np.array_equal(out[0], O.ml_bruteforce(l[0], gm))


def test_osd_shapes_dtypes_and_errors(cuda_device):
    linear, utils = _mods()
    pcm, _, n, _ = utils.load_parity_check_examples(3)
    dec = linear.OSDecoder(pcm, is_pcm=True, t=2)
    g = torch.Generator().manual_seed(1)
    for s in ([n], [10, 20, 30, n], [1, 40, n], [10, 2, 3, 4, 3, n]):
        llr = (torch.randn(s, generator=g) * 3 - 2).to(cuda_device)
        assert torch.equal(dec(llr).reshape(-1, n), dec(llr.reshape(-1, n)))
    pcm1, _, n1, _ = utils.load_parity_check_examples(1)
    gm1 = O.pcm2gm(pcm1)
    llr = torch.randn(100, n1, device=cuda_device) * 4
    for dt in (torch.float16, torch.float32, torch.float64):
        for prec, out_dt in (("single", torch.float32), ("double", torch.float64)):
            c = linear.OSDecoder(gm1, precision=prec)(llr.to(dt))
            assert c.dtype == out_dt
    pcm2, k2, n2, _ = utils.load_parity_check_examples(2)
    d2 = linear.OSDecoder(pcm2, is_pcm=True)
    d2(torch.zeros(20, n2, device=cuda_device))
    d2(torch.zeros(21, n2, device=cuda_device))
    with pytest.raises(ValueError):
        d2(torch.zeros(20, n2 + 1, device=cuda_device))
    bad = pcm2.copy()
    bad[1, 2] = 2
    with pytest.raises(TypeError):
        linear.OSDecoder(bad)
    with pytest.raises(TypeError):
        linear.OSDecoder(bad, is_pcm=True)
    with pytest.raises(AttributeError):
        linear.OSDecoder()
    with pytest.raises(ValueError):                              # rank deficient
        linear.OSDecoder(np.array([[1, 1, 0], [1, 1, 0]]))
    with pytest.raises(ResourceWarning):
        linear.OSDecoder(pcm2, is_pcm=True, t=8)
    with pytest.raises(ValueError):                              # n > 1024
        linear.OSDecoder(np.eye(4, 1100, dtype=np.int64), t=1)
    assert (d2.k, d2.n, d2.t) == (k2, n2, 0)
    assert d2._num_error_patterns(45, 3) == 14190 and d2._gen_error_patterns(10, 3).shape == (120, 3)


def test_osd_equal_llrs_batch_independent(cuda_device):
    linear, utils = _mods()
    pcm = utils.load_parity_check_examples(1)[0]
    dec = linear.OSDecoder(pcm, is_pcm=True, t=2)
    rng = np.random.default_rng(6)
    n = pcm.shape[1]
    alone = np.where(rng.integers(0, 2, (8, n)) > 0, 1.5, -1.5).astype(np.float32)
    alone[:, ::3] = 0.0
    batch = rng.normal(size=(1000, n)).astype(np.float32)
    pos = rng.choice(1000, 8, replace=False)
    batch[pos] = alone
    ref = _decode(dec, alone, cuda_device)
    for i in range(8):
        assert np.array_equal(_decode(dec, alone[i:i + 1], cuda_device)[0], ref[i])
    assert np.array_equal(_decode(dec, batch, cuda_device)[pos], ref)


def test_osd_encoder_argument(cuda_device):
    linear, _ = _mods()
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder
    from sionna_b200.phy.fec.conv import ConvEncoder
    from sionna_b200.phy.fec.turbo import TurboEncoder
    g = _tutorial_gm()
    assert np.array_equal(linear.OSDecoder(encoder=LDPC5GEncoder(64, 128), t=1).gm.cpu().numpy(), g)
    conv = ConvEncoder(rate=1 / 2, constraint_length=3)
    with pytest.raises(AttributeError):
        linear.OSDecoder(encoder=conv)
    conv(torch.zeros(1, 20, device=cuda_device))
    turbo = TurboEncoder(constraint_length=4, rate=1 / 3, terminate=True, interleaver_type="random")
    turbo(torch.zeros(1, 20, device=cuda_device))
    lin = linear.LinearEncoder(g)
    for e in (conv, turbo, lin):
        gm = linear.OSDecoder(encoder=e, t=1).gm
        ref = e(torch.eye(e.k, device=cuda_device)[None])[0]
        assert torch.equal(gm.cpu(), ref.cpu().to(gm.dtype))


# ---------------------------------------------------------------- links

def _bpsk_model(enc, dec, dev):
    def run(batch_size, ebno_db):
        k, n = enc.k, enc.n
        b = torch.randint(0, 2, (batch_size, k), device=dev).float()
        c = enc(b)
        no = 1 / (10 ** (float(ebno_db) / 10) * k / n)
        y = (2 * c - 1) + torch.randn_like(c) * np.sqrt(no / 2)
        return c, dec(4 * y / no)
    return run


def test_ml_bler_reference_tables(cuda_device):
    linear, utils = _mods()
    from sionna_b200.phy.utils import sim_ber
    torch.manual_seed(0)
    for pid, t, snrs, ref, bs, target in (
            (0, 2, np.linspace(0, 5, 6), [1.832e-01, 1.253e-01, 7.047e-02, 2.899e-02, 1.252e-02, 4.371e-03], 1000,
             10000),
            (1, 4, np.array([0, 1.5, 3., 4]), [6.329e-01, 2.445e-01, 2.595e-02, 2.134e-03], 2000, 1000)):
        pcm = utils.load_parity_check_examples(pid)[0]
        enc = linear.LinearEncoder(pcm, is_pcm=True)
        dec = linear.OSDecoder(encoder=enc, t=t)
        _, bler = sim_ber(_bpsk_model(enc, dec, cuda_device), snrs, batch_size=bs, max_mc_iter=500,
                          num_target_block_errors=target, verbose=False)
        assert np.all(np.isclose(bler.cpu().numpy(), ref, rtol=0.2)), (pid, bler)


def test_osd4_no_worse_than_bp20_on_5g_ldpc(cuda_device):
    linear, _ = _mods()
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    torch.manual_seed(1)
    enc = LDPC5GEncoder(64, 128)
    osd = linear.OSDecoder(encoder=enc, t=4)
    bp = LDPC5GDecoder(enc, num_iter=20, hard_out=True)
    b = torch.randint(0, 2, (2000, 64), device=cuda_device).float()
    c = enc(b)
    no = 1 / (10 ** 0.2 * 0.5)
    llr = 4 * ((2 * c - 1) + torch.randn_like(c) * np.sqrt(no / 2)) / no
    err_osd = int((osd(llr) != c).any(-1).sum())
    err_bp = int((bp(llr) != b).any(-1).sum())
    assert err_osd <= err_bp, (err_osd, err_bp)


@pytest.mark.parametrize("pcm_id", [3, 4])
def test_bp_decodes_linear_encoder_codewords(cuda_device, pcm_id):
    linear, utils = _mods()
    from sionna_b200.phy.fec.ldpc import LDPCBPDecoder
    torch.manual_seed(pcm_id)
    pcm, k, n, _ = utils.load_parity_check_examples(pcm_id)
    enc = linear.LinearEncoder(pcm, is_pcm=True)
    dec = LDPCBPDecoder(pcm, num_iter=10)
    no = 0.3
    c = enc(torch.randint(0, 2, (10, k), device=cuda_device).float())
    llr = 2 / no ** 2 * ((2 * c - 1) + torch.randn_like(c) * np.sqrt(no / 2))
    assert torch.equal(dec(llr), c)
    assert not torch.equal((llr > 0).float(), c)
