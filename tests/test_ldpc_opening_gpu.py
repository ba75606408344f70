"""The opening iterations of the boxplus-phi QC decoder (cn_open_pass, csrc/ldpc_bp_qc.cu).

Rate recovery gives the punctured VNs of a 5G code (base columns 0 and 1) the channel LLR 0, so in iteration 0 every
c2v message except those of a row's only punctured edge is +-0 exactly, and every non-punctured VN keeps its v2c. When
every block row has a punctured column among its first two entries, the kernel evaluates phi once per VN instead of
once per edge, runs iteration 0 on the punctured edges and columns only, and evaluates pass-1 phi in iteration 1 only
at the punctured edges. Every decode here must still equal the oracle (math_mode=1, order="kernel") bit for bit, on
graphs that take the path and on one that does not, for iteration counts at and around the path's bounds.
"""
import math

import numpy as np
import pytest
import torch

from oracle import ldpc as O
from oracle.parity import assert_bit_exact, bpsk_llr

# (k, n) -> base graph, lifting size, whether the opening path is on
BG1_BENCH = (4224, 8448)    # BG1, Z = 192, 24 block rows: the benchmark code
BG1_Z96 = (2000, 2800)      # BG1, Z = 96
BG2_ON = (1024, 2048)       # BG2, Z = 104, 12 block rows, each with column 0 or 1
BG2_OFF = (200, 1000)       # BG2, Z = 26, 33 block rows: rows 26 and 30 have neither column 0 nor 1


def _predicted(enc, dec):
    """The planner's condition from the base matrix: every kept block row holds base column 0 or 1 (the punctured
    columns, at edge position 0 or 1 since a row's entries are in ascending column order)."""
    bm = enc._bm[: math.ceil(dec.num_cns / enc.z)]
    return bool(np.all((bm[:, 0] >= 0) | (bm[:, 1] >= 0)))


def test_opening_condition_follows_base_graph():
    """Host only: the planner enables the path exactly where the base-graph tables predict it."""
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    seen = set()
    for k, n in (BG1_BENCH, BG1_Z96, BG2_ON, BG2_OFF, (4000, 12000), (8448, 25344), (3000, 6000), (500, 1000),
                 (300, 1400), (250, 1200), (640, 3000), (100, 200), (562, 871)):
        enc = LDPC5GEncoder(k, n)
        dec = LDPC5GDecoder(enc)
        assert dec._graph.is_qc()
        on = dec._graph.qc_opening()
        assert on == _predicted(enc, dec), (k, n)
        seen.add(on)
    assert seen == {True, False}
    for k, n, on in ((*BG1_BENCH, True), (*BG1_Z96, True), (*BG2_ON, True), (*BG2_OFF, False)):
        assert LDPC5GDecoder(LDPC5GEncoder(k, n))._graph.qc_opening() == on


def _llr(k, n, bs, seed, lo=0.0, hi=4.0):
    rng = np.random.default_rng(seed)
    enc_r = O.LDPC5GEncoderRef(k, n)
    c = enc_r(rng.integers(0, 2, (bs, k)))
    return enc_r, bpsk_llr(c, np.linspace(lo, hi, bs), k / n, rng)


def _check(code, num_iter, bs, seed, dev, hard_out=False):
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    from bench import host_cores
    k, n = code
    enc_r, llr = _llr(k, n, bs, seed)
    dec = LDPC5GDecoder(LDPC5GEncoder(k, n), hard_out=hard_out, return_infobits=False, num_iter=num_iter,
                        return_state=not hard_out)
    ref = O.LDPC5GDecoderRef(enc_r, hard_out=hard_out, return_infobits=False, num_iter=num_iter,
                             return_state=not hard_out)
    out = dec(torch.from_numpy(llr).to(dev))
    res = ref(llr, math_mode=1, order="kernel", num_threads=host_cores()[0])
    if hard_out:
        assert np.array_equal(out.cpu().numpy(), res)
    else:
        assert_bit_exact(out[0], out[1], res[0], res[1])


@pytest.mark.gpu
@pytest.mark.parametrize("num_iter", [1, 2, 3, 20])
@pytest.mark.parametrize("code", [BG1_BENCH, BG1_Z96, BG2_ON, BG2_OFF], ids=["bg1_z192", "bg1_z96", "bg2_on", "bg2_off"])
def test_opening_soft_and_state_bit_exact(cuda_device, code, num_iter):
    """Soft outputs and the final v2c state equal the oracle's over 0...4 dB, on and off the path."""
    _check(code, num_iter, 48, 1000 + num_iter, cuda_device)


@pytest.mark.gpu
@pytest.mark.parametrize("code", [BG1_BENCH, BG2_ON], ids=["bg1_z192", "bg2_on"])
def test_opening_hard_outputs_bit_exact(cuda_device, code):
    _check(code, 20, 48, 77, cuda_device, hard_out=True)


@pytest.mark.gpu
def test_opening_high_snr_saturates_in_iteration_1(cuda_device):
    """At high SNR the first-pair probe of iteration 1 fires in some rows (edge 1 reads the channel LLR of a
    non-punctured VN), so the voting variant starts in iteration 2, as on the plain path."""
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    from bench import host_cores
    k, n = BG1_BENCH
    enc_r, llr = _llr(k, n, 32, 5, lo=6.0, hi=9.0)
    for it in (3, 4, 20):
        dec = LDPC5GDecoder(LDPC5GEncoder(k, n), hard_out=False, return_infobits=False, num_iter=it, return_state=True)
        ref = O.LDPC5GDecoderRef(enc_r, hard_out=False, return_infobits=False, num_iter=it, return_state=True)
        x, st = dec(torch.from_numpy(llr).to(cuda_device))
        xr, sr = ref(llr, math_mode=1, order="kernel", num_threads=host_cores()[0])
        assert_bit_exact(x, st, xr, sr)


@pytest.mark.gpu
def test_opening_early_stop_equals_fixed_iteration_decodes(cuda_device):
    """early_stop=True keeps the plain opening; each codeword's output equals the fixed-iteration decode (which takes
    the opening path for 3 or more iterations) with its reported iteration count."""
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    k, n = BG1_BENCH
    _, llr = _llr(k, n, 64, 9, lo=0.5, hi=4.0)
    x = torch.from_numpy(llr).to(cuda_device)
    enc = LDPC5GEncoder(k, n)
    dec = LDPC5GDecoder(enc, hard_out=False, return_infobits=False, num_iter=20, early_stop=True)
    y = dec(x).cpu().numpy()
    iters = dec.num_iter_run.cpu().numpy()
    assert iters.min() < 20 and iters.max() == 20
    for v in np.unique(iters):
        sel = np.nonzero(iters == v)[0]
        ref = LDPC5GDecoder(enc, hard_out=False, return_infobits=False, num_iter=int(v))(x[sel]).cpu().numpy()
        assert np.array_equal(y[sel], ref), v
