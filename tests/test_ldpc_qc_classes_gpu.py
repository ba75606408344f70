"""GPU parity of the QC kernel's heavy degree classes against the CPU oracle.

The 5G base graphs have no check of degree > 20 and no variable of degree > 32, so their decodes never run the loop
classes of the QC kernel. The synthetic lifted code below (Z = 40, 36 block rows, the last one cut to 17 checks) has
two rows in the loop class (degree > 20): one of degree 26, which the voting variant of boxplus-phi takes, and one of
degree 36, above the voting variant's 32 edges, which stays on the plain variant. It also has a column of degree 35 (loop
class) and one of degree 36 with an edge into the partial block row (loop class with per-entry limits). Soft outputs and
state must equal the oracle in kernel math and kernel order bit for bit, for every rule, over an Eb/N0 mix where some
codewords converge and others do not, so the boxplus-phi decode switches to the voting variant in some CTAs only.
An early-stop decode of the same inputs, which only the QC kernel runs (the generic kernel refuses early_stop), shows
that the QC kernel is the one being compared, and must match the oracle for every codeword that ran all iterations.
"""
import numpy as np
import pytest
import torch

from oracle import ldpc as O

Z, ROWS, COLS, LAST = 40, 36, 72, 17


def _base_graph():
    """Base entries (row, col, shift): rows 0 and 1 heavy, column 0 in every full row, column 1 in every row."""
    rng = np.random.default_rng(5)
    ents = {}
    for r in range(ROWS):
        cols = {1} | ({0} if r < ROWS - 1 else set())
        deg = 36 if r == 0 else 26 if r == 1 else 6
        cols |= set(rng.choice(np.arange(2, COLS), deg - len(cols), replace=False).tolist())
        for c in cols:
            ents[(r, c)] = int(rng.integers(0, Z))
    for c in range(COLS):                                  # every column gets at least one edge
        if not any((r, c) in ents for r in range(ROWS)):
            ents[(int(rng.integers(2, ROWS - 1)), c)] = int(rng.integers(0, Z))
    br, bc = np.array(list(ents), np.int32).T
    return br, bc, np.array(list(ents.values()), np.int32)


def _lifted_pcm(br, bc, sh):
    C = (ROWS - 1) * Z + LAST
    pcm = np.zeros((ROWS * Z, COLS * Z), np.float64)
    i = np.arange(Z)
    for r, c, s in zip(br, bc, sh):
        pcm[r * Z + i, c * Z + (i + s) % Z] = 1
    return pcm[:C]


def test_graph_has_the_heavy_classes():
    br, bc, sh = _base_graph()
    rdeg, cdeg = np.bincount(br, minlength=ROWS), np.bincount(bc, minlength=COLS)
    assert rdeg[0] > 32 and 20 < rdeg[1] <= 32
    assert cdeg[0] == ROWS - 1 and cdeg[1] == ROWS and cdeg[1] > 32
    assert (cdeg > 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("rule", ["boxplus-phi", "boxplus", "minsum", "offset-minsum"])
def test_heavy_degree_classes_bit_exact(cuda_device, rule):
    from sionna_b200.phy.fec.ldpc import LDPCBPDecoder
    br, bc, sh = _base_graph()
    pcm = _lifted_pcm(br, bc, sh)
    n, bs, it = pcm.shape[1], 96, 20
    rng = np.random.default_rng(17)
    ebno = np.repeat(np.linspace(1.0, 6.0, 6), bs // 6)   # the all-zero codeword, rate 1/2
    no = 1.0 / (10 ** (ebno[:, None] / 10) * 0.5)
    llr = ((-1.0 + rng.normal(size=(bs, n)) * np.sqrt(no / 2)) * 4 / no).astype(np.float32)
    dec = LDPCBPDecoder(pcm, cn_update=rule, hard_out=False, num_iter=it, return_state=True)
    assert dec._graph.set_qc(Z, br, bc, sh)
    assert dec._graph.is_qc()
    x, st = dec(torch.from_numpy(llr).to(cuda_device))
    xr, sr = O.bp_decode(pcm, llr, num_iter=it, cn_update=rule, hard_out=False, return_state=True, math_mode=1,
                         order="kernel")
    assert np.array_equal(x.cpu().numpy(), xr)
    assert np.array_equal(st.cpu().numpy(), sr)
    ok = (xr < 0).all(axis=1)                              # logits: bit 0 is negative
    assert ok.any() and not ok.all()
    dec_e = LDPCBPDecoder(pcm, cn_update=rule, hard_out=False, num_iter=it, early_stop=True)
    assert dec_e._graph.set_qc(Z, br, bc, sh)
    xe = dec_e(torch.from_numpy(llr).to(cuda_device)).cpu().numpy()
    full = dec_e.num_iter_run.cpu().numpy() == it
    assert full.any() and not full.all()
    assert np.array_equal(xe[full], xr[full])
