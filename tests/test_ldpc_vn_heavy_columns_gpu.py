"""GPU parity of the QC kernel's variable-node code for columns of degree 13...32.

The 5G base graphs reach these degrees only in the two punctured columns of base graph 1, and which degree they have
depends on the code rate: 19 and 17 (the exact-degree code of the QC kernel) at the rates that keep 24 block rows, other
values (the guarded buckets of 20 and 32 edges) elsewhere. The synthetic lifted code below has every case at once, with
Z = 40, so the wrap of (j - s) mod Z falls inside a warp and the second lane slice of a block is partly empty:
columns of degree 19 and 17 in full block rows only (exact-degree code), of degree 15 and 20 (bucket of 20), of degree
25 and 32 (bucket of 32), and columns of degree 19, 17 and 13 with an edge into the last block row, which is cut to 17
checks (loop code with per-entry limits). Every row ends in a degree-1 column, so the fused update runs as well.
Soft outputs and state must equal, bit for bit, the generic kernel's and the oracle's in kernel math and kernel order,
for every rule, over an Eb/N0 mix where boxplus-phi switches to its voting variant in some CTAs only.
"""
import numpy as np
import pytest
import torch

from oracle import ldpc as O

Z, ROWS, LAST = 40, 34, 17
# (degree, reaches into the cut last block row)
HEAVY = [(19, False), (17, False), (15, False), (20, False), (25, False), (32, False), (19, True), (17, True), (13, True)]
LIGHT = 30
COLS = len(HEAVY) + LIGHT + ROWS


def _base_graph():
    rng = np.random.default_rng(11)
    ents = {}
    for c, (deg, cut) in enumerate(HEAVY):
        rows = rng.choice(np.arange(ROWS - 1), deg - cut, replace=False).tolist() + ([ROWS - 1] if cut else [])
        for r in rows:
            ents[(r, c)] = int(rng.integers(0, Z))
    for c in range(len(HEAVY), len(HEAVY) + LIGHT):
        for r in rng.choice(np.arange(ROWS), int(rng.integers(2, 6)), replace=False).tolist():
            ents[(r, c)] = int(rng.integers(0, Z))
    for r in range(ROWS):                                  # the row's last column has degree 1
        ents[(r, len(HEAVY) + LIGHT + r)] = int(rng.integers(0, Z))
    br, bc = np.array(list(ents), np.int32).T
    return br, bc, np.array(list(ents.values()), np.int32)


def _lifted_pcm(br, bc, sh):
    C = (ROWS - 1) * Z + LAST
    pcm = np.zeros((ROWS * Z, COLS * Z), np.float64)
    i = np.arange(Z)
    for r, c, s in zip(br, bc, sh):
        pcm[r * Z + i, c * Z + (i + s) % Z] = 1
    return pcm[:C]


def test_graph_has_the_heavy_columns():
    br, bc, sh = _base_graph()
    cdeg = np.bincount(bc, minlength=COLS)
    assert cdeg[:len(HEAVY)].tolist() == [d for d, _ in HEAVY]
    for c, (_, cut) in enumerate(HEAVY):
        assert bool(((bc == c) & (br == ROWS - 1)).any()) == cut
    assert (cdeg[len(HEAVY):len(HEAVY) + LIGHT] <= 12).all() and (cdeg[len(HEAVY) + LIGHT:] == 1).all()
    assert (sh[bc < len(HEAVY)] > 0).any()                 # shifted entries: some lanes wrap, others do not


@pytest.mark.gpu
@pytest.mark.parametrize("rule", ["boxplus-phi", "boxplus", "minsum", "offset-minsum"])
def test_heavy_columns_bit_exact(cuda_device, rule):
    from sionna_b200.phy.fec.ldpc import LDPCBPDecoder
    br, bc, sh = _base_graph()
    pcm = _lifted_pcm(br, bc, sh)
    n, bs, it = pcm.shape[1], 96, 20
    rng = np.random.default_rng(23)
    ebno = np.repeat(np.linspace(0.0, 5.0, 6), bs // 6)   # the all-zero codeword
    no = 1.0 / (10 ** (ebno[:, None] / 10) * 0.5)
    llr = ((-1.0 + rng.normal(size=(bs, n)) * np.sqrt(no / 2)) * 4 / no).astype(np.float32)
    x_in = torch.from_numpy(llr).to(cuda_device)
    qc = LDPCBPDecoder(pcm, cn_update=rule, hard_out=False, num_iter=it, return_state=True)
    assert qc._graph.set_qc(Z, br, bc, sh)
    assert qc._graph.is_qc()
    gen = LDPCBPDecoder(pcm, cn_update=rule, hard_out=False, num_iter=it, return_state=True)
    assert not gen._graph.is_qc()
    x, st = qc(x_in)
    xg, sg = gen(x_in)
    xr, sr = O.bp_decode(pcm, llr, num_iter=it, cn_update=rule, hard_out=False, return_state=True, math_mode=1,
                         order="kernel")
    assert np.array_equal(x.cpu().numpy(), xr)
    assert np.array_equal(st.cpu().numpy(), sr)
    assert np.array_equal(xg.cpu().numpy(), xr)
    assert np.array_equal(sg.cpu().numpy(), sr)
    # only the QC kernel stops early: the decode below shows that it is the one being compared
    qc_e = LDPCBPDecoder(pcm, cn_update=rule, hard_out=False, num_iter=it, early_stop=True)
    assert qc_e._graph.set_qc(Z, br, bc, sh)
    xe = qc_e(x_in).cpu().numpy()
    full = qc_e.num_iter_run.cpu().numpy() == it
    assert np.array_equal(xe[full], xr[full])
