"""GPU parity of the boxplus-phi QC decoder (ldpc_bp_qc_kernel, csrc/ldpc_bp_qc.cu), one section per kernel path.

Every decode here is bit-exact against the oracle in kernel math and kernel order: soft outputs and the final v2c
state equal, bit for bit, those of the CPU oracle run with math_mode=1 (the product's own sb_math.h, including the
table-driven logs of phi) and order="kernel" (each node sums its inputs in ascending neighbour index, the order the
kernels use). A kernel that sums in another order, or evaluates phi differently, fails.

The batches mix Eb/N0 from codewords that do not converge within 20 iterations to codewords that converge early, so
the boxplus-phi decode switches to its voting variant early, late or not at all within one launch, and in some CTAs
only; `assert_mixed_convergence` checks both ends. In the voting iterations a row slice evaluates phi only where some
lane of the warp is unsaturated (the union mask U, bit l: |x_l| < SB_PHI_ZERO in some lane). A row slice whose U holds
no edge but the last takes two phi inline, every other one the out-of-line 2k + 1 walk; a lane outside a row
(lane_i >= zrow) reads a valid slot of the row and must neither vote nor store in it.
"""
import numpy as np
import pytest
import torch

from oracle import ldpc as O
from oracle.parity import assert_bit_exact, assert_mixed_convergence, bpsk_llr, lifted_pcm

PHI_ZERO = np.float32(14.7117348)   # SB_PHI_ZERO of ldpc_bp_qc.cu: the union mask's bound
PHI_HI = np.float32(16.635532)      # SB_PHI_HI: the saturation probe's bound and the clipping bound of phi


def _decode_5g(k, n, llr, enc_r, it, dev):
    """(decoder, oracle decoder, oracle soft outputs) of the 5G decode of llr, asserted bit-exact on the QC kernel."""
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    from bench import host_cores
    dec = LDPC5GDecoder(LDPC5GEncoder(k, n), hard_out=False, return_infobits=False, num_iter=it, return_state=True)
    assert dec._graph.is_qc()
    x, st = dec(torch.from_numpy(llr).to(dev))
    ref = O.LDPC5GDecoderRef(enc_r, hard_out=False, return_infobits=False, num_iter=it, return_state=True)
    xr, sr = ref(llr, math_mode=1, order="kernel", num_threads=host_cores()[0])
    assert_bit_exact(x, st, xr, sr)
    return dec, ref, xr


def _snr_mix(k, n, bs, lo, hi, groups, seed):
    """(oracle encoder, codewords, LLRs) of bs random codewords over `groups` Eb/N0 steps from lo to hi dB."""
    rng = np.random.default_rng(seed)
    enc_r = O.LDPC5GEncoderRef(k, n)
    c = enc_r(rng.integers(0, 2, (bs, k)))
    return enc_r, c, bpsk_llr(c, np.repeat(np.linspace(lo, hi, groups), bs // groups), k / n, rng)


# ---- the phi zero bound -----------------------------------------------------------------------------------------------
# The mask treats |x| >= PHI_ZERO as saturated: phi must be +0 for every fp32 value from there up to PHI_HI, in the
# oracle and on the device.
def _sweep():
    """Every fp32 value in [PHI_ZERO, PHI_HI], and the one just below PHI_ZERO."""
    lo, hi = int(PHI_ZERO.view(np.uint32)), int(PHI_HI.view(np.uint32))
    return np.arange(lo - 1, hi + 1, dtype=np.uint32).view(np.float32)


def test_phi_zero_bound_oracle():
    x = _sweep()
    phi = np.array([O.phi(v, 1) for v in x])
    assert phi[0] > 0 and np.all(phi[1:] == 0)


@pytest.mark.gpu
def test_phi_zero_bound_device(cuda_device):
    from sionna_b200 import _lib
    x = _sweep()
    x = x[: len(x) // 2 * 2]
    xd = torch.from_numpy(x).to(cuda_device)
    o1, o2 = torch.empty_like(xd), torch.empty_like(xd)
    _lib.check(_lib.lib().sb_debug_phi(_lib.ptr(xd), _lib.ptr(o1), _lib.ptr(o2), len(x), _lib.current_stream()), "sb_debug_phi")
    for o in (o1.cpu().numpy(), o2.cpu().numpy()):
        assert o[0] > 0 and np.all(o[1:].view(np.uint32) == 0)


# ---- voting-pass shapes: partial slices and partial rows --------------------------------------------------------------
# In the voting iterations a warp walks its block rows class-agnostically. The codes below each bring one shape the
# benchmark code (Z = 192, four warp groups of six full block rows) lacks:
#   * k = 1000, n = 2000: Z = 104, not a multiple of 32, so the last 32-lane slice of every row is partly empty; the
#     pruned graph ends in a partial block row (64 of 104 checks);
#   * k = 2000, n = 5000: Z = 208 and a partial last block row (88 checks); warp groups get unequal row counts (6, 6, 5);
#   * k = 700, n = 1600: Z = 72, a partial last block row, eight warp groups of which one gets a single row.
# (k, n, Z, checks in the last block row, block rows per warp group)
VOTING_CODES = [(1000, 2000, 104, 64, [2, 2, 2, 2, 2, 2]),
                (2000, 5000, 208, 88, [6, 6, 5]),
                (700, 1600, 72, 36, [2, 2, 2, 2, 2, 2, 2, 1])]


def _rows_per_group(z, c, n):
    """Block rows dealt to each warp group of the QC kernel (768 threads, one 32-lane slice of a row per warp)."""
    rows, cols = -(-c // z), -(-n // z)
    g = max(1, min(24 // -(-z // 32), max(rows, cols)))
    return [len(range(i, rows, g)) for i in range(g)]


@pytest.mark.parametrize("k, n, z, last, groups", VOTING_CODES)
def test_codes_have_the_shapes(k, n, z, last, groups):
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    enc = LDPC5GEncoder(k, n)
    dec = LDPC5GDecoder(enc, num_iter=1)
    c = dec._num_cns
    assert enc.z == z and c % z == last
    assert _rows_per_group(z, c, dec._num_vns) == groups


@pytest.mark.gpu
@pytest.mark.parametrize("k, n, z, last, groups", VOTING_CODES)
def test_voting_rows_bit_exact(cuda_device, k, n, z, last, groups):
    bs, it = 400, 20
    enc_r, c, llr = _snr_mix(k, n, bs, -1.0, 5.0, 10, k + n)
    _, _, xr = _decode_5g(k, n, llr, enc_r, it, cuda_device)
    assert_mixed_convergence(xr, c, 10)


# ---- the two-phi fast path and its union-mask census -------------------------------------------------------------------
# The codes:
#   * k = 3840, n = 11520: base graph 1 with every row degree of it (3 ... 10 and 19), Z = 176, so the last 32-lane
#     slice of every block row holds 16 checks, and a partial last block row of 112 checks;
#   * k = 1000, n = 4000: base graph 2 at Z = 104 (degrees 3, 4, 5, 6, 8, 10), partial slices and a partial last row.
# From the states after every iteration the test counts, for the iterations that certainly vote (the saturation probe
# fired on the first edge pair of a row slice in an earlier iteration), the row slices whose U is empty, {last}, a
# single inner edge and the full row, for every degree and in the partial slices, and requires each to occur.
FASTPATH_CODES = [(3840, 11520, 176, 112, {3, 4, 5, 6, 7, 8, 9, 10, 19}),
                  (1000, 4000, 104, 88, {3, 4, 5, 6, 8, 10})]


class SliceMasks:
    """Union mask and probe result of every (block row, 32-lane slice) of a lifted graph, from a v2c state [E, B]."""

    def __init__(self, cn, vn, z):
        order = np.lexsort((vn, cn))                          # by check, ascending VN (= ascending base column)
        cn_s = cn[order]
        first = np.searchsorted(cn_s, cn_s, side="left")
        pos = np.arange(len(cn_s)) - first                     # edge position l inside its check
        deg = np.bincount(cn_s)[cn_s]
        row, lane = cn_s // z, cn_s % z
        sl = lane // 32
        nsl = -(-z // 32)
        gid = row * nsl + sl
        g_order = np.lexsort((pos, gid))
        self.edge = order[g_order]
        self.pos = pos[g_order].astype(np.uint32)
        gid = gid[g_order]
        self.start = np.flatnonzero(np.r_[True, gid[1:] != gid[:-1]])
        self.deg = deg[g_order][self.start]
        checks = np.bincount(cn_s // z)                        # edges per block row
        zrow = checks[row[g_order][self.start]] // self.deg   # checks of the slice's block row
        sl0 = sl[g_order][self.start]
        self.partial = (sl0 + 1) * 32 > zrow                   # the slice has lanes outside the row
        p01 = np.flatnonzero(self.pos < 2)
        self.p01_edge, self.p01_gid = self.edge[p01], gid[p01]

    def union(self, st):
        un = (np.abs(st[self.edge]) < PHI_ZERO).astype(np.uint32) << self.pos[:, None]
        return np.bitwise_or.reduceat(un, self.start, axis=0)

    def probe(self, st):
        sat = np.abs(st[self.p01_edge]) >= PHI_HI
        starts = np.flatnonzero(np.r_[True, self.p01_gid[1:] != self.p01_gid[:-1]])
        return np.logical_and.reduceat(sat, starts, axis=0).any(axis=0)


@pytest.mark.gpu
@pytest.mark.parametrize("k, n, z, last, degrees", FASTPATH_CODES)
def test_vote_fast_path_bit_exact(cuda_device, k, n, z, last, degrees):
    bs, it = 240, 20
    enc_r, c, llr = _snr_mix(k, n, bs, -1.0, 5.0, 12, k * 7 + n)
    dec, ref, xr = _decode_5g(k, n, llr, enc_r, it, cuda_device)
    assert dec.encoder.z == z and dec._num_cns % z == last

    # union masks met by the voting iterations t (input: the state after t iterations)
    d_llr = torch.from_numpy(llr).to(cuda_device)
    masks = SliceMasks(*ref.edges, z)
    full = (np.uint64(1) << masks.deg.astype(np.uint64)) - np.uint64(1)
    top = np.uint64(1) << (masks.deg.astype(np.uint64) - np.uint64(1))
    voting = np.zeros(bs, bool)
    seen = {"empty": 0, "last": 0, "inner": 0, "full": 0, "empty partial": 0, "last partial": 0}
    fast_deg = set()
    for t in range(1, it):
        s_t = dec(d_llr, num_iter=t)[1].cpu().numpy()
        if voting.any():
            u = masks.union(s_t)[:, voting].astype(np.uint64)
            one = (u & (u - np.uint64(1))) == 0
            is_last = u == top[:, None]
            kinds = {"empty": u == 0, "last": is_last, "inner": one & (u != 0) & ~is_last,
                     "full": (u == full[:, None]) & (masks.deg[:, None] > 1)}
            for name, m in kinds.items():
                seen[name] += int(m.sum())
            seen["empty partial"] += int(kinds["empty"][masks.partial].sum())
            seen["last partial"] += int(kinds["last"][masks.partial].sum())
            fast = kinds["empty"] | kinds["last"]
            fast_deg |= set(masks.deg[fast.any(axis=1)].tolist())
        voting |= masks.probe(s_t)
    assert all(v > 0 for v in seen.values()), seen
    assert fast_deg >= degrees, (sorted(fast_deg), sorted(degrees))
    assert set(masks.deg.tolist()) == degrees
    assert_mixed_convergence(xr, c, 12)


# ---- union-mask rows on the benchmark code ----------------------------------------------------------------------------
# Eb/N0 from 0.5 to 5 dB on the benchmark's code (k = 4224, n = 8448): the voting row slices meet every case of the
# code: |U| = 0 and U = {last edge} (the two-phi rows), other small |U| with both pair and scalar tails, and |U| = deg
# (tools/phi_work_model.py counts them).
@pytest.mark.gpu
def test_union_mask_rows_bit_exact_over_snr_mix(cuda_device):
    k, n, bs, it = 4224, 8448, 640, 20
    enc_r, c, llr = _snr_mix(k, n, bs, 0.5, 5.0, 10, 2024)
    _, _, xr = _decode_5g(k, n, llr, enc_r, it, cuda_device)
    assert_mixed_convergence(xr, c, 10)


# ---- heavy row classes ------------------------------------------------------------------------------------------------
# The 5G base graphs have no check of degree > 20 and no variable of degree > 32, so their decodes never run the loop
# classes of the QC kernel. The synthetic lifted code below (Z = 40, 36 block rows, the last one cut to 17 checks) has
# two rows in the loop class (degree > 20): one of degree 26, which the voting variant of boxplus-phi takes, and one of
# degree 36, above the voting variant's 32 edges, which stays on the plain variant. It also has a column of degree 35
# (loop class) and one of degree 36 with an edge into the partial block row (loop class with per-entry limits).
# The early-stop decode must match the oracle for every codeword that ran all iterations.
Z, LAST = 40, 17                                           # both synthetic codes: lifting size, checks in the cut row
RULES = ["boxplus-phi", "boxplus", "minsum", "offset-minsum"]
CLASS_ROWS, CLASS_COLS = 36, 72


def _synthetic_decode(graph, rows, cols, rule, seed, lo, hi, dev):
    """20 iterations over 96 all-zero codewords of the code `graph` (base entries and shifts) lifted by Z, Eb/N0 in six
    steps from lo to hi dB (rate 1/2 in the LLRs): the QC-kernel decode asserted bit-exact, and an early-stop decode
    of the same inputs, which only the QC kernel runs (the generic kernel refuses early_stop), so it shows that the QC
    kernel is the one being compared. (pcm, device LLRs, oracle soft outputs and state, early-stop soft outputs, mask
    of the codewords that ran all iterations)."""
    from sionna_b200.phy.fec.ldpc import LDPCBPDecoder
    pcm = lifted_pcm(Z, rows, cols, LAST, *graph)
    n, bs, it = pcm.shape[1], 96, 20
    llr = bpsk_llr(np.zeros((bs, n)), np.repeat(np.linspace(lo, hi, 6), bs // 6), 0.5, np.random.default_rng(seed))
    x_in = torch.from_numpy(llr).to(dev)
    qc = LDPCBPDecoder(pcm, cn_update=rule, hard_out=False, num_iter=it, return_state=True)
    assert qc._graph.set_qc(Z, *graph)
    assert qc._graph.is_qc()
    x, st = qc(x_in)
    xr, sr = O.bp_decode(pcm, llr, num_iter=it, cn_update=rule, hard_out=False, return_state=True, math_mode=1,
                         order="kernel")
    assert_bit_exact(x, st, xr, sr)
    qc_e = LDPCBPDecoder(pcm, cn_update=rule, hard_out=False, num_iter=it, early_stop=True)
    assert qc_e._graph.set_qc(Z, *graph)
    return pcm, x_in, xr, sr, qc_e(x_in).cpu().numpy(), qc_e.num_iter_run.cpu().numpy() == it


def _heavy_class_graph():
    """Base entries (row, col, shift): rows 0 and 1 heavy, column 0 in every full row, column 1 in every row."""
    rng = np.random.default_rng(5)
    ents = {}
    for r in range(CLASS_ROWS):
        cols = {1} | ({0} if r < CLASS_ROWS - 1 else set())
        deg = 36 if r == 0 else 26 if r == 1 else 6
        cols |= set(rng.choice(np.arange(2, CLASS_COLS), deg - len(cols), replace=False).tolist())
        for c in cols:
            ents[(r, c)] = int(rng.integers(0, Z))
    for c in range(CLASS_COLS):                            # every column gets at least one edge
        if not any((r, c) in ents for r in range(CLASS_ROWS)):
            ents[(int(rng.integers(2, CLASS_ROWS - 1)), c)] = int(rng.integers(0, Z))
    br, bc = np.array(list(ents), np.int32).T
    return br, bc, np.array(list(ents.values()), np.int32)


def test_graph_has_the_heavy_classes():
    br, bc, sh = _heavy_class_graph()
    rdeg, cdeg = np.bincount(br, minlength=CLASS_ROWS), np.bincount(bc, minlength=CLASS_COLS)
    assert rdeg[0] > 32 and 20 < rdeg[1] <= 32
    assert cdeg[0] == CLASS_ROWS - 1 and cdeg[1] == CLASS_ROWS and cdeg[1] > 32
    assert (cdeg > 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("rule", RULES)
def test_heavy_degree_classes_bit_exact(cuda_device, rule):
    _, _, xr, _, xe, full = _synthetic_decode(_heavy_class_graph(), CLASS_ROWS, CLASS_COLS, rule, 17, 1.0, 6.0,
                                              cuda_device)
    ok = (xr < 0).all(axis=1)                              # logits: bit 0 is negative
    assert ok.any() and not ok.all()
    assert full.any() and not full.all()
    assert np.array_equal(xe[full], xr[full])


# ---- heavy columns ----------------------------------------------------------------------------------------------------
# The variable-node code for columns of degree 13...32. The 5G base graphs reach these degrees only in the two
# punctured columns of base graph 1, and which degree they have depends on the code rate: 19 and 17 (the exact-degree
# code of the QC kernel) at the rates that keep 24 block rows, other values (the guarded buckets of 20 and 32 edges)
# elsewhere. The synthetic lifted code below has every case at once, with Z = 40, so the wrap of (j - s) mod Z falls
# inside a warp and the second lane slice of a block is partly empty: columns of degree 19 and 17 in full block rows
# only (exact-degree code), of degree 15 and 20 (bucket of 20), of degree 25 and 32 (bucket of 32), and columns of
# degree 19, 17 and 13 with an edge into the last block row, which is cut to 17 checks (loop code with per-entry
# limits). Every row ends in a degree-1 column, so the fused update runs as well. The generic kernel must give the same
# bits as the QC kernel and the oracle.
COLUMN_ROWS = 34
# (degree, reaches into the cut last block row)
HEAVY = [(19, False), (17, False), (15, False), (20, False), (25, False), (32, False), (19, True), (17, True), (13, True)]
LIGHT = 30
COLUMN_COLS = len(HEAVY) + LIGHT + COLUMN_ROWS


def _heavy_column_graph():
    rng = np.random.default_rng(11)
    ents = {}
    for c, (deg, cut) in enumerate(HEAVY):
        rows = rng.choice(np.arange(COLUMN_ROWS - 1), deg - cut, replace=False).tolist() + ([COLUMN_ROWS - 1] if cut else [])
        for r in rows:
            ents[(r, c)] = int(rng.integers(0, Z))
    for c in range(len(HEAVY), len(HEAVY) + LIGHT):
        for r in rng.choice(np.arange(COLUMN_ROWS), int(rng.integers(2, 6)), replace=False).tolist():
            ents[(r, c)] = int(rng.integers(0, Z))
    for r in range(COLUMN_ROWS):                           # the row's last column has degree 1
        ents[(r, len(HEAVY) + LIGHT + r)] = int(rng.integers(0, Z))
    br, bc = np.array(list(ents), np.int32).T
    return br, bc, np.array(list(ents.values()), np.int32)


def test_graph_has_the_heavy_columns():
    br, bc, sh = _heavy_column_graph()
    cdeg = np.bincount(bc, minlength=COLUMN_COLS)
    assert cdeg[:len(HEAVY)].tolist() == [d for d, _ in HEAVY]
    for c, (_, cut) in enumerate(HEAVY):
        assert bool(((bc == c) & (br == COLUMN_ROWS - 1)).any()) == cut
    assert (cdeg[len(HEAVY):len(HEAVY) + LIGHT] <= 12).all() and (cdeg[len(HEAVY) + LIGHT:] == 1).all()
    assert (sh[bc < len(HEAVY)] > 0).any()                 # shifted entries: some lanes wrap, others do not


@pytest.mark.gpu
@pytest.mark.parametrize("rule", RULES)
def test_heavy_columns_bit_exact(cuda_device, rule):
    from sionna_b200.phy.fec.ldpc import LDPCBPDecoder
    pcm, x_in, xr, sr, xe, full = _synthetic_decode(_heavy_column_graph(), COLUMN_ROWS, COLUMN_COLS, rule, 23, 0.0, 5.0,
                                                    cuda_device)
    gen = LDPCBPDecoder(pcm, cn_update=rule, hard_out=False, num_iter=20, return_state=True)
    assert not gen._graph.is_qc()
    assert_bit_exact(*gen(x_in), xr, sr)
    assert np.array_equal(xe[full], xr[full])
