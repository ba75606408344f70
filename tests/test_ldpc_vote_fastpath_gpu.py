"""GPU parity of the two-phi rows of the boxplus-phi QC decoder's voting pass, with the union masks they meet counted.

In a voting iteration a row slice whose union mask U (bit l: |x_l| < 14.7117348 in some lane of the warp) holds no
edge but the last is finished inline in the kernel (two phi, then the sign-mask stores, then the fused degree-1
update from a register); every other row slice takes the out-of-line 2k + 1 walk. A lane outside the row
(lane_i >= zrow) reads a valid slot of the row and must drop its bits and store nothing.

The codes:
  * k = 3840, n = 11520: base graph 1 with every row degree of it (3 ... 10 and 19), Z = 176, so the last 32-lane slice
    of every block row holds 16 checks, and a partial last block row of 112 checks;
  * k = 1000, n = 4000: base graph 2 at Z = 104 (degrees 3, 4, 5, 6, 8, 10), partial slices and a partial last row.
Eb/N0 is spread over -1 ... 5 dB, so a launch holds codewords that vote early, late or never. From the states after
every iteration the test counts, for the iterations that certainly vote (the saturation probe fired on the first edge
pair of a row slice in an earlier iteration), the row slices whose U is empty, {last}, a single inner edge and the
full row, for every degree and in the partial slices, and requires each to occur. Soft outputs and the final v2c state
must equal the oracle in kernel math and kernel order bit for bit.
"""
import numpy as np
import pytest
import torch

from oracle import ldpc as O

PHI_ZERO = np.float32(14.7117348)   # SB_PHI_ZERO of ldpc_bp_qc.cu: the union mask's bound
PHI_HI = np.float32(16.635532)      # SB_PHI_HI: the probe's bound

CODES = [(3840, 11520, 176, 112, {3, 4, 5, 6, 7, 8, 9, 10, 19}),
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
@pytest.mark.parametrize("k, n, z, last, degrees", CODES)
def test_vote_fast_path_bit_exact(cuda_device, k, n, z, last, degrees):
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    from bench import host_cores
    bs, it = 240, 20
    rng = np.random.default_rng(k * 7 + n)
    enc_r = O.LDPC5GEncoderRef(k, n)
    c = enc_r(rng.integers(0, 2, (bs, k)))
    ebno = np.repeat(np.linspace(-1.0, 5.0, 12), bs // 12)
    no = 1.0 / (10 ** (ebno[:, None] / 10) * (k / n))
    y = (2.0 * c - 1.0) + rng.normal(size=c.shape) * np.sqrt(no / 2)
    llr = (4 * y / no).astype(np.float32)
    enc = LDPC5GEncoder(k, n)
    assert enc.z == z
    dec = LDPC5GDecoder(enc, hard_out=False, return_infobits=False, num_iter=it, return_state=True)
    assert dec._graph.is_qc() and dec._num_cns % z == last
    d_llr = torch.from_numpy(llr).to(cuda_device)
    x, st = dec(d_llr)
    ref = O.LDPC5GDecoderRef(enc_r, hard_out=False, return_infobits=False, num_iter=it, return_state=True)
    xr, sr = ref(llr, math_mode=1, order="kernel", num_threads=host_cores()[0])
    assert np.array_equal(x.cpu().numpy(), xr)
    assert np.array_equal(st.cpu().numpy(), sr)

    # union masks met by the voting iterations t (input: the state after t iterations)
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
    err = ((xr > 0) != (c > 0)).any(axis=1)
    assert err[: bs // 12].any() and not err[-bs // 12:].any()   # failing and converged codewords in the same launch
