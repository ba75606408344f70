"""The 5G LDPC encoder and decoders at every lifting size Z of both base graphs, against the oracle bit for bit.

The quasi-cyclic (QC) decoder kernel changes shape with Z at almost every level: Zb = ceil(Z / 32) lane slices per block
row (1 ... 12), G = max(1, min(24 / Zb, max(rows, cols))) warp groups, a partial last slice whenever Z % 32 != 0, idle
lanes below Z = 32, partial last block rows after pruning, 16, 8 or 1 copies of the phi log table, the TMA or plain
channel-LLR load, and whether the code fits in shared memory at all (if not, the generic kernel decodes it). A 5G code
can take any of 51 lifting sizes in each base graph; this file builds, on the host, a table of codes that reaches all
102 (base graph, Z) pairs at low, middle and high rate, with and without filler bits, and checks on the device:

  * the encoder kernel against `oracle.ldpc.LDPC5GEncoderRef` (B solved over GF(2), no code shared with the product),
    with batch tails of 1 ... 31 codewords in the last 32-codeword group and more groups than the grid holds;
  * the QC decoder with every check-node rule, soft and hard output, and its v2c state against `LDPC5GDecoderRef` in
    kernel math and kernel order, on launches that hold converging and non-converging codewords;
  * early termination against fixed-iteration decodes, wherever the QC kernel runs;
  * the generic kernel (SB_LDPC_DISABLE_QC=1) on the same table, on chip and with the global workspace;
  * which kernel ran (from the kernel names in a CUDA trace) against the planner's shared-memory rule, restated here;
  * misaligned input pointers (TMA load vs plain load) and batches of 1 and of several codewords per persistent CTA.
Every comparison is np.array_equal / torch.equal: no tolerances.
"""
import dataclasses
import re
import zlib

import numpy as np
import pytest
import torch

from oracle import ldpc as O
from sionna_b200.phy.fec.ldpc.encoding import sel_lifting

RULES = ["boxplus-phi", "boxplus", "minsum", "offset-minsum"]
NUM_ITER = 10
DEC_BATCH = 24
QC_THREADS = 768            # kQcThreads of ldpc_bp_qc.cu
LOGTAB_N = 64               # SB_LOGTAB_N of sb_logtab.h
SMEM_OPTIN_H100 = 232448    # opt-in shared memory per block of sm_90 (227 KB)


@dataclasses.dataclass(frozen=True)
class Code:
    """One table entry and the shape of its pruned decoding graph (from the oracle's LDPC5GDecoderRef)."""
    bg: str
    z: int
    k: int
    n: int
    m: object               # num_bits_per_symbol (output interleaver) or None
    C: int                  # check nodes of the pruned graph
    N: int                  # variable nodes of the pruned graph
    E: int                  # edges
    rows: int               # base rows / columns of the pruned graph (the last ones may be partial)
    cols: int
    nnz: int                # base entries (circulants) of the pruned graph
    max_cn_deg: int
    max_vn_deg: int

    @property
    def id(self):
        return f"{self.bg}-z{self.z}-k{self.k}-n{self.n}" + (f"-m{self.m}" if self.m else "")

    @property
    def group(self):
        return self.bg, self.z, self.k

    @property
    def zb(self):
        return (self.z + 31) // 32

    @property
    def g_plan(self):
        """Warp groups the host planner balances the rows and columns for."""
        return max(1, (QC_THREADS // 32) // self.zb)

    @property
    def g_launch(self):
        """Warp groups of the launch."""
        return max(1, min(self.g_plan, max(self.rows, self.cols)))

    @property
    def partial_row(self):
        return self.C % self.z != 0

    @property
    def partial_slice(self):
        return self.z % 32 != 0

    def qc_smem(self, rep, early=False):
        """qc_smem_bytes of ldpc_bp_qc.cu."""
        return ((self.N + 16 if early else 0) + (self.nnz * self.z + self.N) * 4 + 16 + self.cols * 16 + self.rows * 16
                + self.nnz * 8 + 16 + 16 + rep * LOGTAB_N * 8)

    def qc_plan(self, rule, optin, early=False):
        """Log-table copies the QC kernel runs with for `rule` (0: a rule without the table), None: generic kernel."""
        for rep in ((16, 8, 1) if rule == "boxplus-phi" else (0,)):
            if self.qc_smem(rep, early) <= optin:
                return rep
        return None

    def generic_on_chip(self, optin):
        """graph_on_chip of ldpc_bp.cu (flooding schedule)."""
        return self.E <= 65535 and (self.E + self.N) * 4 + (2 * self.max_cn_deg + 2 * self.max_vn_deg + 2) * 4 + 32 <= optin


def _code(bg, k, n, m=None):
    enc_r = O.LDPC5GEncoderRef(k, n, num_bits_per_symbol=m, bg=bg)
    dec_r = O.LDPC5GDecoderRef(enc_r)
    c_, n_ = dec_r.pcm.shape
    z = enc_r.z
    rows, cols = -(-c_ // z), -(-n_ // z)
    deg = dec_r.pcm.astype(bool)
    return Code(bg, z, k, n, m, c_, n_, int(deg.nnz), rows, cols, int((enc_r.bm[:rows, :cols] >= 0).sum()),
                int(deg.sum(axis=1).max()), int(deg.sum(axis=0).max()))


def _k_per_lifting():
    """{(bg, Z): [k, ...]}: every k (base graph forced) that selects lifting size Z. BG2's k_b switches at 192, 560 and
    640 make some of these k ranges non-contiguous; the scan finds them."""
    ks = {}
    for bg, k_max in (("bg1", 8448), ("bg2", 3840)):
        for k in range(12, k_max + 1):
            ks.setdefault((bg, sel_lifting(k, bg)[0]), []).append(k)
    return ks


def _rate_points(bg, z, k, i):
    """Up to three n for (bg, Z, k): the lowest rate allowed (or the largest transmittable n), a rate near 1/2 and one
    near 0.9; `i` varies n % 4 and gives some codes an output interleaver. Returns [(n, num_bits_per_symbol)]."""
    nb, kb, lo = (68, 22, 3) if bg == "bg1" else (52, 10, 5)
    n_max = nb * z - (kb * z - k) - 2 * z                     # LDPC5GEncoder: 2Z + n <= n_ldpc - fillers
    n_min = -(-k * 20 // 19)                                   # rate <= 0.95
    pts = [(min(lo * k, n_max), None)]
    n_mid = min(2 * k + i % 4, n_max)
    m = None
    if i % 5 == 0:                                             # a few codes per base graph with an interleaver
        m = (2, 4, 6, 8)[(i // 5) % 4]
        n_mid = n_mid // m * m
    pts.append((n_mid, m))
    n_hi = -(-k * 10 // 9)
    n_hi = n_hi + (-n_hi) % 4 if i % 2 == 0 else n_hi + (n_hi % 4 == 0)
    pts.append((max(n_min, min(n_hi, n_max)), None))
    out = []
    for n, m in pts:
        if n >= n_min and all(n != o for o, _ in out):
            out.append((n, m))
    return out


def code_keys():
    """(bg, k, n, num_bits_per_symbol) of every table entry: for every (bg, Z) the largest k that selects Z (no filler
    bits) and, where it differs, the smallest (most filler bits), each at up to three rates."""
    keys = []
    for i, ((bg, z), ks) in enumerate(sorted(_k_per_lifting().items())):
        for j, k in enumerate(sorted({max(ks), min(ks)}, reverse=True)):
            keys += [(bg, k, n, m) for n, m in _rate_points(bg, z, k, 2 * i + j)]
    return keys


KEYS = code_keys()
_CODES = {}


def code(key):
    if key not in _CODES:
        _CODES[key] = _code(*key)
    return _CODES[key]


def table():
    return [code(key) for key in KEYS]


def _key_id(key):
    bg, k, n, m = key
    return f"{bg}-k{k}-n{n}" + (f"-m{m}" if m else "")


def _seed(*key):
    return zlib.crc32(repr(key).encode())


# ---- host: the table's coverage and the oracle encoder ---------------------------------------------------------------
def test_table_covers_every_lifting_size():
    """The table reaches all 102 (bg, Z) pairs, Zb = 1 ... 12, idle lanes, full and partial slices and last block rows,
    launches with fewer warp groups than the planner's 24 / Zb, both channel-LLR loads, every interleaver order, filler
    bits, both rate limits, and (by the planner's rule on an H100) every kernel variant."""
    tab = table()
    lifting = sorted({z for s in O._S_VAL for z in s})
    assert len(lifting) == 51
    assert {(c.bg, c.z) for c in tab} == {(bg, z) for bg in ("bg1", "bg2") for z in lifting}
    assert {c.zb for c in tab} == set(range(1, 13))
    assert any(c.z < 32 for c in tab) and any(c.z % 32 == 0 for c in tab) and any(c.z > 32 and c.z % 32 for c in tab)
    assert any(c.g_launch < c.g_plan for c in tab)
    for bg in ("bg1", "bg2"):
        sub = [c for c in tab if c.bg == bg]
        assert any(c.partial_row for c in sub) and any(not c.partial_row for c in sub)
        assert any(c.n % 4 == 0 for c in sub) and any(c.n % 4 != 0 for c in sub)
        assert {c.m for c in sub} >= {None, 2, 4, 6, 8}
        assert any(c.k < c.z * (22 if bg == "bg1" else 10) for c in sub)          # filler bits
        rates = [c.k / c.n for c in sub]
        assert min(rates) == pytest.approx(1 / 3 if bg == "bg1" else 1 / 5) and max(rates) > 0.85
    # the planner's fallback: some large low-rate codes leave the QC kernel, every high-rate code stays on it
    assert any(c.qc_plan("boxplus-phi", SMEM_OPTIN_H100) is None for c in tab)
    assert all(c.qc_plan("boxplus-phi", SMEM_OPTIN_H100) is not None for c in tab if c.k / c.n > 0.85)
    assert {c.qc_plan("boxplus-phi", SMEM_OPTIN_H100) for c in tab} >= {16, 8, 1}
    assert any(not c.generic_on_chip(SMEM_OPTIN_H100) for c in tab) and any(c.generic_on_chip(SMEM_OPTIN_H100) for c in tab)


def test_oracle_encoder_codewords_satisfy_parity_checks():
    """H c = 0 for the oracle encoder's full codewords on a sample of the table: this guards the oracle itself."""
    sample = {}
    for c in table():
        if c.z in (2, 3, 15, 26, 36, 112, 208, 240, 352, 384):
            sample.setdefault((c.bg, c.z, c.k), c)
    assert len(sample) >= 30
    for (bg, z, k), c in sample.items():
        enc_r = O.LDPC5GEncoderRef(k, c.n, bg=bg)
        rng = np.random.default_rng(_seed(bg, z, k))
        u = rng.integers(0, 2, (5, k))
        u[0], u[1] = 0, 1
        cw = enc_r.encode_full(u)
        assert cw.shape == (5, enc_r.n_ldpc)
        assert not ((enc_r.pcm @ cw.T) % 2).any(), (bg, z, k)
        assert np.array_equal(cw[:, :k], u) and not cw[:, k:enc_r.k_ldpc].any()
        assert not cw[0].any()


# ---- device ------------------------------------------------------------------------------------------------------------
def _optin():
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rate_matched(enc_r, u, c_full):
    """enc_r(u) with the full codewords c_full = enc_r.encode_full(u) solved once for every n of a (bg, Z, k)."""
    enc_r.encode_full = lambda _u: c_full
    return enc_r(u)


def _groups():
    g = {}
    for c in table():
        g.setdefault((c.bg, c.z, c.k), []).append(c)
    return g


def _encoders(bg, k, codes):
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder
    return [(c, O.LDPC5GEncoderRef(k, c.n, num_bits_per_symbol=c.m, bg=bg),
             LDPC5GEncoder(k, c.n, num_bits_per_symbol=c.m, bg=bg)) for c in codes]


@pytest.mark.gpu
@pytest.mark.parametrize("bg", ["bg1", "bg2"])
def test_encoder_every_lifting_size(cuda_device, bg):
    """Every table entry, batches of 1, 31, 33 and 97 codewords (tails of 1 ... 31 in the last 32-codeword group), with
    all-zero and all-one information words among them."""
    for (bg_, z, k), codes in _groups().items():
        if bg_ != bg:
            continue
        rng = np.random.default_rng(_seed(bg, z, k))
        u = rng.integers(0, 2, (97, k))
        u[40], u[95], u[96] = 0, 0, 1
        c_full = O.LDPC5GEncoderRef(k, codes[0].n, bg=bg).encode_full(u)
        u_d = torch.from_numpy(u.astype(np.float32)).to(cuda_device)
        for c, enc_r, enc in _encoders(bg, k, codes):
            ref = _rate_matched(enc_r, u, c_full)
            assert enc.z == z and ref.shape == (97, c.n)
            for b in (1, 31, 33, 97):
                out = enc(u_d[97 - b:]).cpu().numpy()
                assert np.array_equal(out, ref[97 - b:]), (c.id, b)


@pytest.mark.gpu
@pytest.mark.parametrize("bg", ["bg1", "bg2"])
def test_encoder_grid_stride(cuda_device, bg):
    """The smallest and largest n of a base graph with more 32-codeword groups than the grid holds (at most 2048 / 512 = 4
    CTAs per SM), so that CTAs loop over groups. The 97 distinct information words repeat with a period prime to 32."""
    sub = [c for c in table() if c.bg == bg]
    batch = 32 * 4 * _sms() + 33
    for c in (min(sub, key=lambda c: c.n), max(sub, key=lambda c: c.n)):
        rng = np.random.default_rng(_seed(c.id))
        u = rng.integers(0, 2, (97, c.k))
        u[3], u[4] = 0, 1
        (_, enc_r, enc), = _encoders(bg, c.k, [c])
        ref = torch.from_numpy(enc_r(u)).to(cuda_device)
        rows = torch.arange(batch, device=cuda_device) % 97
        out = enc(torch.from_numpy(u.astype(np.float32)).to(cuda_device)[rows])
        assert torch.equal(out, ref[rows]), c.id
        del out


def _llr(c, code, rng):
    """BPSK over AWGN with Eb/N0 spread over -1.5 ... 6.5 dB across the batch: logits log p(1)/p(0)."""
    ebno = np.linspace(-1.5, 6.5, c.shape[0])[:, None]
    no = 1.0 / (10 ** (ebno / 10) * (code.k / code.n))
    y = (2.0 * c - 1.0) + rng.normal(size=c.shape) * np.sqrt(no / 2)
    return (4 * y / no).astype(np.float32)


_FULL = {}


def _full_codewords(code, batch):
    """Information words and oracle full codewords of a (bg, Z, k), solved once for all its table entries."""
    key = code.group + (batch,)
    if key not in _FULL:
        _FULL.clear()                                      # the table is walked group by group
        u = np.random.default_rng(_seed("dec", *key)).integers(0, 2, (batch, code.k))
        _FULL[key] = u, O.LDPC5GEncoderRef(code.k, code.n, bg=code.bg).encode_full(u)
    return _FULL[key]


class _Case:
    """Codewords, channel logits and oracle decodes (every rule, soft and hard) of one table entry."""

    def __init__(self, code, batch=DEC_BATCH):
        from bench import host_cores
        self.code = code
        self.enc_r = O.LDPC5GEncoderRef(code.k, code.n, num_bits_per_symbol=code.m, bg=code.bg)
        self.cw = _rate_matched(self.enc_r, *_full_codewords(code, batch))
        self.llr = _llr(self.cw, code, np.random.default_rng(_seed("llr", code.id, batch)))
        self.threads = host_cores()[0]
        self._ref = {}

    def ref(self, rule, hard):
        """(output, v2c state) of the oracle: hard info bits, or soft logits of the transmitted positions."""
        if (rule, hard) not in self._ref:
            r = O.LDPC5GDecoderRef(self.enc_r, cn_update=rule, hard_out=hard, return_infobits=hard, num_iter=NUM_ITER,
                                   return_state=True)
            self._ref[rule, hard] = r(self.llr, math_mode=1, order="kernel", num_threads=self.threads)
        return self._ref[rule, hard]


def _decoder(code, qc, enc=None, **kw):
    """LDPC5GDecoder of a table entry; `qc=False` keeps it on the generic kernel (SB_LDPC_DISABLE_QC=1)."""
    import os
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    if enc is None:
        enc = LDPC5GEncoder(code.k, code.n, num_bits_per_symbol=code.m, bg=code.bg)
    old = os.environ.get("SB_LDPC_DISABLE_QC")
    os.environ["SB_LDPC_DISABLE_QC"] = "0" if qc else "1"
    try:
        dec = LDPC5GDecoder(enc, **kw)
    finally:
        if old is None:
            del os.environ["SB_LDPC_DISABLE_QC"]
        else:
            os.environ["SB_LDPC_DISABLE_QC"] = old
    assert dec._graph.is_qc() == qc
    return dec


@pytest.mark.gpu
@pytest.mark.parametrize("key", KEYS, ids=_key_id)
def test_decoder_every_lifting_size(cuda_device, key):
    """Every table entry: the default path (the QC kernel where the code fits on chip) with all four rules, the generic
    kernel with boxplus-phi and min-sum, soft and hard output and the v2c state; early termination wherever the QC
    kernel runs. Eb/N0 spreads over the launch, so converged codewords run the voting CN pass of boxplus-phi while
    others in the same launch do not."""
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder
    from sionna_b200._lib import SbError
    code_ = code(key)
    case = _Case(code_)
    x = torch.from_numpy(case.llr).to(cuda_device)
    err = ((case.ref("boxplus-phi", False)[0] > 0) != (case.cw > 0)).any(axis=1)
    assert err.any() and not err.all(), code_.id          # converged and non-converged codewords in the same launch

    enc = LDPC5GEncoder(code_.k, code_.n, num_bits_per_symbol=code_.m, bg=code_.bg)
    soft = {}
    for qc, rules in ((True, RULES), (False, ["boxplus-phi", "minsum"])):
        for rule in rules:
            for hard in (False, True):
                dec = _decoder(code_, qc, enc, cn_update=rule, hard_out=hard, return_infobits=hard, num_iter=NUM_ITER,
                               return_state=True)
                out, st = dec(x)
                ref, ref_st = case.ref(rule, hard)
                where = (code_.id, "qc" if qc else "generic", rule, "hard" if hard else "soft")
                assert np.array_equal(out.cpu().numpy(), ref), where
                assert np.array_equal(st.cpu().numpy(), ref_st), where
                if qc and not hard:
                    soft[rule] = dec

    # early termination: an early_stop decode runs only on the QC kernel (the generic one refuses it). The syndrome is
    # checked before iterations 1 ... NUM_ITER - 2, so a codeword that first satisfies every check later runs them all.
    optin = _optin()
    stopped = []
    for rule in RULES:
        dec = _decoder(code_, True, enc, cn_update=rule, hard_out=False, return_infobits=False, num_iter=NUM_ITER,
                       early_stop=True)
        if code_.qc_plan(rule, optin, early=True) is None:
            with pytest.raises(SbError, match="early termination needs"):
                dec(x)
            continue
        y = dec(x).cpu().numpy()
        iters = dec.num_iter_run.cpu().numpy()
        assert iters.min() >= 2 and iters.max() <= NUM_ITER, (code_.id, rule)
        for v in np.unique(iters):
            sel = np.flatnonzero(iters == v)
            fixed = soft[rule](x[sel], num_iter=int(v))[0].cpu().numpy()
            assert np.array_equal(y[sel], fixed), (code_.id, rule, v)
        full = iters == NUM_ITER
        assert full.any(), (code_.id, rule)
        assert np.array_equal(y[full], case.ref(rule, False)[0][full]), (code_.id, rule)
        stopped.append(not full.all())
    assert not stopped or any(stopped), code_.id           # some codeword stopped early under some rule


_QC_NAME = re.compile(r"ldpc_bp_qc_kernel(?:<[^,>]*,\s*(?:\(int\))?(\d+)|ILi\d+ELi(\d+)E)")
_GENERIC_NAME = re.compile(r"ldpc_bp_kernel(?:<[^,>]*,\s*(true|false)|ILi\d+ELb([01])E)")


def _kernel_kind(name):
    """'qc16', 'qc8', 'qc1', 'generic-smem' or 'generic-ws' from a decoder kernel's (demangled or mangled) name."""
    m = _QC_NAME.search(name)
    if m:
        return f"qc{m.group(1) or m.group(2)}"
    m = _GENERIC_NAME.search(name)
    if m:
        return "generic-smem" if (m.group(1) or m.group(2)) in ("true", "1") else "generic-ws"
    return None


def planned_kernels(code, optin):
    """Kernel kinds the planners choose for a boxplus-phi decode with the QC path allowed and with it disabled."""
    rep = code.qc_plan("boxplus-phi", optin)
    generic = "generic-smem" if code.generic_on_chip(optin) else "generic-ws"
    return (generic if rep is None else f"qc{rep}"), generic


def traced_kernels(codes, device):
    """For every code, the decoder kernel that ran for a 2-codeword boxplus-phi decode with the QC path allowed and
    with it disabled, read from the kernel names of one CUDA trace, and `on_chip` of the generic decoder."""
    from torch.profiler import profile, ProfilerActivity
    decs = [(_decoder(c, True, num_iter=1), _decoder(c, False, num_iter=1)) for c in codes]
    xs = [torch.zeros(2, c.n, device=device) for c in codes]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for (dq, dg), x in zip(decs, xs):
            dq(x)
            dg(x)
        torch.cuda.synchronize()
    kernels = sorted((e.time_range.start, _kernel_kind(e.name)) for e in prof.events()
                     if e.device_type == torch.autograd.DeviceType.CUDA and _kernel_kind(e.name))
    kinds = [k for _, k in kernels]
    assert len(kinds) == 2 * len(codes), len(kinds)
    return [(q, g, dg.on_chip) for q, g, (_, dg) in zip(kinds[0::2], kinds[1::2], decs)]


@pytest.mark.gpu
def test_kernel_selection_every_lifting_size(cuda_device):
    """The kernel that ran for every table entry equals the planners' choice restated from qc_smem_bytes
    (ldpc_bp_qc.cu) and graph_on_chip (ldpc_bp.cu) against the device's opt-in shared memory; large low-rate codes leave
    the QC kernel, and the log-table copies drop from 16 to 8 to 1 as the messages grow."""
    optin = _optin()
    tab = table()
    ran = traced_kernels(tab, cuda_device)
    for c, (q, g, on_chip) in zip(tab, ran):
        assert (q, g) == planned_kernels(c, optin), c.id
        assert on_chip == (g == "generic-smem"), c.id
    default = {q for q, _, _ in ran}
    assert default == {"qc16", "qc8", "qc1", "generic-smem", "generic-ws"}, default    # large low-rate codes fall back
    assert {g for _, g, _ in ran} == {"generic-smem", "generic-ws"}


# ---- input-pointer and batch edges ------------------------------------------------------------------------------------
EDGE_CODES = [("bg1", 44, 88), ("bg1", 8448, 9392), ("bg2", 12, 24), ("bg2", 3840, 4268), ("bg1", 4576, 5088)]


@pytest.mark.gpu
@pytest.mark.parametrize("qc", [True, False], ids=["qc", "generic"])
@pytest.mark.parametrize("bg, k, n", EDGE_CODES)
def test_misaligned_input_and_batch_edges(cuda_device, bg, k, n, qc):
    """The same logits as a view at storage offset 1, 2 and 3 floats of a flat buffer (contiguous, not 16-byte aligned:
    the plain load instead of the bulk copy) give the same bits as the aligned tensor; batches of 1 and of more than 3
    codewords per SM (each persistent CTA decodes several codewords) equal the oracle."""
    c = _code(bg, k, n)
    assert c.n % 4 == 0
    batch = 3 * _sms() + 7
    case = _Case(c, batch)
    x = torch.from_numpy(case.llr).to(cuda_device)
    for rule in ("boxplus-phi", "minsum"):
        ref = case.ref(rule, False)[0]
        dec = _decoder(c, qc, cn_update=rule, hard_out=False, return_infobits=False, num_iter=NUM_ITER)
        out = dec(x).cpu().numpy()
        assert np.array_equal(out, ref), (c.id, rule)
        assert np.array_equal(dec(x[5:6]).cpu().numpy(), ref[5:6]), (c.id, rule)
        buf = torch.empty(batch * n + 4, device=cuda_device)
        for off in (1, 2, 3):
            view = buf[off:off + batch * n].view(batch, n)
            view.copy_(x)
            assert view.is_contiguous() and view.data_ptr() % 16 != 0
            assert np.array_equal(dec(view).cpu().numpy(), out), (c.id, rule, off)
