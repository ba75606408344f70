"""The turbo and BCJR decoders (csrc/conv.cu) against float64 in every state count and storage plan.

The kernels' shape depends on the state count ns (G = 32 / ns codewords per warp below 32 states), on where alpha and
the turbo extrinsic buffer live (shared memory or the workspace) and on the branch-metric table chunk ch. The plan is
restated here from its definition and checked against the library's workspace sizes on the CPU; the GPU tests decode
at the last length of each regime and the first of the next, for every ns, and compare with oracle/turbo.py and
oracle/conv.py in float64, errors relative to each codeword's rms LLR: soft outputs within 2x (rms) / 4x (max) of the
float32 oracle's error (parity.envelope) and within a fixed multiple of float32 eps, hard outputs equal to float64's
wherever |LLR| exceeds 4x the oracle's error. The decoder's demultiplexing table is checked against the oracle's
depuncturing, so that neither these tests nor the composed loop of test_turbo_gpu.py can share a wrong table with the
kernel; turbo3gpp_perm's pruning is checked against oracle.turbo.qpp_perm for every k. Both read the same QPP table,
whose structure test_oracle_turbo.py checks."""
import itertools
import math

import numpy as np
import pytest
import torch

from oracle import conv as C
from oracle import turbo as O
from oracle.parity import envelope, rel_err

# ---- the plan, restated (conv.cu: warp_plan, turbo_plan, turbo_syms, workspace_bytes) ---------------------------------
WARPS, TABLE_FLOATS, ON_CHIP = 4, 2048, 48 * 1024
STATES = (2, 4, 8, 16, 32, 64, 128, 256)
REGIMES = ("both on chip", "alpha off chip", "both off chip")
# turbo component codes: constraint_length 3 ... 6 for 4 ... 32 states, these polynomials for the others
GEN_POLY = {2: ("11", "10"), 64: ("1011011", "1111001"), 128: ("11100101", "10011111"),
            256: ("110101001", "101110111")}
# BCJR codes: rate 1/2 with 2, 4 and 8 states, rate 1/3 with 16, rate 1/4 with 64
BCJR_CODES = {"r2s2": ("11", "10"), "r2s4": ("101", "111"), "r2s8": ("1101", "1011"),
              "r3s16": ("10101", "11011", "11111"), "r4s64": ("1011011", "1111001", "1100101", "1110111")}


def group(ns):
    return 32 // ns if ns < 32 else 1


def chunk(ns, conv_n):
    """Steps per branch-metric table chunk; the table has 2^conv_n metrics and the prior per step."""
    return max(1, min(32, TABLE_FLOATS // (group(ns) * ((1 << conv_n) + 1))))


def turbo_syms(ns, k, terminate):
    return k + (int(math.log2(ns)) if terminate else 0)


def turbo_plan(ns, k, terminate):
    """(alpha bytes, extrinsic bytes) per codeword, whether each is on chip, T and ch."""
    G, T = group(ns), turbo_syms(ns, k, terminate)
    alpha, ext = T * ns * 4, k * 4
    return dict(alpha=alpha, ext=ext, alpha_chip=WARPS * G * alpha <= ON_CHIP, ext_chip=WARPS * G * ext <= ON_CHIP,
                T=T, ch=chunk(ns, 2))


def regime(ns, k, terminate):
    p = turbo_plan(ns, k, terminate)
    assert not (p["alpha_chip"] and not p["ext_chip"]), "alpha is never smaller than the extrinsics"
    return 0 if p["alpha_chip"] else 1 if p["ext_chip"] else 2


def rows(ns, batch):
    per_cta = WARPS * group(ns)
    return -(-batch // per_cta) * per_cta


def turbo_ws(ns, k, terminate, batch):
    p = turbo_plan(ns, k, terminate)
    return rows(ns, batch) * ((0 if p["alpha_chip"] else p["alpha"]) + (0 if p["ext_chip"] else p["ext"]))


def bcjr_ws(ns, num_syms, batch):
    alpha = num_syms * ns * 4
    return 0 if WARPS * group(ns) * alpha <= ON_CHIP else rows(ns, batch) * alpha


def boundaries(ns, terminate, k_max=8000):
    """Last k of every regime but the final one, as k grows from 1."""
    out, prev = [], regime(ns, 1, terminate)
    for k in range(2, k_max):
        r = regime(ns, k, terminate)
        if r != prev:
            assert r == prev + 1
            out.append(k - 1)
            prev = r
    return out


# ---- the cases --------------------------------------------------------------------------------------------------------
def _turbo_cases():
    """(ns, k, terminate, algorithm, rate, num_iter, interleaver, batch): the last length of each regime and the first
    of the next for every ns, algorithm, rate, iterations and interleaver cycling; then a random interleaver beyond
    6144, ten iterations, T < ch, and a batch of one."""
    algs = itertools.cycle(("map", "log", "maxlog", "log", "map"))
    rates = itertools.cycle((1 / 3, 1 / 2, 1 / 2))
    iters = itertools.cycle((2, 1, 6, 2))
    ils = itertools.cycle(("3GPP", "3GPP", "random", "3GPP", "3GPP", "3GPP", "random"))
    terms = itertools.cycle((True, False, False))
    cases = []
    for ns in STATES:
        per_cta = WARPS * group(ns)
        for b, term in zip(range(2), terms):
            k_last = boundaries(ns, term)[b]
            for k in (k_last, k_last + 1):
                alg, it = next(algs), next(iters)
                if alg == "maxlog" and k > 1000:
                    it = 1                      # beyond, float32 maxlog drifts from float64 (see test_turbo_envelope)
                big = k * ns * it > 600_000                      # keep the numpy oracle's time modest
                batch = per_cta + (1 if big else per_cta // 2 + 1)
                if b == 0:
                    batch += per_cta
                cases.append((ns, k, term, alg, next(rates), it, next(ils), batch))
    cases += [(8, 10000, False, "log", 1 / 3, 2, "random", 5),          # beyond the 3GPP interleaver
              (4, 200, True, "map", 1 / 2, 10, "3GPP", 35),             # ten iterations
              (2, 20, False, "maxlog", 1 / 3, 6, "random", 77),         # T < ch = 25
              (4, 27, True, "log", 1 / 3, 2, "3GPP", 29),               # T < ch = 32
              (16, 700, True, "log", 1 / 3, 2, "3GPP", 1)]              # one codeword
    return cases


TURBO_CASES = _turbo_cases()


def _bcjr_cases():
    """(code, rsc, terminate, algorithm, prior, k, batch): alpha in the workspace (T > 96, or 48 at 64 states), every
    algorithm, rate 1/2, 1/3 and 1/4, with and without a prior, batches with a partial G-codeword group and CTA."""
    cases = []
    algs = itertools.cycle(("log", "map", "maxlog", "log"))
    flags = itertools.cycle(((False, True, True), (True, False, False), (True, True, True), (False, False, False)))
    for code, k in (("r2s2", 300), ("r2s4", 97), ("r2s8", 1000), ("r3s16", 400), ("r4s64", 129)):
        ns = 2 ** (len(BCJR_CODES[code][0]) - 1)
        per_cta = WARPS * group(ns)
        for batch in (2 * per_cta + group(ns) // 2 + 1, per_cta - 1 if per_cta > 1 else 3):
            rsc, term, prior = next(flags)
            cases.append((code, rsc, term, next(algs), prior, k, batch))
    return cases


BCJR_CASES = _bcjr_cases()


def _id(case):
    return "-".join(f"{v:.2f}" if isinstance(v, float) else str(v) for v in case)


# ---- CPU: the plan and the host tables --------------------------------------------------------------------------------
def test_regime_table():
    """The regimes of terminated codes as DESIGN §3.12 states them."""
    table = {2: [95, 192], 4: [94, 384], 8: [93, 768], 16: [92, 1536], 32: [91, 3072], 64: [42, 3072],
             128: [17, 3072], 256: [4, 3072]}
    for ns, b in table.items():
        assert boundaries(ns, True) == b, ns


def test_workspace_sizes(sb_lib):
    """sb_turbo_workspace_bytes / sb_bcjr_workspace_bytes equal the restated off-chip parts, batches rounded up to
    whole CTAs, at and either side of every regime boundary."""
    for ns, term in itertools.product(STATES, (False, True)):
        per_cta = WARPS * group(ns)
        ks = {1, 2, 40, 1000, 6144, 10000}
        for b in boundaries(ns, term):
            ks |= {b - 1, b, b + 1, b + 2}
        for k, batch in itertools.product(sorted(ks), (0, 1, per_cta - 1, per_cta, per_cta + 1, 1001)):
            assert sb_lib.sb_turbo_workspace_bytes(batch, k, int(term), ns) == turbo_ws(ns, k, term, batch), \
                (ns, k, term, batch)
        last_on = ON_CHIP // (WARPS * group(ns) * ns * 4)                  # longest trellis with alpha on chip
        for T, batch in itertools.product((1, 2, last_on - 1, last_on, last_on + 1, 5000),
                                          (1, per_cta - 1, per_cta + 1, 777)):
            assert sb_lib.sb_bcjr_workspace_bytes(batch, T, ns) == bcjr_ws(ns, T, batch), (ns, T, batch)
            assert (bcjr_ws(ns, T, batch) == 0) == (T <= last_on)


def test_cases_cover_every_regime():
    """Every state count decodes in each regime it reaches, at a boundary's both sides; the chunk tails are hit."""
    for ns in STATES:
        reach = {regime(ns, k, t) for k in range(1, 8000, 7) for t in (False, True)}
        got = {regime(ns, k, t) for n, k, t, *_ in TURBO_CASES if n == ns}
        assert got == reach == {0, 1, 2}, ns
    for ns, term in itertools.product(STATES, (False, True)):
        assert len(boundaries(ns, term)) == 2
    tails = [turbo_plan(ns, k, t)["T"] % turbo_plan(ns, k, t)["ch"] for ns, k, t, *_ in TURBO_CASES]
    assert sum(x != 0 for x in tails) >= len(tails) // 2
    assert any(turbo_plan(ns, k, t)["T"] < turbo_plan(ns, k, t)["ch"] for ns, k, t, *_ in TURBO_CASES if ns == 2)
    assert any(turbo_plan(ns, k, t)["T"] < turbo_plan(ns, k, t)["ch"] for ns, k, t, *_ in TURBO_CASES if ns == 4)
    assert {c[3] for c in TURBO_CASES} == {"map", "log", "maxlog"} and {c[4] for c in TURBO_CASES} == {1 / 3, 1 / 2}
    assert {c[5] for c in TURBO_CASES} >= {1, 2, 6, 10} and {c[6] for c in TURBO_CASES} == {"3GPP", "random"}
    assert any(c[1] > 6144 and c[6] == "random" for c in TURBO_CASES)
    assert any(c[7] == 1 for c in TURBO_CASES)
    assert all(c[7] % (WARPS * group(c[0])) for c in TURBO_CASES if c[7] > 1)
    for code, rsc, term, alg, prior, k, batch in BCJR_CASES:
        g = BCJR_CODES[code]
        ns = 2 ** (len(g[0]) - 1)
        assert bcjr_ws(ns, k + (len(g[0]) - 1 if term else 0), batch) > 0, code
    assert {c[3] for c in BCJR_CASES} == {"map", "log", "maxlog"} and {c[4] for c in BCJR_CASES} == {False, True}


@pytest.mark.parametrize("mu", range(1, 9))
def test_demux_table_equals_depuncture(sb_lib, monkeypatch, mu):
    """The decoder's demultiplexing table (turbo_layout plus decoder 2's systematic positions through pi) reads the
    positions oracle.turbo.depuncture assigns, for both rates, terminated or not, 3GPP and random interleavers."""
    from sionna_b200.phy.fec.turbo import decoding
    monkeypatch.setattr(decoding, "dev_i32", lambda a: np.ascontiguousarray(a, np.int32))
    gen = ("1" * (mu + 1), "1" * mu + "0")
    for rate, term, k, il in itertools.product((1 / 3, 1 / 2), (False, True), (40, 41, 97, 112, 6144),
                                               ("3GPP", "random")):
        dec = decoding.TurboDecoder(gen_poly=gen, rate=rate, terminate=term, interleaver=il)
        n = len(O.encode(np.zeros((1, k), np.int64), gen, np.arange(k), rate, term)[0])
        dec.build((1, n))
        dec._prepare()
        perm = decoding.interleaver_perm(dec.internal_interleaver, k)
        y1, y2 = O.depuncture(np.arange(1, n + 1)[None], k, mu, perm, rate, term)
        assert np.array_equal(dec._demux + 1, np.concatenate([y1[0], y2[0]])), (rate, term, k, il)


def test_turbo3gpp_perm_equals_qpp():
    """The pruning of the QPP permutation to k bits, for every k; the table is shared with the oracle."""
    from sionna_b200.phy.fec.interleaving import qpp_table, turbo3gpp_perm
    tab = qpp_table()
    for k in range(1, 6145):
        assert np.array_equal(turbo3gpp_perm(k), O.qpp_perm(k, tab)), k


# ---- GPU: turbo decoder -----------------------------------------------------------------------------------------------
SNR = (-1.0, 1.5, 6.0)          # dB per row, cycling: low, mid, and high enough that the +-20 extrinsic clip binds


def _noisy(x, rng):
    snr = np.array(SNR)[np.arange(len(x)) % len(SNR)]
    no = 10 ** (-snr / 10)[:, None]
    return (2 / no * ((2 * x - 1) + rng.normal(size=x.shape) * np.sqrt(no))).astype(np.float32)


def _gpu(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


EPS = float(np.finfo(np.float32).eps)
# The float32 oracle's rms error, relative to each codeword's rms LLR, must stay below F32_DRIFT: beyond it the oracle
# has drifted off float64's trajectory (maxlog over several iterations at long k does) and 2x its error bounds nothing.
F32_DRIFT = 1e-3
# The float32 oracle keeps alpha and beta unnormalised, so its error grows with the trellis length; the kernel
# normalises them every step. So the kernel's own error, relative to each codeword's rms LLR, is also held to a fixed
# (rms, max) multiple of float32 eps per algorithm, which binds at every length. Measured on an H100 (worst over the
# cases): map / log 4.2 / 21 eps. maxlog 20 / 232 eps (16 states, k = 92, 2 iterations): a maxlog extrinsic follows
# whichever path wins each max, so where two paths nearly tie a rounding difference switches the winner and is
# passed on, amplified, through the iterations (the float32 oracle drifts 10x further in maxlog too); one maxlog
# BCJR pass stays at 1.2 / 6.7 eps.
KERNEL_BAR = {"map": (8 * EPS, 64 * EPS), "log": (8 * EPS, 64 * EPS), "maxlog": (64 * EPS, 512 * EPS)}


def _check_soft(what, alg, got, f32, ref, floor):
    """Errors relative to each codeword's rms LLR, so the low-SNR rows weigh as much as the high ones: the float32
    oracle close to float64, the kernel within 2x / 4x of the oracle's error and within KERNEL_BAR[alg]."""
    assert np.all(np.isfinite(got)), what
    drift = float(np.sqrt(np.mean(rel_err(f32, ref, axis=-1) ** 2)))
    assert drift < F32_DRIFT, f"{what}: the float32 oracle is {drift:.1e} off float64, its envelope bounds nothing"
    bad = envelope(what, got, f32, ref, (2.0, 4.0), floor=floor, axis=-1)
    assert not bad, bad
    e = rel_err(got, ref, axis=-1)
    rms, mx = float(np.sqrt(np.mean(e ** 2))), float(e.max())
    bar = KERNEL_BAR[alg]
    print(f"{what}: kernel rms {rms / EPS:.2f} eps max {mx / EPS:.2f} eps (bar {bar[0] / EPS:g} / {bar[1] / EPS:g} eps)")
    assert rms <= bar[0] and mx <= bar[1], f"{what}: kernel error beyond the fixed bar"


@pytest.mark.gpu
@pytest.mark.parametrize("ns,k,terminate,alg,rate,num_iter,il,batch", TURBO_CASES, ids=map(_id, TURBO_CASES))
def test_turbo_envelope(cuda_device, sb_lib, ns, k, terminate, alg, rate, num_iter, il, batch):
    from sionna_b200.phy.fec.turbo import TurboDecoder
    from sionna_b200.phy.fec.turbo.encoding import interleaver_perm
    code = dict(gen_poly=GEN_POLY[ns]) if ns in GEN_POLY else dict(constraint_length=int(math.log2(ns)) + 1)
    soft = TurboDecoder(**code, rate=rate, interleaver=il, terminate=terminate, num_iter=num_iter, hard_out=False,
                        algorithm=alg)
    hard = TurboDecoder(**code, rate=rate, interleaver=il, terminate=terminate, num_iter=num_iter, hard_out=True,
                        algorithm=alg)
    hard.internal_interleaver = soft.internal_interleaver
    assert soft.trellis.ns == ns
    perm = interleaver_perm(soft.internal_interleaver, k)
    rng = np.random.default_rng(ns * 10007 + k)
    u = rng.integers(0, 2, (batch, k))
    y = _noisy(O.encode(u, soft.gen_poly, perm, rate, terminate), rng)

    p = turbo_plan(ns, k, terminate)
    ws = sb_lib.sb_turbo_workspace_bytes(batch, k, int(terminate), ns)
    assert ws == turbo_ws(ns, k, terminate, batch)
    assert (ws == 0) == (regime(ns, k, terminate) == 0)
    what = (f"turbo ns={ns} k={k} T={p['T']} ch={p['ch']} [{REGIMES[regime(ns, k, terminate)]}] {alg} "
            f"rate={rate:.2f} term={terminate} it={num_iter} {il} batch={batch}")

    got = soft(_gpu(y)).cpu().numpy().astype(np.float64)
    dec = hard(_gpu(y)).cpu().numpy()
    ref, peak = O.decode(y.astype(np.float64), soft.gen_poly, perm, rate, terminate, num_iter,
                         "log" if alg == "map" else alg, np.float64, return_peak_ext=True)
    f32 = O.decode(y, soft.gen_poly, perm, rate, terminate, num_iter, alg, np.float32).astype(np.float64)
    if batch >= len(SNR):
        assert peak.max() > 20, f"{what}: the extrinsic clip did not bind"
    assert np.array_equal(dec, (got > 0).astype(np.float32)), what
    _check_soft(what, alg, got, f32, ref, (1e-7, 1e-6))
    sure = np.abs(ref) > 4 * np.abs(f32 - ref).max()
    assert np.array_equal((got > 0)[sure], (ref > 0)[sure]), what


# ---- GPU: BCJR with alpha in the workspace ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("code,rsc,terminate,alg,prior,k,batch", BCJR_CASES, ids=map(_id, BCJR_CASES))
def test_bcjr_off_chip(cuda_device, sb_lib, code, rsc, terminate, alg, prior, k, batch):
    from sionna_b200.phy.fec.conv import BCJRDecoder
    g = BCJR_CODES[code]
    ns, n = 2 ** (len(g[0]) - 1), len(g)
    rng = np.random.default_rng(ns * 31 + k + batch)
    u = rng.integers(0, 2, (batch, k))
    x = C.encode(u, g, rsc, terminate)
    T = x.shape[1] // n
    assert sb_lib.sb_bcjr_workspace_bytes(batch, T, ns) == bcjr_ws(ns, T, batch) > 0
    llr = _noisy(x, rng)
    la = (rng.normal(size=(batch, T)) * 2).astype(np.float32) if prior else None
    args = dict(gen_poly=g, rsc=rsc, terminate=terminate, algorithm=alg)
    a = None if la is None else _gpu(la)
    got = BCJRDecoder(**args, hard_out=False)(_gpu(llr), llr_a=a).cpu().numpy().astype(np.float64)
    hard = BCJRDecoder(**args, hard_out=True)(_gpu(llr), llr_a=a).cpu().numpy()
    ref = C.bcjr(llr.astype(np.float64), g, rsc, terminate, "log" if alg == "map" else alg,
                 None if la is None else la.astype(np.float64))[:, :k]
    f32 = C.bcjr(llr, g, rsc, terminate, alg, la, dtype=np.float32)[:, :k].astype(np.float64)
    what = f"bcjr ns={ns} rate=1/{n} k={k} T={T} {alg} rsc={rsc} term={terminate} prior={prior} batch={batch}"
    _check_soft(what, alg, got, f32, ref, (1e-6, 1e-5))
    err = np.abs(f32 - ref)
    sure = np.abs(ref) > 4 * max(float(err.max()), 1e-5 * float(np.sqrt(np.mean(ref ** 2))))
    assert np.array_equal(hard[sure], (ref[sure] > 0).astype(np.float32)), what
