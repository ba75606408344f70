"""The unfused receive front-end against float64 references, over a table of pilot layouts: resource-grid mapping
(sb_rg_map), the grid gathers (sb_gather_rows: RemoveNulledSubcarriers, ResourceGridDemapper, nearest-neighbour
interpolation), LS estimation at the pilots (sb_ls_at_pilots), PUSCH CDM de-spreading (sb_pusch_ls_combine) and linear
interpolation (sb_interp_lin), driven by ResourceGridMapper, LSChannelEstimator, NearestNeighborInterpolator,
LinearInterpolator and PUSCHLSChannelEstimator. Their h_hat / err_var feed every detector that does not take the fused
front-end.

Pure copies (mapping, gathers, nearest-neighbour interpolation of the kernel's own pilot estimates) must be bit-exact.
Arithmetic is held to oracle.parity.envelope: the kernel's rms and max error against the float64 evaluation
(oracle.ofdm.ls_estimate -> oracle.nr.pusch_ls_combine -> lin_interp / nn_interp) must be at most 2x and 4x the error
of the same formula evaluated in complex64 / float32, unless BARS names an exception. Errors are relative to the rms of
each (frame, rx, antenna, tx, stream) row of the float64 output, and the yardstick is floored at 2^-24 of that scale.
Every comparison prints its ratios (pytest -s).

The table (`table()`, checked on the CPU by test_table_covers_every_branch) holds the Kronecker grids, multi-UE and
multi-stream grids, guard carriers and DC nulls, custom pilot patterns and every PUSCH DMRS configuration. Between them
they reach every branch of LinearInterpolator's index tables: a pilot symbol with one non-zero pilot, zero pilots
skipped while bracketing, pilots on the first / last subcarrier and OFDM symbol with extrapolation beyond them, streams
with different masks and different numbers of pilot symbols, and negative extrapolated error variances (the kernel's
floor). They also reach the launch edges: S = 1, F = 1, F > 256 (a thread loops over subcarriers) and more rows than the
grid-stride kernels launch CTAs for.
"""
import dataclasses
import functools
import zlib

import numpy as np
import pytest
import torch

from oracle import ofdm as F
from oracle import nr as ON
from oracle.parity import cnormal, envelope

DEFAULT_BAR = (2.0, 4.0)
BARS = {}                                       # (rms, max) bar of a comparison that needs its own: worst measured ratio
FLOOR = (2.0 ** -24, 2.0 ** -24)                # several steps are exact in both precisions
H100_SMS = 132                                  # H100 SXM5; the grid-stride kernels launch at most 16 CTAs per SM
INTERPS = ("nn", "lin", "lin_time_avg")


# ---- the table of pilot layouts --------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    make: object                                # () -> ResourceGrid
    batch: int = 2
    rx: int = 2
    ant: int = 2
    pusch: tuple = None                         # (dmrs_length, additional_position, num_cdm_groups_without_data)

    @functools.cached_property
    def rg(self):
        return self.make()

    @property
    def mask(self):
        return np.asarray(self.rg.pilot_pattern.mask).astype(bool)

    @property
    def pilots(self):
        return np.asarray(self.rg.pilot_pattern.pilots)

    @property
    def rows(self):
        """(frame, rx, antenna, tx, stream) rows of the estimator's kernels."""
        return self.batch * self.rx * self.ant * self.rg.num_tx * self.rg.num_streams_per_tx


def _kron(num_tx, num_streams, num_sym, fft, pilot_syms, guards=(0, 0), dc=False):
    from sionna_b200.phy.ofdm import ResourceGrid
    return lambda: ResourceGrid(num_sym, fft, 30e3, num_tx=num_tx, num_streams_per_tx=num_streams,
                                num_guard_carriers=guards, dc_null=dc, pilot_pattern="kronecker",
                                pilot_ofdm_symbol_indices=list(pilot_syms))


def _custom(mask_pilots, fft=None, guards=(0, 0), dc=False):
    def make():
        from sionna_b200.phy.ofdm import ResourceGrid, PilotPattern
        mask, pil = mask_pilots()
        tx, st, s_, f_ = mask.shape
        return ResourceGrid(s_, fft or f_, 30e3, num_tx=tx, num_streams_per_tx=st, num_guard_carriers=guards,
                            dc_null=dc, pilot_pattern=PilotPattern(mask, pil.astype(np.complex64)))
    return make


def _qpsk(rng, shape):
    return ((rng.integers(0, 2, shape) * 2 - 1) + 1j * (rng.integers(0, 2, shape) * 2 - 1)) / np.sqrt(2)


def _sparse():
    """Rows 2, 3, 10, 11 of 14 x 64 masked for four UEs; UE 0 has two non-zero pilots, UEs 1 ... 3 one each."""
    mask = np.zeros((4, 1, 14, 64), bool)
    mask[..., [2, 3, 10, 11], :] = True
    pil = np.zeros((4, 1, 256), complex)
    pil[0, 0, [10, 234]] = 1
    pil[1, 0, 20] = pil[2, 0, 70] = pil[3, 0, 120] = 1
    return mask, pil


def _diamond():
    """Staggered combs: pilot symbols 1, 5, 9, 13 alternate between two comb offsets, and the two UEs' combs are
    shifted by one subcarrier (UE 1 reaches the last subcarrier)."""
    mask = np.zeros((2, 1, 14, 48), bool)
    for t in range(2):
        for k, s in enumerate((1, 5, 9, 13)):
            mask[t, 0, s, 2 * (k % 2) + t::4] = True
    return mask, _qpsk(np.random.default_rng(1), (2, 1, 48))


def _per_stream_masks():
    """One UE, three streams with different masks: two pilot symbols on even subcarriers, one full pilot symbol, and
    three pilot symbols (the first and the last) on subcarriers 2, 5, ..., 47 (the last)."""
    mask = np.zeros((1, 3, 14, 48), bool)
    mask[0, 0, [2, 11], 0::2] = True
    mask[0, 1, 5, :] = True
    mask[0, 2, [0, 4, 13], 2::3] = True
    return mask, _qpsk(np.random.default_rng(2), (1, 3, 48))


def _random_pilots():
    """Random complex pilots of modulus 0.2 ... 2 on symbols 1, 6, 12, about 30 % of them zero; stream (0, 0) has a
    single non-zero pilot on symbol 6, stream (1, 1) none on symbol 12, stream (0, 1) non-zero pilots on both edge
    subcarriers of symbol 1, stream (1, 0) zeros on the two outermost subcarriers of each side."""
    rng = np.random.default_rng(3)
    mask = np.zeros((2, 2, 14, 40), bool)
    mask[..., [1, 6, 12], :] = True
    pil = rng.uniform(0.2, 2.0, (2, 2, 120)) * np.exp(2j * np.pi * rng.uniform(size=(2, 2, 120)))
    pil[rng.uniform(size=pil.shape) < 0.3] = 0
    pil[0, 0, 40:80] = 0
    pil[0, 0, 57] = 0.7 - 0.4j
    pil[1, 1, 80:] = 0
    pil[0, 1, [0, 39]] = [1.5, -0.3j]
    for k in (0, 1):
        pil[1, 0, 40 * k + np.array([0, 1, 38, 39])] = 0
        pil[1, 0, 40 * k + 2] = 1.1j
    return mask, pil


def _one_symbol():
    """S = 1 with data REs: two streams on interleaved combs, the second reaching the last subcarrier."""
    mask = np.zeros((1, 2, 1, 24), bool)
    mask[0, 0, 0, 0::3] = True
    mask[0, 1, 0, 2::3] = True
    return mask, _qpsk(np.random.default_rng(4), (1, 2, 8))


def _one_subcarrier():
    """F = 1: every pilot symbol holds exactly one pilot; the second stream's pilots sit on the first and last symbol."""
    mask = np.zeros((1, 2, 14, 1), bool)
    mask[0, 0, [3, 9], 0] = True
    mask[0, 1, [0, 13], 0] = True
    return mask, np.array([[[1.0, -1j], [0.5 + 0.5j, 2.0]]])


def _pusch(num_layers, length, additional_position, config_type, groups):
    def make():
        from sionna_b200.phy.nr import PUSCHConfig, PUSCHPilotPattern
        from sionna_b200.phy.ofdm import ResourceGrid
        pc = PUSCHConfig(num_layers=num_layers, num_antenna_ports=num_layers)
        pc.n_size_bwp = 4
        pc.dmrs.length = length
        pc.dmrs.additional_position = additional_position
        pc.dmrs.config_type = config_type
        pc.dmrs.num_cdm_groups_without_data = groups
        pp = PUSCHPilotPattern(pc)
        return ResourceGrid(14, pc.num_subcarriers, 30e3, num_tx=1, num_streams_per_tx=num_layers, pilot_pattern=pp)
    return make


def pusch_configs():
    """(layers, dmrs_length, additional_position, config_type, num_cdm_groups_without_data) of every DMRS configuration
    with the default port set: positions 0 ... 3 for single-symbol and 0 ... 1 for double-symbol DMRS, one to three CDM
    groups without data (two for type 1), and two groups at least for four layers (ports 2 and 3)."""
    return [(n, length, add, ct, g) for n in (1, 2, 4) for length in (1, 2) for add in range(4 if length == 1 else 2)
            for ct in (1, 2) for g in range(1 if n < 4 else 2, (2 if ct == 1 else 3) + 1)]


@functools.lru_cache(None)
def table():
    cases = [
        Case("kron_2_11", _kron(4, 1, 14, 64, [2, 11])),
        Case("kron_2", _kron(4, 1, 14, 64, [2])),
        Case("kron_16ue_16sc", _kron(16, 1, 14, 16, [2])),
        Case("kron_4ue_2st_2_5_8", _kron(4, 2, 14, 64, [2, 5, 8]), rx=2, ant=3),
        Case("kron_all_pilots", _kron(1, 1, 5, 64, range(5))),
        Case("kron_2_3_8_11", _kron(4, 1, 14, 64, [2, 3, 8, 11])),
        Case("kron_0_13_guards_dc", _kron(2, 1, 14, 76, [0, 13], guards=(5, 6), dc=True)),
        Case("kron_guards", _kron(2, 1, 14, 72, [2, 11], guards=(4, 4))),
        Case("kron_odd_fft_dc", _kron(2, 2, 14, 65, [3, 10], dc=True)),
        Case("kron_3276_subcarriers", _kron(4, 3, 14, 4096, [2, 11], guards=(410, 409), dc=True), batch=1, rx=1),
        Case("kron_many_rows", _kron(16, 1, 14, 16, [2, 11]), batch=160, rx=1, ant=8),
        Case("sparse", _custom(_sparse)),
        Case("diamond", _custom(_diamond)),
        Case("per_stream_masks", _custom(_per_stream_masks)),
        Case("random_pilots", _custom(_random_pilots), rx=1, ant=3),
        Case("one_symbol", _custom(_one_symbol, fft=28, guards=(2, 1), dc=True)),
        Case("one_subcarrier", _custom(_one_subcarrier)),
    ]
    for n, length, add, ct, g in pusch_configs():
        cases.append(Case(f"pusch_{n}l_len{length}_add{add}_type{ct}_cdm{g}", _pusch(n, length, add, ct, g), rx=1,
                          pusch=(length, add, g)))
    return {c.name: c for c in cases}


NAMES = list(table())
PLAIN = [n for n in NAMES if table()[n].pusch is None]


def _row_cap(cols):
    """Rows that the row-wise kernels (row_launch) cover in one pass of their grid on an H100."""
    tx = min(256, max(32, (cols + 31) // 32 * 32))
    return 16 * H100_SMS * max(1, 256 // tx)


def _nonzero(case):
    """[ts, S, F]: the REs that carry a non-zero pilot."""
    mask, pil = case.mask, case.pilots
    tx, st, s_, f_ = mask.shape
    z = np.zeros((tx * st, s_, f_), bool)
    for r, (m, p) in enumerate(zip(mask.reshape(-1, s_, f_), pil.reshape(tx * st, -1))):
        z[r][m] = np.abs(p) > 0
    return z


def test_table_covers_every_branch():
    """The table reaches every layout LinearInterpolator's index tables and the kernels' launch loops distinguish."""
    tab = table()
    plain = [tab[n] for n in PLAIN]
    seen = set()
    for c in plain:
        z, mask, pil = _nonzero(c), c.mask, c.pilots
        ts, s_, f_ = z.shape
        per_sym = z.sum(-1)                                               # [ts, S]
        m2 = mask.reshape(ts, s_, f_)
        if (per_sym == 1).any():
            seen.add("one non-zero pilot in a pilot symbol")
        for r in range(ts):
            for a in np.nonzero(per_sym[r] >= 2)[0]:
                lo, hi = np.nonzero(z[r, a])[0][[0, -1]]
                if (m2[r, a, lo:hi] & ~z[r, a, lo:hi]).any():
                    seen.add("zero pilot between two non-zero pilots")
                if lo > 0:
                    seen.add("extrapolation below the first pilot subcarrier")
                if hi < f_ - 1:
                    seen.add("extrapolation above the last pilot subcarrier")
            syms = np.nonzero(per_sym[r])[0]
            if len(syms) >= 2 and syms[0] > 0:
                seen.add("extrapolation before the first pilot symbol")
            if len(syms) >= 2 and syms[-1] < s_ - 1:
                seen.add("extrapolation after the last pilot symbol")
        if z[:, :, 0].any():
            seen.add("pilot on the first subcarrier")
        if z[:, :, -1].any():
            seen.add("pilot on the last subcarrier")
        if z[:, 0].any():
            seen.add("pilot on the first symbol")
        if z[:, -1].any():
            seen.add("pilot on the last symbol")
        if any(not np.array_equal(m2[0], m2[r]) for r in range(ts)):
            seen.add("streams with different masks")
        npil = (per_sym > 0).sum(-1)
        if len(set(npil)) > 1:
            seen.add("streams with different numbers of pilot symbols")
            if ((per_sym == 0) & (per_sym.max(0, keepdims=True) > 0)).any():
                seen.add("a symbol with pilots for one stream and none for another")
        mod = np.abs(pil.reshape(ts, -1))
        if any(len(np.unique(np.round(m[m > 0], 6))) > 1 for m in mod):
            seen.add("non-zero pilots of different modulus")
        ev = np.divide(0.1, mod ** 2, out=np.zeros_like(mod), where=mod > 0).reshape(pil.shape)
        if F.lin_interp(ev, mask, pil).real.min() < 0:
            seen.add("negative extrapolated error variance")
        if c.rg.pilot_pattern.num_data_symbols == 0:
            seen.add("no data REs")
        gc, dc = np.sum(c.rg.num_guard_carriers) > 0, c.rg.dc_null
        seen.add(f"guards {'on' if gc else 'off'}, DC null {'on' if dc else 'off'}")
        if s_ == 1:
            seen.add("S = 1")
        if f_ == 1:
            seen.add("F = 1")
        if f_ > 256:
            seen.add("F > 256")
        p = pil.shape[-1]
        if c.rows > 16 * H100_SMS and c.rows > _row_cap(p) and \
                c.batch * ts > _row_cap(c.rg.num_ofdm_symbols * c.rg.fft_size):
            seen.add("more rows than one grid pass")
    want = {"one non-zero pilot in a pilot symbol", "zero pilot between two non-zero pilots",
            "extrapolation below the first pilot subcarrier", "extrapolation above the last pilot subcarrier",
            "extrapolation before the first pilot symbol", "extrapolation after the last pilot symbol",
            "pilot on the first subcarrier", "pilot on the last subcarrier", "pilot on the first symbol",
            "pilot on the last symbol", "streams with different masks", "streams with different numbers of pilot symbols",
            "a symbol with pilots for one stream and none for another", "non-zero pilots of different modulus",
            "negative extrapolated error variance", "no data REs", "S = 1", "F = 1", "F > 256",
            "more rows than one grid pass"} | {f"guards {g}, DC null {d}" for g in ("on", "off") for d in ("on", "off")}
    assert want <= seen, sorted(want - seen)
    # the reference's Kronecker grids, multi-UE / multi-stream grids and the 3276-subcarrier grid
    kron = {tuple(np.nonzero(c.mask[0, 0].any(-1))[0]) for c in plain if c.name.startswith("kron")}
    assert {(2, 11), (2,), (2, 5, 8), (2, 3, 8, 11), (0, 1, 2, 3, 4), (0, 13)} <= kron
    assert any(c.rg.num_tx == 4 and c.rg.num_streams_per_tx == 2 for c in plain)
    assert any(c.rg.num_tx == 16 and c.rg.num_effective_subcarriers == 16 and (_nonzero(c).sum(-1) <= 1).all()
               for c in plain)
    assert any(c.rg.num_effective_subcarriers == 3276 and c.rg.fft_size == 4096 for c in plain)
    # every PUSCH DMRS configuration
    cfgs = pusch_configs()
    assert len(cfgs) == 78 and sum(tab[n].pusch is not None for n in NAMES) == 78
    assert {c[0] for c in cfgs} == {1, 2, 4} and {c[3] for c in cfgs} == {1, 2} and {c[4] for c in cfgs} == {1, 2, 3}
    assert {(c[1], c[2]) for c in cfgs} == {(1, 0), (1, 1), (1, 2), (1, 3), (2, 0), (2, 1)}


def test_interpolator_tables_match_oracle():
    """NearestNeighborInterpolator's gather table is oracle.ofdm.nn_interp of the pilot indices, for every layout (its
    host code once built an [S F, P] distance matrix: 10 GB and 90 s at 3276 subcarriers)."""
    from sionna_b200.phy.ofdm import NearestNeighborInterpolator
    for name in NAMES:
        case = table()[name]
        pil = case.pilots
        idx = np.broadcast_to(np.arange(pil.shape[-1]), pil.shape)
        want = F.nn_interp(idx, case.mask, pil).reshape(-1, case.mask[0, 0].size)
        assert np.array_equal(NearestNeighborInterpolator(case.rg.pilot_pattern)._gather_ind, want), name


# ---- inputs and oracles -----------------------------------------------------------------------------------------------
def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def _grid(rng, case):
    """[B, tx, st, S, fft] complex128: QPSK data on the data REs, the pattern's pilots, zeros on the nulled REs."""
    rg = case.rg
    tx, st = rg.num_tx, rg.num_streams_per_tx
    xd = _qpsk(rng, (case.batch, tx, st, rg.pilot_pattern.num_data_symbols))
    return F.rg_map(xd, case.pilots.reshape(tx, st, -1), rg.build_type_grid())


def _channel(rng, case, per_re=0.05, affine=False):
    """[B, rx, ant, tx, st, S, fft]: a gain with a slow phase ramp over frequency and time plus a small per-RE part, or
    (affine) a + b s + c f."""
    rg = case.rg
    s_, n = rg.num_ofdm_symbols, rg.fft_size
    lead = (case.batch, case.rx, case.ant, rg.num_tx, rg.num_streams_per_tx, 1, 1)
    s, f = np.arange(s_)[:, None], np.arange(n)[None, :]
    if affine:                                  # affine in the effective subcarrier index (nulled REs carry nothing)
        a, b, c = (cnormal(rng, lead, dtype=np.complex128) for _ in range(3))
        f = np.searchsorted(rg.effective_subcarrier_ind, f)
        return a + 0.1 * b * s + (0.5 / n) * c * f
    ramp = rng.uniform(-0.5, 0.5, lead) * f / n + rng.uniform(-0.02, 0.02, lead) * s
    return cnormal(rng, lead, dtype=np.complex128) * np.exp(2j * np.pi * ramp) + \
        per_re * cnormal(rng, lead[:5] + (s_, n), dtype=np.complex128)


def _received(rng, case, no, affine=False):
    """y [B, rx, ant, S, fft] complex64 through `_channel` plus CN(0, no) noise (no: [B, rx, ant] or None)."""
    y = np.einsum("brmtksf,btksf->brmsf", _channel(rng, case, affine=affine), _grid(rng, case))
    if no is not None:
        y = y + cnormal(rng, y.shape, dtype=np.complex128) * np.sqrt(no)[..., None, None]
    return y.astype(np.complex64)


def _noise(rng, case):
    return rng.uniform(0.01, 0.1, (case.batch, case.rx, case.ant)).astype(np.float32)


def _oracle(case, y, no, interp, dtype):
    """(h, err_var) of the estimator in dtype (np.complex128 / np.complex64): [B, rx, ant, tx, st, P] at the pilots
    (interp None), else over the grid."""
    rdt = np.float64 if dtype == np.complex128 else np.float32
    mask, pil = case.mask, case.pilots
    h, err = F.ls_estimate(y[..., case.rg.effective_subcarrier_ind].astype(dtype), mask, pil, np.asarray(no, rdt),
                           dtype=dtype)
    if case.pusch is not None:
        length, _, groups = case.pusch
        h, err = ON.pusch_ls_combine(h, err, len(_dmrs_symbols(case)), length, groups)
        h, err = h.astype(dtype), err.astype(rdt)
    if interp is None:
        return h, err
    if interp == "nn":
        return F.nn_interp(h, mask, pil, dtype=dtype), F.nn_interp(err, mask, pil, dtype=rdt)
    ta = interp == "lin_time_avg"
    return F.lin_interp(h, mask, pil, ta, dtype=dtype), np.maximum(F.lin_interp(err, mask, pil, ta, dtype=dtype).real, 0)


def _dmrs_symbols(case):
    return np.nonzero(case.mask[0, 0].any(-1))[0]


def _estimator(case, interp, precision=None):
    if case.pusch is None:
        from sionna_b200.phy.ofdm import LSChannelEstimator
        return LSChannelEstimator(case.rg, interp, precision=precision)
    from sionna_b200.phy.nr import PUSCHLSChannelEstimator
    length, _, groups = case.pusch
    add = len(_dmrs_symbols(case)) // length - 1
    return PUSCHLSChannelEstimator(case.rg, length, add, groups, interpolation_type=interp, precision=precision)


def _run(est, y, no, dev):
    h, e = est(torch.from_numpy(y).to(dev), torch.as_tensor(np.array(no)).to(dev))
    return h.cpu().numpy(), e.cpu().numpy()


def _env(what, got, f32, ref, axis):
    key = what.split(": ", 1)[-1]
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    return envelope(what, got, f32, ref, BARS.get(key, DEFAULT_BAR), floor=FLOOR, axis=axis)


ROW = (-2, -1)                                  # rows of the interpolated outputs: one (S, F) grid


# ---- 2. bit-exact parts -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_grid_mapping_and_gathers_bit_exact(cuda_device, name):
    """sb_rg_map against oracle.ofdm.rg_map / type_grid; RemoveNulledSubcarriers and ResourceGridDemapper (sb_gather_rows
    with 1, 2 and 4 words per element) against NumPy indexing."""
    from sionna_b200.phy.ofdm import ResourceGridMapper, RemoveNulledSubcarriers, ResourceGridDemapper
    from sionna_b200.phy.mimo import StreamManagement
    case = table()[name]
    rg, rng = case.rg, _rng("gathers", name)
    tx, st, s_, n = rg.num_tx, rg.num_streams_per_tx, rg.num_ofdm_symbols, rg.fft_size
    tg = F.type_grid(case.mask, n, rg.num_guard_carriers, rg.dc_null)
    assert np.array_equal(rg.build_type_grid(), tg)
    nd = rg.pilot_pattern.num_data_symbols
    x = cnormal(rng, (case.batch, tx, st, nd))
    got = ResourceGridMapper(rg)(torch.from_numpy(x).to(cuda_device)).cpu().numpy()
    assert np.array_equal(got, F.rg_map(x, case.pilots.reshape(tx, st, -1), tg)), name
    eff = np.asarray(rg.effective_subcarrier_ind)
    y = rng.normal(size=(case.batch, case.rx, case.ant, s_, n)) + 1j * rng.normal(size=(case.batch, case.rx, case.ant, s_, n))
    sm = StreamManagement(np.ones((1, tx), int), st)
    for precision, dt in (("single", np.float32), ("single", np.complex64), ("double", np.complex128),
                          ("double", np.float64)):
        v = (y.real if dt in (np.float32, np.float64) else y).astype(dt)
        out = RemoveNulledSubcarriers(rg, precision=precision)(torch.from_numpy(v).to(cuda_device)).cpu().numpy()
        assert out.dtype == dt and np.array_equal(out, v[..., eff]), (name, precision, dt)
        # demapper input [B, 1 rx, tx * st streams, S, fft] (+ a data dimension of 2 for real types)
        g = (rng.normal(size=(case.batch, 1, tx * st, s_, n, 2)) if dt in (np.float32, np.float64)
             else cnormal(rng, (case.batch, 1, tx * st, s_, n), dtype=np.complex128)).astype(dt)
        out = ResourceGridDemapper(rg, sm, precision=precision)(torch.from_numpy(g).to(cuda_device)).cpu().numpy()
        want = np.zeros((case.batch, tx, st, nd) + g.shape[5:], dt)
        streams = g[:, 0][:, np.asarray(sm.stream_ind)][:, :, :, eff]                       # [B, ts, S, F, (dd)]
        for r in range(tx * st):
            flat = streams[:, r].reshape((case.batch, -1) + g.shape[5:])
            want[:, r // st, r % st] = flat[:, ~case.mask.reshape(tx * st, -1)[r]]
        assert out.dtype == dt and np.array_equal(out, want), (name, precision, dt)
    print(f"{name}: mapper, RemoveNulledSubcarriers and ResourceGridDemapper bit-exact (fp32, complex64, complex128, fp64)")


# ---- 3. LS at the pilots, and nearest-neighbour interpolation of the kernel's own pilot estimates --------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_ls_at_pilots_and_nearest_neighbour(cuda_device, name):
    """sb_ls_at_pilots (and for PUSCH sb_pusch_ls_combine): h and err_var within the envelope of float64
    oracle.ofdm.ls_estimate (+ oracle.nr.pusch_ls_combine), exactly 0 at zero pilots; the nearest-neighbour estimate
    is oracle.ofdm.nn_interp of the kernel's own pilot estimates, bit for bit."""
    case = table()[name]
    rng = _rng("ls", name)
    no = _noise(rng, case)
    y = _received(rng, case, no)
    hp, ep = _run(_estimator(case, None), y, no, cuda_device)
    h64, e64 = _oracle(case, y, no, None, np.complex128)
    h32, e32 = _oracle(case, y, no, None, np.complex64)
    bad = [_env(f"{name}: LS h", hp, h32, h64, -1), _env(f"{name}: LS err_var", ep, e32, e64, -1)]
    zero = np.broadcast_to(case.pilots == 0, hp.shape)
    assert (hp[zero] == 0).all() and (ep[zero] == 0).all(), name
    hn, en = _run(_estimator(case, "nn"), y, no, cuda_device)
    assert np.array_equal(hn, F.nn_interp(hp, case.mask, case.pilots)), name
    assert np.array_equal(en, F.nn_interp(ep, case.mask, case.pilots)), name
    print(f"{name}: nearest-neighbour h / err_var bit-exact")
    assert not any(bad), "\n".join(x for x in bad if x)


# ---- 4a. the linear interpolator alone --------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_linear_interpolator_alone(cuda_device, name):
    """LinearInterpolator (sb_interp_lin) on inputs exact in float32, against float64 oracle.ofdm.lin_interp: complex
    h, real err_var unfloored, and floored inside the kernel (exactly max(unfloored, 0)); lin and lin_time_avg."""
    from sionna_b200.phy.ofdm import LinearInterpolator
    case = table()[name]
    rng = _rng("lin alone", name)
    mask, pil = case.mask, case.pilots
    lead = (case.batch * case.rx * case.ant,) + pil.shape
    h = cnormal(rng, lead)
    ev = rng.uniform(0.0, 1.0, lead).astype(np.float32)
    bad = []
    for ta in (False, True):
        what = f"{name}: {'lin_time_avg' if ta else 'lin'}"
        itp = LinearInterpolator(case.rg.pilot_pattern, time_avg=ta)
        hk, ek = (t.cpu().numpy() for t in itp(torch.from_numpy(h).to(cuda_device), torch.from_numpy(ev).to(cuda_device)))
        hf, ef = (t.cpu().numpy() for t in itp.interpolate_floored(torch.from_numpy(h).to(cuda_device),
                                                                   torch.from_numpy(ev).to(cuda_device)))
        assert np.array_equal(hf, hk) and np.array_equal(ef, np.maximum(ek, np.float32(0))), what
        e64 = F.lin_interp(ev.astype(np.float64), mask, pil, ta).real
        e32 = F.lin_interp(ev, mask, pil, ta, dtype=np.complex64).real
        bad += [_env(f"{what} h", hk, F.lin_interp(h, mask, pil, ta, dtype=np.complex64),
                     F.lin_interp(h.astype(np.complex128), mask, pil, ta), ROW),
                _env(f"{what} err_var", ek, e32, e64, ROW),
                _env(f"{what} err_var floored", ef, np.maximum(e32, np.float32(0)), np.maximum(e64, 0), ROW)]
    assert not any(bad), "\n".join(x for x in bad if x)


# ---- 4b / 5. the whole estimator with linear interpolation --------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_ls_estimator_linear(cuda_device, name):
    """LSChannelEstimator / PUSCHLSChannelEstimator with lin and lin_time_avg from y with noise on a channel that varies
    in frequency and time plus a per-RE part, against the float64 chain."""
    case = table()[name]
    rng = _rng("estimator", name)
    no = _noise(rng, case)
    y = _received(rng, case, no)
    bad = []
    for interp in ("lin", "lin_time_avg"):
        hk, ek = _run(_estimator(case, interp), y, no, cuda_device)
        h64, e64 = _oracle(case, y, no, interp, np.complex128)
        h32, e32 = _oracle(case, y, no, interp, np.complex64)
        bad += [_env(f"{name}: {interp} h", hk, h32, h64, ROW), _env(f"{name}: {interp} err_var", ek, e32, e64, ROW)]
    assert not any(bad), "\n".join(x for x in bad if x)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kron_2_11", "kron_4ue_2st_2_5_8", "kron_0_13_guards_dc", "kron_2_3_8_11",
                                  "kron_odd_fft_dc", "kron_3276_subcarriers"])
def test_affine_channel_recovered_exactly(cuda_device, name):
    """Noiseless, with a channel affine in (symbol, effective subcarrier) and orthogonal (Kronecker) pilots: linear
    interpolation and extrapolation are exact in float64, so the estimate must equal the true channel within the
    envelope."""
    case = table()[name]
    rng = _rng("affine", name)
    h_true = _channel(rng, case, affine=True)
    y = np.einsum("brmtksf,btksf->brmsf", h_true, _grid(rng, case)).astype(np.complex64)
    truth = h_true[..., case.rg.effective_subcarrier_ind]
    no = np.zeros((case.batch, case.rx, case.ant), np.float32)
    hk, _ = _run(_estimator(case, "lin"), y, no, cuda_device)
    h64, _ = _oracle(case, y, no, "lin", np.complex128)
    h32, _ = _oracle(case, y, no, "lin", np.complex64)
    assert np.abs(h64 - truth).max() < 1e-6 * np.abs(truth).max(), name            # y is complex64: ~1e-7 relative
    bad = envelope(f"{name}: affine channel h vs truth", hk, h32, truth, DEFAULT_BAR, floor=FLOOR, axis=ROW)
    assert not bad, bad


# ---- noise shapes, double precision, the all-pilot grid -----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("interp", INTERPS)
def test_noise_shapes(cuda_device, interp):
    """Every accepted shape of `no` (scalar, [B], [B, rx], [B, rx, ant]) equals the explicitly expanded [B, rx, ant]."""
    case = table()["kron_4ue_2st_2_5_8"]
    rng = _rng("noise shapes", interp)
    no = _noise(rng, case)
    y = _received(rng, case, no)
    est = _estimator(case, interp)
    for shape_no in (no[0, 0, 0], no[:, 0, 0], no[:, :, 0], no, no[:, :1, :]):
        full = np.broadcast_to(np.reshape(shape_no, np.shape(shape_no) + (1,) * (3 - np.ndim(shape_no))), no.shape)
        got = _run(est, y, np.ascontiguousarray(shape_no), cuda_device)
        want = _run(est, y, np.ascontiguousarray(full), cuda_device)
        assert all(np.array_equal(g, w) for g, w in zip(got, want)), np.shape(shape_no)
    got = _run(est, y, float(no[0, 0, 0]), cuda_device)                              # a Python float
    want = _run(est, y, np.full(no.shape, no[0, 0, 0], np.float32), cuda_device)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))


@pytest.mark.gpu
@pytest.mark.parametrize("interp", INTERPS)
def test_double_precision_estimator(cuda_device, interp):
    """precision="double": complex128 / float64 in and out, the single-precision kernels inside, so the estimates are
    the single-precision ones widened. The nulled subcarriers are dropped by a bit copy of the complex128 grid, and the
    LS kernel is fed complex64 (it once read the complex128 grid as complex64 pairs)."""
    case = table()["kron_0_13_guards_dc"]
    rng = _rng("double", interp)
    no = _noise(rng, case)
    y = _received(rng, case, no)
    hs, es = _run(_estimator(case, interp), y, no, cuda_device)
    hd, ed = _run(_estimator(case, interp, precision="double"), y.astype(np.complex128), no.astype(np.float64),
                  cuda_device)
    assert hd.dtype == np.complex128 and ed.dtype == np.float64
    assert np.array_equal(hd, hs.astype(np.complex128)) and np.array_equal(ed, es.astype(np.float64))


@pytest.mark.gpu
def test_all_pilot_grid(cuda_device):
    """Every RE a pilot (num_data_symbols == 0): ResourceGridMapper maps an empty data tensor (its device pointer is
    null) to the pilots, ResourceGridDemapper returns an empty tensor, and the estimator recovers a noiseless channel
    that is constant over the grid exactly."""
    from sionna_b200.phy.ofdm import ResourceGridMapper, ResourceGridDemapper
    from sionna_b200.phy.mimo import StreamManagement
    case = table()["kron_all_pilots"]
    rg = case.rg
    assert rg.num_data_symbols == 0
    x = torch.zeros((3, 1, 1, 0), dtype=torch.complex64, device=cuda_device)
    grid = ResourceGridMapper(rg)(x)
    assert grid.shape == (3, 1, 1, 5, 64)
    assert np.array_equal(grid.cpu().numpy()[0, 0, 0].reshape(-1), case.pilots[0, 0])
    out = ResourceGridDemapper(rg, StreamManagement(np.ones((1, 1), int), 1))(grid.reshape(3, 1, 1, 5, 64))
    assert out.shape == (3, 1, 1, 0)
    chan = cnormal(_rng("all pilots"), (3, 1, 2), dtype=np.complex64)
    y = (torch.from_numpy(chan)[..., None, None].to(cuda_device) * grid[:, :, 0][:, :, None]).reshape(3, 1, 2, 5, 64)
    for interp in INTERPS:
        h, e = _estimator(case, interp)(y, 0.0)
        want = np.broadcast_to(chan[..., None, None, None, None], h.shape)
        assert np.allclose(h.cpu().numpy(), want, rtol=1e-6, atol=0) and (e.cpu().numpy() == 0).all(), interp
