"""The fused receive front-end (sb_ofdm_frontend, csrc/frontend.cu, through FusedLSLinearDetector) against a float64
oracle assembled from oracle pieces that share no code with it:

    oracle.ofdm.ls_estimate -> (PUSCH: oracle.nr.pusch_ls_combine) -> nn_interp / lin_interp (time_avg)
    -> ofdm_lmmse_equalize -> oracle.mimo.logits_to_llrs(-|x_hat - c|^2 / max(no_eff, tiny))

The error variance goes through the same interpolator and is floored at 0, as LSChannelEstimator does; the LLRs are the
reference's 2-D Demapper formula. The yardstick is the same sequence in complex64 / float32 (ls_estimate and the
interpolators with dtype=np.complex64, ofdm_lmmse_equalize_f32, logits_to_llrs on float32 logits): how far any
single-precision evaluation of the chain sits from float64. Errors are relative per element for x_hat and no_eff, and
relative to the rms of the float64 LLRs of each (frame, stream) row for LLRs. The kernel's rms and max error must be at
most 2x and 3x the yardstick's, unless BARS names an exception (the worst ratio measured on an H100 80GB HBM3 is written
beside it). Every comparison prints its ratios (pytest -s).

Cases and the branches they pin:
  test_soft_llrs_all_variants     every ofdm_frontend_kernel<K, H, METHOD> (K = 1..4 streams, H = 1..5 bits per
                                  dimension, app / maxlog) on Kronecker grids, nn / lin / lin_time_avg, antenna tails
                                  (ANT % 4 != 0) and ANT >= 16 for every K, a single partial tile (< 128 listed REs)
                                  and partial last tiles; x_hat / no_eff through equalize(); hard_out for one method
                                  per (K, H): bit-exact against soft > 0, and equal to the float64 decisions wherever
                                  the float64 |LLR| exceeds the soft-output bound
  test_high_snr_app               the app demapper's underflow fallback (|LLR| > ~85), levels in kernel-parameter space;
                                  constellations whose real and imaginary levels differ tell the two dimensions apart
  test_pusch_tables               CDM de-spreading folded into the tables; NT = 16 terms (double-symbol DMRS, one
                                  additional position, linear interpolation), with 4 layers the opt-in shared memory
  test_batch_slices               the batch-slice loop: more frames than ceil(8 SMs / (tiles * RX)), so a CTA walks
                                  several frames; results per frame independent of the batch
  test_noise_shapes               every accepted shape of `no` equals the explicitly expanded [B, 1, ANT] tensor
  test_two_receivers_c_abi        num_rx = 2 through the C-ABI equals two num_rx = 1 calls
"""
import zlib

import numpy as np
import pytest
import torch

from oracle import ofdm as F
from oracle import nr as ON
from oracle.mimo import logits_to_llrs
from oracle.parity import cnormal, envelope

pytestmark = pytest.mark.gpu

DEFAULT_BAR = (2.0, 3.0)
BARS = {                                        # (rms, max) bar of a comparison that needs its own: worst measured ratio
    "x_hat": (3.2, 7.0),                        # 2.58 / 5.66: whitening by rsqrt (<= 2 ulp) and x_hat through
                                                # A^-1 = C^-H C^-1 in registers, as the LMMSE envelope's "ofdm diag x_hat"
    "x_hat ANT=1<K": (400.0, 800.0),            # 307.7 / 655.8: one antenna, several streams. The reference solves
                                                # G = A^-1 h^H along A's dominant eigenvector, exact to a few ulp in
                                                # complex64; the kernel has only B = h^H h and forms diag(A^-1 B), which
                                                # cancels by 1 + |h_w|^2 (numpy float32 evaluation of the same formula:
                                                # 2e-4 ... 6e-4 relative). With 2 <= ANT < K the reference loses the same
                                                # accuracy and the ratio is <= 2 (x_hat) / 2.5 (no_eff, LLRs, below)
    "no_eff ANT<K": (3.0, 3.5),                 # 2.47 / 2.41
    "llr ANT<K": (3.0, 3.5),                    # 2.41 / 2.90
}
HARD_EXCLUDED = {5: 0.08}                       # fraction of hard bits below the soft-output bound, by H, default 1 %:
                                                # 1024-QAM 6.5 % (the complex64 2-D demapper's own LLR error grows with
                                                # the symbol's largest logit, about 1e5 here)
TINY = 1.17549435e-38                           # float32 tiny: the demapper's floor of no (mapping.py:653)
METHODS = ("app", "maxlog")
ANTS = (1, 2, 3, 5, 7, 8, 13, 16, 17)
INTERPS = ("nn", "lin", "lin_time_avg")


def _grid(k, num_sym, fft, pilots, guards=(0, 0), dc=False):
    from sionna_b200.phy.ofdm import ResourceGrid
    return ResourceGrid(num_sym, fft, 15e3, num_tx=1, num_streams_per_tx=k, cyclic_prefix_length=0,
                        num_guard_carriers=guards, dc_null=dc, pilot_pattern="kronecker",
                        pilot_ofdm_symbol_indices=list(pilots))


def _demapper_constellation(h, kind="qam"):
    """Square QAM with 2^(2h) points, or ("asym") a separable constellation whose imaginary levels are the real ones
    reversed and scaled by 0.75, so that the two dimensions cannot be confused."""
    from sionna_b200.phy.mapping import Constellation, separable_levels_np
    const = Constellation("qam", 2 * h)
    if kind == "qam":
        return const
    lev_re, _ = separable_levels_np(const.points.numpy(), 2 * h)
    lev_im = (0.75 * lev_re[::-1]).astype(np.float32)
    j = np.arange(1 << (2 * h))
    bits = (j[:, None] >> np.arange(2 * h - 1, -1, -1)) & 1
    w = 1 << np.arange(h - 1, -1, -1)
    pts = (lev_re[bits[:, 0::2] @ w] + 1j * lev_im[bits[:, 1::2] @ w]).astype(np.complex64)
    out = Constellation("custom", 2 * h, points=pts, normalize=False, center=False)
    got = separable_levels_np(out.points.numpy(), 2 * h)
    assert got is not None and not np.array_equal(got[0], got[1])
    return out


def _no_scale(h, ant=1, k=1):
    """Squared PAM level spacing relative to QPSK's times the receive diversity max(1, ANT - K + 1): no in [0.01, 0.1]
    times this gives every constellation and antenna count a similar spread of LLR magnitudes, most of them below the
    app demapper's underflow threshold."""
    return 3.0 / (4 ** h - 1) * max(1, ant - k + 1)


def _received(rng, rg, b, ant, pts, no, rx=1):
    """y [b, rx, ant, S, fft] complex64: the grid (uniformly drawn data points, the pattern's pilots) through a channel
    with a slow phase ramp over frequency and time plus a small per-RE part, and CN(0, no) noise (no broadcastable to
    [b, rx, ant])."""
    pp = rg.pilot_pattern
    tx, st = rg.num_tx, rg.num_streams_per_tx
    xd = pts[rng.integers(0, len(pts), (b, tx, st, pp.num_data_symbols))]
    grid = F.rg_map(xd, np.asarray(pp.pilots).reshape(tx, st, -1), rg.build_type_grid())
    s_, n = rg.num_ofdm_symbols, rg.fft_size
    lead = (b, rx, ant, tx, st, 1, 1)
    ramp = rng.uniform(-0.003, 0.003, lead) * np.arange(n) + rng.uniform(-0.01, 0.01, lead) * np.arange(s_)[:, None]
    h = cnormal(rng, lead, dtype=np.complex128) * np.exp(2j * np.pi * ramp) + \
        0.02 * cnormal(rng, (b, rx, ant, tx, st, s_, n), dtype=np.complex128)
    y = np.einsum("brmtksf,btksf->brmsf", h, grid)
    no_b = np.broadcast_to(np.reshape(no, np.shape(no) + (1,) * (3 - np.ndim(no))), (b, rx, ant))
    return (y + cnormal(rng, y.shape, dtype=np.complex128) * np.sqrt(no_b)[..., None, None]).astype(np.complex64)


def _oracle(rg, y, no, interp, pts, method, dtype, pusch=None):
    """(x_hat, no_eff [B, tx, st, nd], LLRs [B, tx, st, nd * m]) of the chain in dtype (np.complex128 / np.complex64)
    for one receiver; pusch = (num_dmrs_syms, dmrs_length, num_cdm_groups_without_data) inserts the CDM de-spreading."""
    rdt = np.float64 if dtype == np.complex128 else np.float32
    pp = rg.pilot_pattern
    mask, pil = np.asarray(pp.mask).astype(bool), np.asarray(pp.pilots)
    y_eff = y[..., np.asarray(rg.effective_subcarrier_ind)]
    no = np.asarray(no, rdt)
    h, err = F.ls_estimate(y_eff, mask, pil, no, dtype=dtype)
    if pusch is not None:
        h, err = ON.pusch_ls_combine(h, err, *pusch)
        h, err = h.astype(dtype), err.astype(rdt)
    if interp == "nn":
        h, err = F.nn_interp(h, mask, pil, dtype=dtype), F.nn_interp(err, mask, pil, dtype=rdt)
    else:
        ta = interp == "lin_time_avg"
        h, err = F.lin_interp(h, mask, pil, ta, dtype=dtype), F.lin_interp(err, mask, pil, ta, dtype=dtype).real
    err = np.maximum(err, rdt(0))
    smr = F.stream_management([[1]], rg.num_streams_per_tx)
    eq = F.ofdm_lmmse_equalize if dtype == np.complex128 else F.ofdm_lmmse_equalize_f32
    x, ne = eq(y_eff, h, err, no, mask, smr)
    m = int(np.log2(len(pts)))
    c = np.asarray(pts).astype(dtype)
    logits = -np.abs(x[..., None] - c) ** 2 / np.maximum(ne, rdt(TINY))[..., None]
    llr = logits_to_llrs(logits, m, method)
    return x, ne, llr.reshape(llr.shape[:-2] + (-1,))


def _hard_check(what, hard, soft, ref, f32, m, bar=DEFAULT_BAR):
    """hard_out is exactly soft > 0 of the same kernel, and equals the float64 decisions wherever the float64 |LLR|
    exceeds bar[1] times the yardstick's largest absolute LLR error among the m bits of the same symbol; fewer than 1 %
    of the bits excluded (HARD_EXCLUDED)."""
    assert np.array_equal(hard, (soft > 0).astype(np.float32)), f"{what}: hard_out differs from soft > 0"
    err = np.abs(f32 - ref).reshape(ref.shape[:-1] + (-1, m))
    bound = bar[1] * np.broadcast_to(err.max(-1, keepdims=True), err.shape).reshape(ref.shape)
    keep = np.abs(ref) > bound
    excluded = 1.0 - keep.mean()
    limit = HARD_EXCLUDED.get(m // 2, 0.01)
    print(f"{what}: hard outputs, {excluded:.3%} excluded (limit {limit:.0%})")
    assert excluded < limit, what
    assert np.array_equal(hard[keep], (ref[keep] > 0).astype(np.float32)), what


def _detector(est, rg, k, const, method, hard_out=False):
    from sionna_b200.phy.ofdm import FusedLSLinearDetector
    from sionna_b200.phy.mimo import StreamManagement
    sm = StreamManagement(np.ones((1, 1), int), k)
    return FusedLSLinearDetector(est, rg, sm, method, constellation=const, hard_out=hard_out)


def _run(det, y, no, dev):
    yd, nd = torch.from_numpy(y).to(dev), torch.as_tensor(no).to(dev)
    return det(yd, nd).cpu().numpy(), tuple(t.cpu().numpy() for t in det.equalize(yd, nd))


def _compare(tag, rg, est_kind, y, no, const, method, soft, eq, pusch=None, ant=None):
    """Envelope of x_hat, no_eff and the LLRs; returns the failures and (float64, float32) LLRs. ant: the antenna
    count when it is below the number of streams (BARS)."""
    pts = const.points.numpy()
    x64, n64, l64 = _oracle(rg, y.astype(np.complex128), no, est_kind, pts, method, np.complex128, pusch)
    x32, n32, l32 = _oracle(rg, y, no, est_kind, pts, method, np.complex64, pusch)
    assert soft.shape == l64.shape and eq[0].shape == x64.shape, tag
    low = ant is not None and ant < rg.num_streams_per_tx
    bad = [envelope(f"{tag} x_hat", eq[0], x32, x64, BARS["x_hat ANT=1<K" if low and ant == 1 else "x_hat"],
                    scale=np.abs(x64)),
           envelope(f"{tag} no_eff", eq[1], n32, n64, BARS["no_eff ANT<K"] if low else DEFAULT_BAR, scale=np.abs(n64)),
           envelope(f"{tag} llr", soft, l32, l64, BARS["llr ANT<K"] if low else DEFAULT_BAR)]
    return bad, l64, l32


# ---- 1. all 40 kernel variants ---------------------------------------------------------------------------------------
def _variant(k, h, method):
    """(ANT, interpolation, pilot symbols, OFDM symbols, fft size, guards, dc, batch) of variant (k, h, method)."""
    j = 2 * (h - 1) + (method == "maxlog")                         # 0..9 within one K
    i = 10 * (k - 1) + j
    ant = ANTS[(j + 2 * k) % len(ANTS)]                            # every K walks all 9 antenna counts
    interp = INTERPS[i % 3]
    s_ = 14 if h <= 3 else 5                                       # 1024- / 256-QAM: a few thousand REs
    pilots = ([[2], [2, 11], [0, 5, 13]] if s_ == 14 else [[1], [0, 4], [0, 2, 4]])[(i // 3) % 3]
    odd = i % 2 == 1
    return ant, interp, pilots, s_, 66 if odd else 60, (2, 3) if odd else (0, 0), odd, 3 if h <= 3 else 2


VARIANTS = [(k, h, meth) for k in (1, 2, 3, 4) for h in (1, 2, 3, 4, 5) for meth in METHODS]
assert len(set(VARIANTS)) == 40 == 4 * 5 * 2
for _k in (1, 2, 3, 4):                                            # antenna tails and >= 16 antennas for every K
    _a = {_variant(_k, _h, _m)[0] for _h in range(1, 6) for _m in METHODS}
    assert any(a % 4 for a in _a) and any(a >= 16 for a in _a) and _a == set(ANTS), _k
_LISTED = {v: (_variant(*v)[3] - len(_variant(*v)[2])) * 60 for v in VARIANTS}
assert any(n < 128 for n in _LISTED.values()) and any(n > 128 and n % 128 for n in _LISTED.values())


@pytest.mark.parametrize("k,h,method", VARIANTS, ids=[f"K{k}-H{h}-{m}" for k, h, m in VARIANTS])
def test_soft_llrs_all_variants(cuda_device, k, h, method):
    from sionna_b200.phy.ofdm import LSChannelEstimator
    ant, interp, pilots, s_, fft, guards, dc, b = _variant(k, h, method)
    rng = np.random.default_rng(zlib.crc32(f"variant {k} {h} {method}".encode()))
    rg = _grid(k, s_, fft, pilots, guards, dc)
    assert rg.num_effective_subcarriers == 60
    const = _demapper_constellation(h)
    det = _detector(LSChannelEstimator(rg, interp), rg, k, const, method)
    assert det._sm.num_streams_per_rx == k and const.num_bits_per_symbol == 2 * h and det._method == METHODS.index(method)
    assert det._num_listed == _LISTED[(k, h, method)]             # < 128: one partial tile; else a partial last tile
    assert det._num_listed % 128 != 0
    no = (rng.uniform(0.01, 0.1, (b, 1, ant)) * _no_scale(h, ant, k)).astype(np.float32)
    y = _received(rng, rg, b, ant, const.points.numpy(), no)
    soft, eq = _run(det, y, no, cuda_device)
    tag = f"K={k} H={h} {method} ANT={ant} {interp} pilots={pilots} listed={det._num_listed}"
    bad, l64, l32 = _compare(tag, rg, interp, y, no, const, method, soft, eq, ant=ant)
    if method == METHODS[(k + h) % 2]:                             # hard output: one method per (K, H)
        hard, _ = _run(_detector(LSChannelEstimator(rg, interp), rg, k, const, method, hard_out=True), y, no, cuda_device)
        _hard_check(tag, hard, soft, l64, l32, 2 * h)
    assert not any(bad), "\n".join(x for x in bad if x)


# ---- 2. high SNR: the app demapper's underflow fallback --------------------------------------------------------------
HIGH_SNR = [(2, "qam"), (3, "qam"), (4, "qam"), (5, "qam"), (3, "asym"), (5, "asym")]


@pytest.mark.parametrize("h,kind", HIGH_SNR, ids=[f"H{h}-{kd}" for h, kd in HIGH_SNR])
def test_high_snr_app(cuda_device, h, kind):
    """no between 1e-4 and 1e-3: a bit group of a dimension underflows as a whole next to the dimension's largest
    exponent (|LLR| > ~85), and demap_qam_group_fallback sums it from the levels in kernel-parameter space."""
    from sionna_b200.phy.ofdm import LSChannelEstimator
    k, ant, b = 2, 5, 2
    rng = np.random.default_rng(zlib.crc32(f"high snr {h} {kind}".encode()))
    rg = _grid(k, 5, 60, [1])
    const = _demapper_constellation(h, kind)
    det = _detector(LSChannelEstimator(rg, "lin"), rg, k, const, "app")
    no = rng.uniform(1e-4, 1e-3, (b, 1, ant)).astype(np.float32)
    y = _received(rng, rg, b, ant, const.points.numpy(), no)
    soft, eq = _run(det, y, no, cuda_device)
    tag = f"high SNR K={k} H={h} {kind} app"
    bad, l64, _ = _compare(tag, rg, "lin", y, no, const, "app", soft, eq)
    big = np.abs(l64) > 85
    print(f"{tag}: {big.mean():.1%} of the float64 |LLR| > 85")
    assert big.mean() > 0.05                                       # the fallback runs on these bits
    assert np.all(np.isfinite(soft))
    assert not any(bad), "\n".join(x for x in bad if x)


# ---- 3. PUSCH: CDM de-spreading, NT = 16, opt-in shared memory ---------------------------------------------------------
# (layers, DMRS config type, length, additional position, CDM groups without data, interpolation, bits per symbol,
#  method, antennas)
PUSCH = [(1, 1, 2, 1, 1, "lin", 4, "maxlog", 4),                   # NT = 16
         (2, 2, 2, 1, 3, "lin", 6, "app", 8),                      # NT = 16
         (4, 1, 2, 1, 2, "lin", 4, "maxlog", 16),                  # NT = 16, 12 * 4 * 16 * 128 B of tables > 48 KB
         (1, 2, 1, 0, 2, "nn", 8, "maxlog", 3),
         (2, 1, 1, 1, 2, "lin", 2, "app", 5),
         (4, 2, 1, 0, 3, "nn", 6, "app", 8),
         (2, 2, 2, 0, 1, "nn", 4, "maxlog", 7)]


@pytest.mark.parametrize("cfg", PUSCH, ids=[f"L{c[0]}-type{c[1]}-len{c[2]}-add{c[3]}-cdm{c[4]}-{c[5]}" for c in PUSCH])
def test_pusch_tables(cuda_device, cfg):
    from sionna_b200.phy.nr import PUSCHConfig, PUSCHTransmitter
    from sionna_b200.phy.nr.pusch_channel_estimation import PUSCHLSChannelEstimator
    layers, ctype, length, addpos, cdm, interp, m, method, ant = cfg
    pc = PUSCHConfig(num_layers=layers, num_antenna_ports=layers)
    pc.carrier.n_size_grid = 4
    pc.dmrs.config_type = ctype
    pc.dmrs.length = length
    pc.dmrs.additional_position = addpos
    pc.dmrs.num_cdm_groups_without_data = cdm
    tx = PUSCHTransmitter(pc)
    rg = tx.resource_grid
    est = PUSCHLSChannelEstimator(rg, tx._dmrs_length, tx._dmrs_additional_position, tx._num_cdm_groups_without_data,
                                  interpolation_type=interp)
    const = _demapper_constellation(m // 2)
    det = _detector(est, rg, layers, const, method)
    if length == 2 and addpos == 1 and interp == "lin":
        assert det._num_terms == 16
        if layers == 4:                                            # the launch opts in to > 48 KB of shared memory
            assert 12 * layers * det._num_terms * 128 > 48 * 1024
    rng = np.random.default_rng(zlib.crc32(str(cfg).encode()))
    b = 2
    no = (rng.uniform(0.01, 0.1, (b, 1, ant)) * _no_scale(m // 2, ant, layers)).astype(np.float32)
    y = _received(rng, rg, b, ant, const.points.numpy(), no)
    soft, eq = _run(det, y, no, cuda_device)
    tag = f"PUSCH {cfg} NT={det._num_terms}"
    bad, _, _ = _compare(tag, rg, interp, y, no, const, method, soft, eq,
                         pusch=(est._num_dmrs_syms, est._dmrs_length, est._num_cdm_groups_without_data))
    assert not any(bad), "\n".join(x for x in bad if x)


# ---- 4. batch slices -------------------------------------------------------------------------------------------------
def test_batch_slices(cuda_device):
    """More frames than ceil(8 SMs / (tiles * RX)): every CTA loops over several frames of its batch slice. Frames 0..3
    equal a batch-4 call bit for bit; the first frame of the second round and the last frame match the oracle."""
    from sionna_b200.phy.ofdm import LSChannelEstimator
    k, h, ant, method = 2, 2, 4, "app"
    rg = _grid(k, 14, 600, [2, 11])
    const = _demapper_constellation(h)
    det = _detector(LSChannelEstimator(rg, "lin"), rg, k, const, method)
    tiles = -(-det._num_listed // 128)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    slices = -(-8 * sms // tiles)                                  # batch slices (CTAs per RE tile) of the launch
    b = slices + 5
    assert b > slices
    rng = np.random.default_rng(21)
    no = (rng.uniform(0.01, 0.1, (b, 1, ant)) * _no_scale(h, ant, k)).astype(np.float32)
    y = _received(rng, rg, b, ant, const.points.numpy(), no)
    soft, eq = _run(det, y, no, cuda_device)
    soft4, eq4 = _run(det, y[:4], no[:4], cuda_device)
    assert np.array_equal(soft[:4], soft4) and np.array_equal(eq[0][:4], eq4[0]) and np.array_equal(eq[1][:4], eq4[1])
    pick = [0, slices, b - 1]
    tag = f"batch {b} > {slices} slices ({tiles} tiles, {sms} SMs), frames {pick}"
    bad, _, _ = _compare(tag, rg, "lin", y[pick], no[pick], const, method, soft[pick], (eq[0][pick], eq[1][pick]))
    assert not any(bad), "\n".join(x for x in bad if x)


# ---- 5. noise shapes -------------------------------------------------------------------------------------------------
def test_noise_shapes(cuda_device):
    """Scalar, [B], [B, 1], [1, 1, ANT] and [B, 1, ANT] noise equal the same values as an explicit [B, 1, ANT] tensor."""
    from sionna_b200.phy.ofdm import LSChannelEstimator
    k, h, ant, b = 3, 3, 5, 3
    rg = _grid(k, 14, 60, [2, 11])
    const = _demapper_constellation(h)
    det = _detector(LSChannelEstimator(rg, "nn"), rg, k, const, "app")
    rng = np.random.default_rng(22)
    y = torch.from_numpy(_received(rng, rg, b, ant, const.points.numpy(), 0.003)).to(cuda_device)
    per = rng.uniform(0.001, 0.01, (b, 1, ant)).astype(np.float32)
    for no in (np.float32(0.003), per[:, 0, 0], per[:, :, 0], per[:1, :, :], per):
        full = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(
            np.reshape(no, np.shape(no) + (1,) * (3 - np.ndim(no))), (b, 1, ant)))).to(cuda_device)
        arg = torch.as_tensor(no).to(cuda_device)
        assert torch.equal(det(y, arg), det(y, full)), np.shape(no)
        for a, f in zip(det.equalize(y, arg), det.equalize(y, full)):
            assert torch.equal(a, f), np.shape(no)


# ---- 6. two receivers through the C-ABI ------------------------------------------------------------------------------
def test_two_receivers_c_abi(cuda_device):
    """num_rx = 2 (receiver r detects streams des[r]; the kernel ignores the other receiver's streams by contract)
    equals two num_rx = 1 calls on y[:, r] and no[:, r], bit for bit, for the LLRs and for x_hat / no_eff."""
    from sionna_b200._lib import lib, check, ptr, current_stream
    from sionna_b200.phy.ofdm import LSChannelEstimator
    from sionna_b200.phy.ofdm.equalization import _strides_for
    k_all, k, h, ant, b = 4, 2, 2, 5, 3
    rg = _grid(k_all, 5, 60, [1, 3])
    const = _demapper_constellation(h)
    det = _detector(LSChannelEstimator(rg, "lin"), rg, k_all, const, "app")
    t = det._tables(cuda_device)
    rng = np.random.default_rng(23)
    no = rng.uniform(0.01, 0.1, (b, 2, ant)) * _no_scale(h, ant, k)
    y = torch.from_numpy(_received(rng, rg, b, ant, const.points.numpy(), no, rx=2)).to(cuda_device)
    no = torch.from_numpy(no.astype(np.float32)).to(cuda_device)
    des = torch.tensor([[2, 0], [3, 1]], dtype=torch.int32, device=cuda_device)     # disjoint stream rows
    nd, m = rg.pilot_pattern.num_data_symbols, 2 * h

    def call(yy, nn, dd, want_llr, out):
        bb, rx, aa, s_, nf = yy.shape
        nn, st = _strides_for(nn, [bb, rx, aa])
        llr, xh, ne = (out, None, None) if want_llr else (None, out[0], out[1])
        check(lib().sb_ofdm_frontend(ptr(yy), ptr(nn), ptr(np.asarray(st, np.int64)), ptr(dd), ptr(dd), ptr(t["data_pos"]),
                                     ptr(t["re_full"]), ptr(t["t_idx"]), ptr(t["t_w"]), ptr(t["e_sum"]), ptr(det._lev[0]),
                                     ptr(det._lev[1]), ptr(llr), ptr(xh), ptr(ne), bb, rx, aa, k_all, det._num_listed,
                                     s_ * nf, k, det._num_terms, nd, h, det._method, 0, current_stream()), "sb_ofdm_frontend")

    for want_llr in (True, False):
        def buf():
            if want_llr:
                return torch.zeros((b, 1, k_all, nd * m), dtype=torch.float32, device=cuda_device)
            return (torch.zeros((b, 1, k_all, nd), dtype=torch.complex64, device=cuda_device),
                    torch.zeros((b, 1, k_all, nd), dtype=torch.float32, device=cuda_device))
        both, split = buf(), buf()
        call(y, no, des, want_llr, both)
        for r in range(2):
            call(y[:, r:r + 1].contiguous(), no[:, r:r + 1].contiguous(), des[r:r + 1].contiguous(), want_llr, split)
        for a, s in zip(both if isinstance(both, tuple) else (both,), split if isinstance(split, tuple) else (split,)):
            assert bool((a != 0).any(-1).all()), "a stream row was not written"
            assert torch.equal(a, s)
