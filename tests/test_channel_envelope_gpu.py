"""csrc/channel.cu against float64 references over its advertised range: the CIR -> channel conversion (sb_phase_table,
sb_cir_gram, sb_cir_link_scale, sb_cir_apply), the TDL taps (sb_tdl_sos), the spatial correlation (sb_spatial_corr) and
the channel application (sb_apply_ofdm_channel, sb_apply_time_channel; their noise is checked in
test_rng_streams_gpu.py).

Yardstick: the same formula evaluated in complex64 / float32 with NumPy (oracle.ofdm with dtype=np.complex64): the
kernel's error against float64 must be at most 2x (rms) and 4x (max) the yardstick's, unless BARS names an exception.
Errors are taken relative to the natural scale of each output (sqrt(sum |a_p|^2) for a CIR contraction, sqrt(sum
|L_ij|^2 |v_j|^2) for a matrix-vector product, ...) so that outputs near a zero of the channel do not dominate, and the
yardstick is floored at 2^-24 of that scale (some cases are exact in both). Every comparison prints its ratios
(pytest -s).

The normalisation has its own, absolute bar: on nearly flat channels (delays << 1 / bandwidth) the Gram matrix of the
table is almost rank one, and on a link in a deep fade the quadratic form a^H G a cancels to a tiny fraction of its
terms. The factor must still equal the float64 one computed from the kernel's own table to 5e-6 (unit energy to 1e-5).
"""
import numpy as np
import pytest
import torch

from oracle import ofdm as F
from oracle.parity import cnormal, envelope

pytestmark = pytest.mark.gpu

DEFAULT_BAR = (2.0, 4.0)
BARS = {                                        # (rms, max) bar of a comparison that needs its own: worst measured ratio
    "tdl_sos": (3.0, 4.0),                      # 2.53 / 3.54: each output is up to 15 complex multiplications down the
                                                # 16-step phasor recurrence from its fp32 sincosf anchor, against one
                                                # complex exp per sinusoid and step in the float32 evaluation; the worst
                                                # |a - a64| is 1.6e-6 of the path amplitude at every T, 30 706 included
}
FLOOR = (2.0 ** -24, 2.0 ** -24)                # least complex64 (rms, max) error, relative to the scale


def _dev(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _call(fn, *args):
    """C-ABI call; tensor arguments are passed as device pointers and stay referenced until the kernel has finished (a
    temporary freed early would hand its memory to the next allocation while the kernel still reads it)."""
    from sionna_b200._lib import lib, check, ptr, current_stream
    check(getattr(lib(), fn)(*[ptr(x) if isinstance(x, torch.Tensor) else x for x in args], current_stream()), fn)
    torch.cuda.synchronize()


def _tap_scale(a):
    """sqrt(sum_p |a_p|^2) per (row, t): [B, RX, RA, TX, TA, T, 1]."""
    return np.sqrt((np.abs(a.astype(np.complex128)) ** 2).sum(-2))[..., None]


def _link_norm(h, axes=(2, 4, 5, 6), denom_axis=None):
    """c = sqrt(mean |h|^2) over the link's antenna pairs, time steps and columns (OFDM), or over antenna pairs and time
    steps of the summed tap energy (time channel: denom_axis = 6), in h's precision; keepdims."""
    e = np.abs(h) ** 2
    if denom_axis is not None:
        e = e.sum(denom_axis, keepdims=True)
        axes = tuple(x for x in axes if x != denom_axis)
    return np.sqrt(e.mean(axis=axes, keepdims=True))


def _normalised(h, c):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(c > 0, h / np.where(c > 0, c, 1), 0).astype(h.dtype)


# ---- 1. sb_cir_apply through cir_to_ofdm_channel / cir_to_time_channel ---------------------------------------------
# (mode, columns F, time steps T, paths P, per-link delays): F > 48 takes the 16 x 256 tile, F <= 48 the 128 x 32 one;
# every F and T of the list appears, partial tiles on both axes, and P up to the 96-path limit.
CIR = [("ofdm", 1, 1, 1, False), ("ofdm", 31, 15, 24, True), ("ofdm", 32, 16, 64, False), ("ofdm", 33, 17, 96, True),
       ("ofdm", 48, 129, 24, False), ("ofdm", 49, 128, 1, True), ("ofdm", 255, 17, 24, True),
       ("ofdm", 256, 16, 96, False), ("ofdm", 257, 15, 64, True), ("ofdm", 4096, 1, 24, False),
       ("ofdm", 4096, 17, 7, True), ("ofdm", 76, 127, 3, False),
       ("time", 1, 129, 24, False), ("time", 31, 127, 96, True), ("time", 32, 128, 24, True), ("time", 33, 15, 1, False),
       ("time", 48, 1, 64, True), ("time", 49, 16, 24, False), ("time", 19, 1000, 24, True)]


@pytest.mark.parametrize("mode,f,t,p,per_link", CIR, ids=[f"{c[0]}-F{c[1]}-T{c[2]}-P{c[3]}-{'link' if c[4] else 'shared'}" for c in CIR])
def test_cir_apply_envelope(cuda_device, mode, f, t, p, per_link):
    from sionna_b200.phy.channel import cir_to_ofdm_channel, cir_to_time_channel, subcarrier_frequencies
    rng = np.random.default_rng(1000 * f + 10 * t + p)
    b, rx, ra, tx, ta = (2, 1, 2, 2, 1) if f * t < 50000 else (1, 1, 2, 1, 1)
    a = cnormal(rng, (b, rx, ra, tx, ta, p, t))
    a[0, 0, 0, 0, 0, :, :1] = 0                                     # one zero time step of one row
    if mode == "ofdm":
        bw, lo, hi = f * 30e3, None, None
        freqs = subcarrier_frequencies(f, 30e3)
        tau_max = 5e-6
    else:
        bw, lo = 15.36e6, -6
        hi = lo + f - 1
        tau_max = max(hi, 1) / bw
    tau = np.sort(rng.uniform(0, tau_max, (b, rx, tx, p) if per_link else (p,))).astype(np.float32)
    tau_d = _dev(tau, cuda_device) if per_link else _dev(tau, cuda_device).reshape(1, 1, 1, p).expand(b, rx, tx, p)
    ad = _dev(a, cuda_device)
    bad = []
    for normalize in (False, True):
        if mode == "ofdm":
            got = cir_to_ofdm_channel(freqs, ad, tau_d, normalize=normalize).cpu().numpy()
            ref = F.cir_to_ofdm(freqs.numpy(), a, tau)
            f32 = F.cir_to_ofdm(freqs.numpy(), a, tau, np.complex64)
            kw = {}
        else:
            got = cir_to_time_channel(bw, ad, tau_d, lo, hi, normalize=normalize).cpu().numpy()
            ref = F.cir_to_time(bw, a, tau, lo, hi)
            f32 = F.cir_to_time(bw, a, tau, lo, hi, np.complex64)
            kw = {"denom_axis": 6}
        assert got.shape == ref.shape == (b, rx, ra, tx, ta, t, f)
        scale = _tap_scale(a)
        if normalize:
            c64, c32 = _link_norm(ref, **kw), _link_norm(f32, **kw)
            ref, f32 = _normalised(ref, c64), _normalised(f32, c32)
            scale = scale / np.where(c64 > 0, c64, 1)
        assert np.all(np.isfinite(got))
        assert np.all(got[0, 0, 0, 0, 0, 0] == 0)
        bad.append(envelope(f"cir {mode} normalize={normalize}", got, f32, ref, DEFAULT_BAR, FLOOR, scale=scale))
    assert not any(bad), "\n".join(x for x in bad if x)


def test_cir_more_than_96_paths_named(cuda_device):
    """Both kernels accept up to 96 paths; beyond that the error names the limit, with or without normalisation."""
    from sionna_b200.phy.channel import cir_to_ofdm_channel, subcarrier_frequencies
    from sionna_b200._lib import SbError
    a = torch.ones((1, 1, 1, 1, 1, 97, 1), dtype=torch.complex64, device=cuda_device)
    tau = torch.zeros((1, 1, 1, 97), device=cuda_device)
    for normalize in (False, True):
        with pytest.raises(SbError, match="more than 96 paths"):
            cir_to_ofdm_channel(subcarrier_frequencies(12, 15e3), a, tau, normalize=normalize)


# ---- 2. sb_phase_table and sb_cir_gram ---------------------------------------------------------------------------------
def test_phase_table_large_f_tau_and_sinc_edges(cuda_device):
    """exp(-j 2 pi f tau) at f tau up to 4000 turns (tau up to 20 us, |f| up to 200 MHz): the table equals the float64
    value of the fp32 inputs to 1 ulp (only the double-precision turn reduction keeps the phase; fp32 would be off by
    ~1e-3). Sinc table: u = 0 exactly gives 1, |u| ~ 1e-7 stays accurate."""
    from sionna_b200._lib import ptr
    rng = np.random.default_rng(7)
    p, fcols = 6, 301
    tau = np.concatenate([[0.0, 20e-6], rng.uniform(0, 20e-6, p - 2)]).astype(np.float32)
    freq = np.concatenate([[-200e6, 200e6, 0.0], rng.uniform(-200e6, 200e6, fcols - 3)]).astype(np.float32)
    e = torch.empty((1, p, fcols), dtype=torch.complex64, device=cuda_device)
    _call("sb_phase_table", _dev(tau, cuda_device), _dev(freq, cuda_device), 0.0, 0, ptr(e), 1, p, fcols)
    ref = np.exp(-2j * np.pi * (tau.astype(np.float64)[:, None] * freq.astype(np.float64)[None, :]))
    err = float(np.abs(e.cpu().numpy()[0] - ref).max())
    print(f"phase table: max |e - e64| = {err:.2e} at f tau up to {float(np.abs(tau[:, None] * freq).max()):.0f} turns")
    assert err <= 2.0 ** -23
    # sinc: scale W = 1; tau * W = lag exactly (u = 0), and u of about -2.4e-7 / 1e-7 near lags 3, 0 and 2
    bw = np.float32(3.0000001)                                      # 3 + 2^-22 in fp32
    tau = np.array([1.0, 2.0 / 3.0000001, 1e-7 / 3.0000001, 0.0], np.float32)
    lags = np.arange(-3, 5, dtype=np.float32)
    e = torch.empty((1, 4, len(lags)), dtype=torch.complex64, device=cuda_device)
    _call("sb_phase_table", _dev(tau, cuda_device), _dev(lags, cuda_device), float(bw), 1, ptr(e), 1, 4, len(lags))
    got = e.cpu().numpy()[0]
    u = lags.astype(np.float64)[None, :] - tau.astype(np.float64)[:, None] * np.float64(bw)
    k = np.rint(u)                                                   # sin(pi u) = (-1)^k sin(pi (u - k)), u - k exact:
    with np.errstate(invalid="ignore"):                              # np.sinc rounds pi * u and loses the small values
        ref = np.where(u == 0, 1.0, (1 - 2 * (k % 2)) * np.sin(np.pi * (u - k)) / (np.pi * u))
    assert np.all(got.imag == 0) and got[3, 3] == 1.0                # tau = 0, lag 0: u = 0 exactly
    rel = np.abs(got.real - ref) / np.maximum(np.abs(ref), 1e-30)
    print(f"sinc table: max relative error {rel.max():.2e}, smallest |value| {np.abs(ref).min():.2e}")
    assert rel.max() <= 2.0 ** -23


@pytest.mark.parametrize("f,p", [(1, 1), (1, 24), (31, 5), (33, 24), (100, 96), (4096, 3)])
def test_cir_gram_double(cuda_device, f, p):
    """G = E E^H of the kernel's own table, accumulated in double: equal to the float64 product to 1e-12 of
    sum_j |e_pj| |e_qj| (an fp32 accumulation misses this by ~1e-7)."""
    from sionna_b200._lib import ptr
    rng = np.random.default_rng(f * 100 + p)
    n_tab = 3
    e = cnormal(rng, (n_tab, p, f))
    g = torch.empty((n_tab, p, p), dtype=torch.complex128, device=cuda_device)
    _call("sb_cir_gram", _dev(e, cuda_device), ptr(g), n_tab, p, f)
    e64 = e.astype(np.complex128)
    ref = np.einsum("tpj,tqj->tpq", e64, e64.conj())
    bound = np.einsum("tpj,tqj->tpq", np.abs(e64), np.abs(e64))
    err = float((np.abs(g.cpu().numpy() - ref) / bound).max())
    print(f"gram F={f} P={p}: max error {err:.2e} of sum |e_p| |e_q|")
    assert err <= 1e-12


# ---- 3. normalisation on deep fades of nearly flat channels -------------------------------------------------------------
def _kernel_table(tau, x, mode, scale, dev):
    from sionna_b200._lib import ptr
    p = tau.shape[-1]
    e = torch.empty((1, p, x.shape[0]), dtype=torch.complex64, device=dev)
    _call("sb_phase_table", _dev(tau, dev), _dev(x, dev), float(scale), mode, ptr(e), 1, p, x.shape[0])
    return e.cpu().numpy()[0].astype(np.complex128)


@pytest.mark.parametrize("mode,spread", [("ofdm", 1e-9), ("ofdm", 10e-9), ("time", 1e-9), ("time", 10e-9)])
def test_normalisation_deep_fades(cuda_device, mode, spread):
    """SISO, T = 1, TDL-A taps, 20 000 links, 12 subcarriers of 15 kHz (OFDM) or taps at 1.92 MHz (time channel): the
    factor of every link equals 1 / sqrt(mean energy) computed in float64 from the fp32 taps and the kernel's own
    table, to 5e-6, so the energy is 1 to 1e-5 however deep the fade. An all-zero link stays exactly zero, and no other
    link gets the factor 0."""
    from sionna_b200.phy.channel import TDL, cir_to_ofdm_channel, cir_to_time_channel, subcarrier_frequencies
    links = 20000
    tdl = TDL("A", spread, 3.5e9)
    a, tau = tdl(links, 1, 1.0)
    a[7] = 0
    taus = tdl.delays.numpy()
    if mode == "ofdm":
        x = subcarrier_frequencies(12, 15e3)
        h = cir_to_ofdm_channel(x, a, tau).cpu().numpy().astype(np.complex128)
        hn = cir_to_ofdm_channel(x, a, tau, normalize=True).cpu().numpy().astype(np.complex128)
        e = _kernel_table(taus, x.numpy(), 0, 0.0, cuda_device)
        denom = 12
    else:
        bw, lo, hi = 1.92e6, -6, 7
        x = torch.arange(lo, hi + 1, dtype=torch.float32)
        h = cir_to_time_channel(bw, a, tau, lo, hi).cpu().numpy().astype(np.complex128)
        hn = cir_to_time_channel(bw, a, tau, lo, hi, normalize=True).cpu().numpy().astype(np.complex128)
        e = _kernel_table(taus, x.numpy(), 1, bw, cuda_device)
        denom = 1
    an = a.cpu().numpy().astype(np.complex128).reshape(links, -1)    # [links, P]
    energy = (np.abs(an @ e) ** 2).sum(-1) / denom                   # float64 from the kernel's table
    h, hn = h.reshape(links, -1), hn.reshape(links, -1)
    assert np.all(hn[7] == 0) and np.all(h[7] == 0)
    live = np.arange(links) != 7
    # the kernel's factor, from its own normalised and unnormalised output (same accumulation, hn = fl(h * c))
    c_k = (np.conj(h) * hn).real.sum(-1) / np.maximum((np.abs(h) ** 2).sum(-1), 1e-300)
    assert np.all(c_k[live] > 0), "a non-zero link was scaled by 0"
    c_ref = 1.0 / np.sqrt(energy[live])
    rel = np.abs(c_k[live] / c_ref - 1.0)
    fade = np.abs(an.sum(-1))[live] / np.abs(an).sum(-1)[live]
    print(f"normalisation {mode} {spread * 1e9:.0f} ns: worst |c / c64 - 1| = {rel.max():.2e} (median {np.median(rel):.1e}),"
          f" deepest fade |sum a| / sum |a| = {fade.min():.1e}")
    assert rel.max() <= 5e-6
    assert np.abs(c_k[live] ** 2 * energy[live] - 1.0).max() <= 1e-5          # unit mean energy


# ---- 4. sb_spatial_corr -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 8, 32, 128])
def test_spatial_corr_envelope(cuda_device, n):
    """out = L v for a lower-triangular L; at n = 128 the factor takes n^2 * 8 B = 128 KB of shared memory, above the
    48 KB default; cols = 77 is not a multiple of the 128-thread block."""
    from sionna_b200._lib import ptr
    rng = np.random.default_rng(n)
    bsz, cols = 3, 77
    m = cnormal(rng, (n, 2 * n)).astype(np.complex128)
    l = np.linalg.cholesky(m @ m.conj().T / (2 * n) + 0.1 * np.eye(n)).astype(np.complex64)
    v = cnormal(rng, (bsz, n, cols))
    out = torch.empty((bsz, n, cols), dtype=torch.complex64, device=cuda_device)
    _call("sb_spatial_corr", _dev(v, cuda_device), _dev(l, cuda_device), ptr(out), bsz, n, cols)
    ref = np.einsum("ij,bjc->bic", l.astype(np.complex128), v.astype(np.complex128))
    f32 = np.einsum("ij,bjc->bic", l, v)
    scale = np.sqrt(np.einsum("ij,bjc->bic", np.abs(l).astype(np.float64) ** 2, np.abs(v).astype(np.float64) ** 2))
    bad = envelope(f"spatial corr n={n}", out.cpu().numpy(), f32, ref, DEFAULT_BAR, FLOOR, scale=scale)
    assert not bad, bad


# ---- 5. sb_tdl_sos ----------------------------------------------------------------------------------------------------
LONG_T = 14 * (2048 + 144) + 19 - 1                                 # a time channel: 14 symbols of 2048 + 144, l_tot = 19
TDL_CASES = [("A", 20, 1), ("A", 20, 15), ("D", 20, 16), ("A", 1, 17), ("D", 64, 17), ("A", 64, 16), ("D", 1, 15),
             ("A", 20, LONG_T), ("D", 20, LONG_T)]


@pytest.mark.parametrize("speed", [(3.0, 3.0), (30.0, 60.0)])
@pytest.mark.parametrize("model,ns,t", TDL_CASES, ids=[f"{c[0]}-Ns{c[1]}-T{c[2]}" for c in TDL_CASES])
def test_tdl_sos_envelope(cuda_device, model, ns, t, speed):
    """The kernel's 16-step phasor recurrence against float64, on identical draws, LoS (D) and NLoS (A); long T is a
    time channel sampled at 30.72 MHz. Error relative to sqrt(P_p) (the path's rms amplitude); the worst |a - a64| is
    printed per T."""
    from sionna_b200.phy.channel import TDL
    long_t = t == LONG_T
    tdl = TDL(model, 100e-9, 3.5e9, num_sinusoids=ns, min_speed=speed[0], max_speed=speed[1],
              num_rx_ant=1 if long_t else 2, num_tx_ant=1 if long_t else 2)
    fs = 30.72e6 if long_t else 14e3
    draws = tdl.draws(2 if long_t else 16)
    got = tdl.synthesize(draws, t, fs).cpu().numpy()
    d = [None if x is None else x.cpu().numpy() for x in draws]
    args = (d[0], d[1], d[2], d[3], tdl._powers, tdl._los_power, tdl._los_aoa, t, fs)
    ref = F.tdl_sos(*args)
    f32 = F.tdl_sos(*args, dtype=np.float32)
    pw = np.asarray(tdl._powers, np.float64).copy()
    if tdl.los:
        pw[0] += tdl._los_power
    scale = np.sqrt(pw)[None, None, :, None]
    print(f"tdl {model} Ns={ns} T={t} speed {speed}: worst |a - a64| = {np.abs(got - ref).max():.2e}")
    bad = envelope(f"tdl_sos T={t}", got, f32, ref, BARS["tdl_sos"], FLOOR, scale=scale)
    assert not bad, bad


# ---- 6. channel application (noiseless; the noise is pinned in test_rng_streams_gpu.py) --------------------------------
@pytest.mark.parametrize("r,tt,re", [(1, 1, 1), (16, 16, 301), (4, 2, 1000), (2, 8, 129), (3, 1, 4097)])
def test_apply_ofdm_channel_envelope(cuda_device, r, tt, re):
    from sionna_b200.phy.channel import ApplyOFDMChannel
    rng = np.random.default_rng(r * tt + re)
    b, s = 2, 1
    h = cnormal(rng, (b, 1, r, 1, tt, s, re))
    x = cnormal(rng, (b, 1, tt, s, re))
    got = ApplyOFDMChannel()(_dev(x, cuda_device), _dev(h, cuda_device)).cpu().numpy()
    ref = np.einsum("brmtksf,btksf->brmsf", h.astype(np.complex128), x.astype(np.complex128))
    f32 = np.einsum("brmtksf,btksf->brmsf", h, x)
    scale = np.sqrt(np.einsum("brmtksf,btksf->brmsf", np.abs(h).astype(np.float64) ** 2, np.abs(x).astype(np.float64) ** 2))
    bad = envelope(f"apply ofdm R={r} Tt={tt} RE={re}", got, f32, ref, DEFAULT_BAR, FLOOR, scale=scale)
    assert not bad, bad


@pytest.mark.parametrize("tt,n,l", [(1, 3, 8), (2, 1, 5), (3, 40, 1), (1, 1, 1), (4, 600, 19), (2, 17, 17)])
def test_apply_time_channel_envelope(cuda_device, tt, n, l):
    """N < L, L = 1, N = L, and the first / last L - 1 outputs where the l0 / l1 clamps cut the sum."""
    from sionna_b200.phy.channel import ApplyTimeChannel
    rng = np.random.default_rng(100 * n + l)
    b, r = 2, 3
    h = cnormal(rng, (b, 1, r, 1, tt, n + l - 1, l))
    x = cnormal(rng, (b, 1, tt, n))
    got = ApplyTimeChannel(n, l)(_dev(x, cuda_device), _dev(h, cuda_device)).cpu().numpy()[:, 0]
    h3, x3 = h[:, 0, :, 0], x[:, 0]
    ref = F.apply_time_channel(x3, h3)
    f32 = F.apply_time_channel(x3, h3, np.complex64)
    scale = np.sqrt(F.apply_time_channel(np.abs(x3) ** 2, np.abs(h3) ** 2).real)
    bad = envelope(f"apply time N={n} L={l}", got, f32, ref, DEFAULT_BAR, FLOOR, scale=scale)
    edges = np.r_[0:min(l - 1, n + l - 1), max(n, 0):n + l - 1]
    bad2 = envelope(f"apply time N={n} L={l} edges", got[..., edges], f32[..., edges], ref[..., edges], DEFAULT_BAR,
                    FLOOR, scale=scale[..., edges]) if len(edges) else ""
    assert not bad and not bad2, bad + bad2
