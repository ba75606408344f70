"""Pin the OFDM / MIMO oracle (oracle/ofdm.py) with the reference's own test recipes (no TensorFlow needed):
CP correctness and mod->demod round trip for every cp in [0, 72] at fft_size 72 with max error < 1e-5
(test/unit/ofdm/test_ofdm.py:15-96), trailing-sample truncation (:111-123), interpolators reproduce channels that are
linear in frequency / time exactly, LMMSE: noiseless recovery and the statistical identity err_var == mean(no_eff)
of test/unit/mimo/test_mimo_equalizers.py:55-102 (reduced sample count)."""
import numpy as np
import pytest

from oracle import ofdm as F


def test_cyclic_prefix_and_round_trip():
    rng = np.random.default_rng(0)
    n = 72
    x = rng.normal(size=(4, 14, n)) + 1j * rng.normal(size=(4, 14, n))
    for cp in range(0, n + 1, 7):
        t = F.ofdm_modulate(x, cp).reshape(4, 14, n + cp)
        assert np.array_equal(t[..., :cp], t[..., n:])                     # CP = copy of the symbol's tail
        assert np.abs(F.ofdm_demodulate(t.reshape(4, -1), n, 0, cp) - x).max() < 1e-5
    cps = rng.integers(0, n, 14)                                           # per-symbol CP
    t = F.ofdm_modulate(x, cps)
    assert t.shape[-1] == 14 * n + cps.sum()
    assert np.abs(F.ofdm_demodulate(t, n, 0, cps) - x).max() < 1e-5
    t2 = np.concatenate([F.ofdm_modulate(x, 5), np.zeros((4, 40))], -1)    # trailing samples are dropped
    assert np.abs(F.ofdm_demodulate(t2, n, 0, 5) - x).max() < 1e-5


def test_phase_compensation_undoes_timing_offset():
    rng = np.random.default_rng(1)
    n, cp, l_min = 64, 8, -3
    x = rng.normal(size=(2, 3, n)) + 1j * rng.normal(size=(2, 3, n))
    t = F.ofdm_modulate(x, cp)
    t = np.roll(t, -l_min, axis=-1)                                        # channel delays the signal by -l_min samples
    # every OFDM symbol (except for samples wrapped across the frame edge by np.roll) is recovered
    assert np.abs(F.ofdm_demodulate(t, n, l_min, cp) - x)[:, 1:-1].max() < 1e-5


def test_interpolators_exact_on_linear_channels():
    mask = F.kronecker_mask(2, 1, 14, 24, [2, 11])
    pil = np.zeros((2, 1, 2, 24), complex)
    pil[0, 0, :, 0::2] = 1.0
    pil[1, 0, :, 1::2] = 1j
    pil = pil.reshape(2, 1, -1)
    s_, f_ = np.meshgrid(np.arange(14), np.arange(24), indexing="ij")
    htrue = 1 + 0.1 * s_ + 0.05j * f_
    hp = np.zeros((3, 2, 1, 48), complex)
    for tx in range(2):
        for k, (a, c) in enumerate(np.argwhere(mask[tx, 0])):
            hp[:, tx, 0, k] = htrue[a, c] if abs(pil[tx, 0, k]) > 0 else 0
    out = F.lin_interp(hp, mask, pil)
    assert np.abs(out - htrue).max() < 1e-12
    avg = F.lin_interp(hp, mask, pil, time_avg=True)
    assert np.abs(avg - (1 + 0.1 * 6.5 + 0.05j * f_)).max() < 1e-12
    nn = F.nn_interp(hp, mask, pil)
    assert np.abs(nn[0, 0, 0, 0, 0] - htrue[2, 0]) < 1e-12 and np.abs(nn[0, 1, 0, 13, 23] - htrue[11, 23]) < 1e-12


def test_lmmse_noiseless_and_statistics():
    rng = np.random.default_rng(2)
    m, k, num = 8, 4, 20000
    h = (rng.normal(size=(num, m, k)) + 1j * rng.normal(size=(num, m, k))) / np.sqrt(2)
    x = (rng.integers(0, 2, (num, k)) * 2 - 1 + 1j * (rng.integers(0, 2, (num, k)) * 2 - 1)) / np.sqrt(2)
    no = 0.2
    a = rng.normal(size=(m, m)) + 1j * rng.normal(size=(m, m))
    s = no * (np.eye(m) + 0.3 * a @ a.conj().T / m)                        # coloured noise covariance
    l = np.linalg.cholesky(s)
    n = (l @ ((rng.normal(size=(num, m, 1)) + 1j * rng.normal(size=(num, m, 1))) / np.sqrt(2)))[..., 0]
    y = (h @ x[..., None])[..., 0] + n
    x_hat, no_eff = F.lmmse_equalizer(y, h, np.broadcast_to(s, (num, m, m)))
    err = x_hat - x
    assert abs(np.mean(err)) < 1e-2
    assert abs(np.var(err) - np.mean(no_eff)) / np.mean(no_eff) < 3e-2
    x0, ne0 = F.lmmse_equalizer((h @ x[..., None])[..., 0], h, np.broadcast_to(1e-9 * np.eye(m), (num, m, m)))
    assert np.abs(x0 - x).max() < 1e-5 and ne0.max() < 1e-6


def test_oracle_channel_generation_restatements():
    """oracle.ofdm.tdl_sos / cir_to_ofdm / cir_to_time / apply_time_channel against independent closed forms."""
    rng = np.random.default_rng(4)
    b, a_pairs, p, ns, t_steps, fs = 3, 2, 4, 20, 6, 1e4
    powers = np.array([0.5, 0.3, 0.15, 0.05])
    theta = rng.uniform(-np.pi / ns, np.pi / ns, (b, p, ns))
    phi = rng.uniform(-np.pi, np.pi, (b, a_pairs, p, ns))
    # zero Doppler: the taps do not depend on time and equal sqrt(P / Ns) * sum_n exp(j phi_n)
    a0 = F.tdl_sos(np.zeros(b), theta, phi, None, powers, 0.0, 0.0, t_steps, fs)
    want = np.sqrt(powers / ns)[None, None, :] * np.exp(1j * phi).sum(-1)
    assert np.allclose(a0, want[..., None]) and a0.shape == (b, a_pairs, p, t_steps)
    # one sinusoid, no angle jitter: a pure complex exponential at w cos(2 pi / 1)
    w = np.array([200.0, 300.0, 0.0])
    a1 = F.tdl_sos(w, np.zeros((b, 1, 1)), np.zeros((b, 1, 1, 1)), None, np.array([1.0]), 0.0, 0.0, t_steps, fs)
    tt = np.arange(t_steps) / fs
    assert np.allclose(a1[:, 0, 0, :], np.exp(1j * w[:, None] * tt[None, :] * np.cos(2 * np.pi)))
    # LoS term on the first path only
    phi0 = rng.uniform(-np.pi, np.pi, b)
    a2 = F.tdl_sos(w, theta, phi, phi0, powers, 0.7, np.pi / 4, t_steps, fs)
    base = F.tdl_sos(w, theta, phi, None, powers, 0.0, 0.0, t_steps, fs)
    spec = np.sqrt(0.7) * np.exp(1j * (w[:, None] * tt[None, :] * np.cos(np.pi / 4) + phi0[:, None]))
    assert np.allclose(a2[:, :, 0, :] - base[:, :, 0, :], spec[:, None, :]) and np.allclose(a2[:, :, 1:], base[:, :, 1:])
    # a single path with delay tau: frequency response exp(-j 2 pi f tau), time response sinc(l - tau W)
    freqs = (np.arange(16) - 8) * 15e3
    tau = np.array([2.5e-6])
    h = F.cir_to_ofdm(freqs, np.ones((1, 1, 3), complex), tau)
    assert np.allclose(h[0], np.exp(-2j * np.pi * freqs * tau[0])[None, :].repeat(3, 0))
    bw = 16 * 15e3
    ht = F.cir_to_time(bw, np.ones((1, 1, 3), complex), np.array([3 / bw]), -2, 5)       # integer delay of 3 samples
    assert np.allclose(ht[0, 0], (np.arange(-2, 6) == 3).astype(float), atol=1e-12)
    # time-variant filtering with constant taps is a plain convolution
    x = rng.normal(size=(2, 2, 10)) + 1j * rng.normal(size=(2, 2, 10))
    taps = rng.normal(size=(2, 3, 2, 4)) + 1j * rng.normal(size=(2, 3, 2, 4))            # [B, R, Tt, L]
    hfull = np.broadcast_to(taps[:, :, :, None, :], (2, 3, 2, 13, 4))
    y = F.apply_time_channel(x, hfull)
    for bb in range(2):
        for r in range(3):
            want = sum(np.convolve(x[bb, t], taps[bb, r, t]) for t in range(2))
            assert np.allclose(y[bb, r], want)


def _interp1_with_linear_extrapolation(xq, xs, ys):
    """Independent 1-D recipe: np.interp inside [xs[0], xs[-1]], straight-line continuation of the first / last segment
    outside; a single support point gives a constant (what the reference's in-test recipe does, test_ofdm_channel_
    estimation.py:17-84)."""
    xs, ys = np.asarray(xs, float), np.asarray(ys)
    if len(xs) == 1:
        return np.full(len(xq), ys[0])
    out = np.interp(xq, xs, ys.real) + 1j * np.interp(xq, xs, ys.imag)
    lo, hi = xq < xs[0], xq > xs[-1]
    out[lo] = ys[0] + (xq[lo] - xs[0]) * (ys[1] - ys[0]) / (xs[1] - xs[0])
    out[hi] = ys[-1] + (xq[hi] - xs[-1]) * (ys[-1] - ys[-2]) / (xs[-1] - xs[-2])
    return out


@pytest.mark.parametrize("pilot_syms", [[2], [2, 11], [0, 5, 13], [3, 4, 9, 10]])
@pytest.mark.parametrize("time_avg", [False, True])
def test_linear_interpolator_random_channels_vs_independent_recipe(pilot_syms, time_avg):
    """oracle.ofdm.lin_interp on RANDOM pilot values (where a wrong bracketing rule shows) for comb pilot patterns of two
    transmitters with zero pilots on each other's combs, against np.interp + explicit edge extrapolation."""
    rng = np.random.default_rng(len(pilot_syms) + 10 * time_avg)
    s_, f_ = 14, 20
    mask = F.kronecker_mask(2, 1, s_, f_, pilot_syms)
    npil = len(pilot_syms) * f_
    pil = np.zeros((2, 1, len(pilot_syms), f_), complex)
    pil[0, 0, :, 0::3] = 1.0                                   # tx 0 sounds subcarriers 0, 3, 6, ...
    pil[1, 0, :, 1::4] = -1j                                   # tx 1 sounds 1, 5, 9, ...
    pil = pil.reshape(2, 1, npil)
    hp = (rng.standard_normal((2, 2, 1, npil)) + 1j * rng.standard_normal((2, 2, 1, npil))) * (np.abs(pil) > 0)
    out = F.lin_interp(hp, mask, pil, time_avg=time_avg)
    fq, sq = np.arange(f_, dtype=float), np.arange(s_, dtype=float)
    for b in range(2):
        for tx in range(2):
            rows = {}
            for k, sym in enumerate(pilot_syms):
                vals = hp[b, tx, 0, k * f_:(k + 1) * f_]
                sup = np.nonzero(np.abs(pil[tx, 0, k * f_:(k + 1) * f_]) > 0)[0]
                rows[sym] = _interp1_with_linear_extrapolation(fq, sup, vals[sup])
            if time_avg:
                avg = sum(rows.values()) / len(rows)
                rows = {sym: avg for sym in rows}
            want = np.stack([_interp1_with_linear_extrapolation(sq, sorted(rows), np.array([rows[s][c] for s in sorted(rows)]))
                             for c in range(f_)], axis=1)
            assert np.allclose(out[b, tx, 0], want, atol=1e-12), (b, tx)


@pytest.mark.parametrize("interp", ["nn", "lin", "lin_time_avg"])
def test_ls_and_interpolation_in_complex64_equal_complex128_to_fp32_rounding(interp):
    """oracle.ofdm.ls_estimate / nn_interp / lin_interp with dtype=np.complex64 evaluate the same sequence in single
    precision (the yardstick the fused front-end's GPU tests measure against): results stay complex64 / float32 and sit
    within fp32 rounding of the complex128 evaluation; the default dtype keeps the complex128 results bit for bit."""
    rng = np.random.default_rng(7)
    mask = F.kronecker_mask(2, 1, 14, 24, [2, 7, 11])
    pil = np.zeros((2, 1, 3, 24), np.complex64)
    pil[0, 0, :, 0::2] = (1 + 1j) / np.sqrt(2)
    pil[1, 0, :, 1::2] = (1 - 1j) / np.sqrt(2)
    pil = pil.reshape(2, 1, -1)
    y = (rng.normal(size=(3, 1, 2, 14, 24)) + 1j * rng.normal(size=(3, 1, 2, 14, 24))).astype(np.complex64)
    no = rng.uniform(0.01, 0.1, size=(3, 1, 2)).astype(np.float32)
    h64, e64 = F.ls_estimate(y.astype(np.complex128), mask, pil, no.astype(np.float64), dtype=np.complex128)
    h32, e32 = F.ls_estimate(y, mask, pil, no, dtype=np.complex64)
    assert h32.dtype == np.complex64 and e32.dtype == np.float32 and h64.dtype == np.complex128 and e64.dtype == np.float64
    h0, e0 = F.ls_estimate(y.astype(np.complex128), mask, pil.astype(np.complex128), no)   # default: as before
    assert np.array_equal(h0, h64) and np.array_equal(e0, e64)
    if interp == "nn":
        r64, r32 = F.nn_interp(h64, mask, pil), F.nn_interp(h32, mask, pil, dtype=np.complex64)
        q64, q32 = F.nn_interp(e64, mask, pil), F.nn_interp(e32, mask, pil, dtype=np.float32)
    else:
        ta = interp == "lin_time_avg"
        r64, r32 = F.lin_interp(h64, mask, pil, ta), F.lin_interp(h32, mask, pil, ta, dtype=np.complex64)
        q64, q32 = F.lin_interp(e64, mask, pil, ta).real, F.lin_interp(e32, mask, pil, ta, dtype=np.complex64).real
        assert np.array_equal(F.lin_interp(h64, mask, pil, ta, dtype=np.complex128), r64)
    assert r32.dtype == np.complex64 and q32.dtype == np.float32
    eps = np.finfo(np.float32).eps
    assert np.abs(r32 - r64).max() <= 8 * eps * np.abs(r64).max()
    assert np.abs(q32 - q64).max() <= 8 * eps * np.abs(q64).max()
    assert np.abs(r32 - r64).max() > 0                                                   # really single precision


def _small_patterns(rng):
    """(mask, pilots) pairs that reach every bracketing rule: Kronecker combs, a pilot symbol with one non-zero pilot,
    zero pilots between non-zero ones, pilots on the first / last symbol and subcarrier, per-stream masks that differ,
    a stream whose pilots sit on one symbol only, S = 1 and F = 1."""
    out = []
    mask = F.kronecker_mask(2, 1, 14, 12, [2, 11])
    pil = np.zeros((2, 1, 2, 12), complex)
    pil[0, 0, :, 0::2], pil[1, 0, :, 1::2] = 1.0, -1j
    out.append((mask, pil.reshape(2, 1, -1)))
    mask = np.zeros((1, 3, 9, 10), bool)
    mask[0, 0, [0, 4], :] = True                                             # 20 pilots each
    mask[0, 1, 8, :] = True
    mask[0, 1, 3, :] = True
    mask[0, 2, :, [0, 9]] = True
    mask[0, 2, 1, 5] = mask[0, 2, 7, 5] = True
    pil = (rng.uniform(0.3, 2.0, (1, 3, 20)) * np.exp(2j * np.pi * rng.uniform(size=(1, 3, 20))))
    pil[0, 0, 1:9] = 0                                                       # symbol 0: pilots on subcarriers 0 and 9 only
    pil[0, 0, 12:] = 0                                                       # symbol 4: one pilot, at subcarrier 1
    pil[0, 0, 10] = 0
    pil[0, 1, 10:] = 0                                                       # stream 1: symbol 3 only
    out.append((mask, pil))
    out.append((np.ones((1, 1, 1, 7), bool), rng.normal(size=(1, 1, 7)) + 1j))        # S = 1
    m1 = np.zeros((1, 2, 6, 1), bool)
    m1[0, 0, [1, 4], 0] = True
    m1[0, 1, [0, 5], 0] = True
    out.append((m1, np.array([[[1.0, 2.0], [0.5j, 0.0]]])))                            # F = 1
    return out


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_vectorised_interpolators_equal_loop_forms(dtype):
    """oracle.ofdm.nn_interp / lin_interp (vectorised, used at thousands of subcarriers) return exactly what the RE-by-RE
    restatements nn_interp_loop / lin_interp_loop return, on every small pattern and in both precisions."""
    rng = np.random.default_rng(11)
    for mask, pil in _small_patterns(rng):
        p = pil.shape[-1]
        x = rng.normal(size=(2, 3) + pil.shape) + 1j * rng.normal(size=(2, 3) + pil.shape)
        for ta in (False, True):
            want = F.lin_interp_loop(x, mask, pil, ta, dtype=dtype)
            got = F.lin_interp(x, mask, pil, ta, dtype=dtype)
            assert got.dtype == want.dtype and np.array_equal(got, want), (mask.shape, ta)
        rdt = np.float32 if dtype == np.complex64 else None
        assert np.array_equal(F.nn_interp(x, mask, pil, dtype=dtype), F.nn_interp_loop(x, mask, pil, dtype=dtype))
        ev = rng.uniform(size=x.shape[:-1] + (p,))
        assert np.array_equal(F.nn_interp(ev, mask, pil, dtype=rdt), F.nn_interp_loop(ev, mask, pil, dtype=rdt))
