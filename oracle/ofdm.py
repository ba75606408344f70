"""Oracle: OFDM (de)modulation, resource-grid mapping, LS channel estimation + interpolation, OFDM LMMSE equalisation.
TEST INFRASTRUCTURE (NumPy, complex128). Literal restatements of /root/reference/src/sionna/phy:
  ofdm/modulator.py:97-124, ofdm/demodulator.py:129-203, signal/utils.py:161-249   -> ofdm_modulate / ofdm_demodulate
  ofdm/resource_grid.py:283-311, 394-412, 461-520                                  -> type_grid / rg_map / rg_demap
  ofdm/pilot_pattern.py:344-372, 117-124                                           -> kronecker_mask_and_pilots
  ofdm/channel_estimation.py:138-173, 257-285, 384-435, 522-734                    -> ls_estimate / nn_interp / lin_interp
  mimo/stream_management.py:200-246                                                -> stream_management
  ofdm/equalization.py:109-275, mimo/equalization.py:11-233, mimo/utils.py:292-357 -> ofdm_lmmse_equalize / lmmse_equalizer
PARITY: unpinned at bit level (TensorFlow's FFT / Cholesky kernels are not available); pinned by the reference's own
tolerances: FFT round trip 1e-5 (test/unit/ofdm/test_ofdm.py:85-96), interpolators vs NumPy re-implementations
(test/unit/ofdm/test_ofdm_channel_estimation.py), LMMSE statistically (test/unit/mimo/test_mimo_equalizers.py:55-102).
"""
import numpy as np


# ---- OFDM ------------------------------------------------------------------------------------------------------------
def ofdm_modulate(x, cp):
    """x [..., S, N] -> [..., sum(N + cp_l)] (modulator.py:100-124)."""
    n = x.shape[-1]
    cp = np.broadcast_to(np.asarray(cp), (x.shape[-2],))
    t = np.fft.ifft(np.fft.ifftshift(x, axes=-1), axis=-1) * np.sqrt(n)
    out = [np.concatenate([t[..., l, n - cp[l]:], t[..., l, :]], axis=-1) for l in range(x.shape[-2])]
    return np.concatenate(out, axis=-1)


def ofdm_demodulate(x, n, l_min, cp):
    """x [..., T] -> [..., S, N] (demodulator.py:162-203)."""
    cp = np.asarray(cp)
    if cp.ndim == 0:
        nsym = x.shape[-1] // (n + int(cp))
        cp = np.full(nsym, int(cp))
    off = np.concatenate([[0], np.cumsum(n + cp)[:-1]])
    sym = np.stack([x[..., off[l] + cp[l]: off[l] + cp[l] + n] for l in range(len(cp))], axis=-2)
    f = np.fft.fft(sym, axis=-1) / np.sqrt(n)
    tmp = (-2 * np.pi * np.float32(l_min) / np.float32(n) * np.arange(n, dtype=np.float32)).astype(np.float32)
    f = f * np.exp(1j * tmp.astype(np.float64))
    return np.fft.fftshift(f, axes=-1)


# ---- resource grid ---------------------------------------------------------------------------------------------------
def kronecker_mask(num_tx, num_streams, num_sym, num_eff, pilot_syms):
    mask = np.zeros([num_tx, num_streams, num_sym, num_eff], bool)
    mask[..., pilot_syms, :] = True
    return mask


def type_grid(mask, fft_size, guards, dc_null):
    """[tx, st, S, fft] RE types: 0 data, 1 pilot, 2 guard, 3 DC (resource_grid.py:283-311)."""
    shape = list(mask.shape[:3])
    dc_ind = int(fft_size / 2 - (fft_size % 2 == 1) / 2)
    split = dc_ind - guards[0]
    return np.concatenate([2 * np.ones(shape + [guards[0]], np.int32), mask[..., :split].astype(np.int32),
                           3 * np.ones(shape + [int(dc_null)], np.int32), mask[..., split:].astype(np.int32),
                           2 * np.ones(shape + [guards[1]], np.int32)], -1)


def rg_map(x, pilots, tg):
    """x [B, tx, st, D], pilots [tx, st, P], tg type grid -> [B, tx, st, S, fft] (resource_grid.py:394-412)."""
    b = x.shape[0]
    out = np.zeros((b,) + tg.shape, np.complex128)
    for i in range(tg.shape[0]):
        for j in range(tg.shape[1]):
            flat = out[:, i, j].reshape(b, -1)
            t = tg[i, j].reshape(-1)
            flat[:, t == 1] = pilots[i, j][None, :]
            flat[:, t == 0] = x[:, i, j]
            out[:, i, j] = flat.reshape((b,) + tg.shape[2:])
    return out


def eff_sc_ind(fft_size, guards, dc_null):
    ind = np.arange(guards[0], fft_size - guards[1])
    if dc_null:
        dc_ind = int(fft_size / 2 - (fft_size % 2 == 1) / 2)
        ind = np.delete(ind, dc_ind - guards[0])
    return ind


# ---- stream management (mimo/stream_management.py:200-246) -----------------------------------------------------------
def stream_management(assoc, num_streams_per_tx):
    a = np.array(assoc, np.int32)
    num_rx, num_tx = a.shape
    spr = int(num_tx * num_streams_per_tx / num_rx)
    sa = np.zeros([num_rx, num_tx, num_streams_per_tx], np.int32)
    for j in range(num_tx):
        c = 0
        for i in range(num_rx):
            if a[i, j]:
                sa[i, j, c:c + spr] = 1
                c += spr
    rx_ids = np.zeros([num_rx, spr], np.int32)
    for i in range(num_rx):
        c = []
        for j in range(num_tx):
            if a[i, j]:
                c += list(np.where(sa[i, j])[0] + j * num_streams_per_tx)
        rx_ids[i] = c
    return {"desired": np.where(sa.reshape(-1) == 1)[0], "undesired": np.where(sa.reshape(-1) == 0)[0],
            "stream_ind": np.argsort(rx_ids.reshape(-1)), "num_rx": num_rx, "num_tx": num_tx, "spr": spr,
            "spt": num_streams_per_tx}


# ---- LS estimation and interpolation ---------------------------------------------------------------------------------
def _real(dtype):
    return np.finfo(dtype).dtype.type


def ls_estimate(y_eff, mask, pilots, no, dtype=None):
    """y_eff [B, rx, ant, S, F]; mask [tx, st, S, F]; pilots [tx, st, P]; no broadcastable to [B, rx, ant] ->
    h, err [B, rx, ant, tx, st, P] (channel_estimation.py:138-150, 257-285). ``dtype`` (np.complex64 / np.complex128)
    evaluates in that precision; None keeps the inputs' types for h and float64 for err."""
    if dtype is not None:
        y_eff, pilots = np.asarray(y_eff).astype(dtype), np.asarray(pilots).astype(dtype)
    rdt = np.float64 if dtype is None else _real(dtype)
    b, rx, ant = y_eff.shape[:3]
    p = pilots.shape[-1]
    yf = y_eff.reshape(b, rx, ant, -1)
    pil_ind = np.argsort(-mask.reshape(mask.shape[0], mask.shape[1], -1).astype(int), axis=-1, kind="stable")[..., :p]
    yp = yf[..., pil_ind]                                            # [B, rx, ant, tx, st, P]
    with np.errstate(divide="ignore", invalid="ignore"):
        h = np.where(pilots == 0, 0, yp / pilots)
        no_b = np.broadcast_to(np.asarray(no, rdt).reshape(np.shape(no) + (1,) * (3 - np.ndim(no))), (b, rx, ant))
        err = np.where(pilots == 0, 0, no_b[..., None, None, None] / np.abs(pilots) ** 2)
    return h, np.broadcast_to(err, h.shape)


def nn_interp_loop(x, mask, pilots, dtype=None):
    """x [..., tx, st, P] -> [..., tx, st, S, F]: nearest non-zero pilot in Manhattan distance (:384-402), in ``dtype``
    (None: the type of x). One RE at a time, as the reference states it; `nn_interp` is the same, vectorised."""
    tx, st, s_, f_ = mask.shape
    if dtype is not None:
        x = np.asarray(x).astype(dtype)
    out = np.zeros(x.shape[:-1] + (s_, f_), x.dtype)
    for i in range(tx):
        for j in range(st):
            i_p, j_p = np.where(mask[i, j])
            for a in range(s_):
                for c in range(f_):
                    d = np.abs(a - i_p) + np.abs(c - j_p)
                    d[np.abs(pilots[i, j]) == 0] = s_ + f_
                    out[..., i, j, a, c] = x[..., i, j, np.argmin(d)]
    return out


def _lerp(x, x0, x1, y0, y1):
    with np.errstate(divide="ignore", invalid="ignore"):
        slope = np.where(x1 - x0 == 0, 0, (y1 - y0) / (x1 - x0))
    return (x - x0) * slope + y0


def lin_interp_loop(x, mask, pilots, time_avg=False, dtype=np.complex128):
    """x [..., tx, st, P] -> [..., tx, st, S, F] (channel_estimation.py:522-734): per pilot-carrying symbol, linear
    inter/extrapolation over frequency from the two bracketing (or nearest two) non-zero pilots, then the same over time.
    Evaluated in ``dtype`` (positions and slopes in its real type). One RE at a time; `lin_interp` is the same,
    vectorised."""
    tx, st, s_, f_ = mask.shape
    rdt = _real(dtype)
    x = np.asarray(x).astype(dtype)
    out = np.zeros(x.shape[:-1] + (s_, f_), dtype)
    for i in range(tx):
        for j in range(st):
            pil = pilots[i, j]
            pos = np.argwhere(mask[i, j])                            # row-major pilot positions <-> pilot index
            hf = {}
            for a in range(s_):
                idx = [k for k in range(len(pil)) if pos[k][0] == a and np.abs(pil[k]) > 0]
                if not idx:
                    continue
                xs = np.array([pos[k][1] for k in idx])
                row = np.zeros(x.shape[:-1][:-2] + (f_,), dtype)
                for c in range(f_):
                    if len(idx) == 1:
                        k0 = k1 = 0
                    else:
                        k1 = int(np.searchsorted(xs, c, side="left"))          # first pilot position >= c
                        k1 = min(max(k1, 1), len(idx) - 1)
                        k0 = k1 - 1
                    row[..., c] = _lerp(rdt(c), rdt(xs[k0]), rdt(xs[k1]), x[..., i, j, idx[k0]], x[..., i, j, idx[k1]])
                hf[a] = row
            syms = sorted(hf)
            if time_avg:
                avg = sum(hf[a] for a in syms) / len(syms)
                hf = {a: avg for a in syms}
            for a in range(s_):
                if len(syms) == 1:
                    out[..., i, j, a, :] = hf[syms[0]]
                else:
                    k1 = int(np.searchsorted(syms, a, side="left"))
                    k1 = min(max(k1, 1), len(syms) - 1)
                    k0 = k1 - 1
                    out[..., i, j, a, :] = _lerp(rdt(a), rdt(syms[k0]), rdt(syms[k1]), hf[syms[k0]], hf[syms[k1]])
    return out


def nn_interp(x, mask, pilots, dtype=None):
    """x [..., tx, st, P] -> [..., tx, st, S, F]: `nn_interp_loop` with the distances of one OFDM symbol's REs to all
    non-zero pilots at once. A zero pilot's distance S + F exceeds every real one, so it is never the first minimum
    and leaving it out changes nothing: the same result bit for bit."""
    tx, st, s_, f_ = mask.shape
    if dtype is not None:
        x = np.asarray(x).astype(dtype)
    out = np.zeros(x.shape[:-1] + (s_, f_), x.dtype)
    cols = np.arange(f_)[:, None]
    for i in range(tx):
        for j in range(st):
            i_p, j_p = np.where(mask[i, j])
            nz = np.nonzero(np.abs(pilots[i, j]) > 0)[0]
            for a in range(s_):
                d = np.abs(a - i_p[nz])[None, :] + np.abs(cols - j_p[nz][None, :])    # [F, non-zero pilots]
                out[..., i, j, a, :] = x[..., i, j, :][..., nz[np.argmin(d, axis=1)]]
    return out


def lin_interp(x, mask, pilots, time_avg=False, dtype=np.complex128):
    """x [..., tx, st, P] -> [..., tx, st, S, F]: `lin_interp_loop` with the brackets of a whole row (frequency) or
    column (time) found by one searchsorted, and the same element-wise operations (the same result bit for bit)."""
    tx, st, s_, f_ = mask.shape
    rdt = _real(dtype)
    x = np.asarray(x).astype(dtype)
    out = np.zeros(x.shape[:-1] + (s_, f_), dtype)
    c = np.arange(f_)
    for i in range(tx):
        for j in range(st):
            pil = pilots[i, j]
            pos = np.argwhere(mask[i, j])                            # row-major pilot positions <-> pilot index
            nz = np.abs(pil) > 0
            hf = {}
            for a in range(s_):
                idx = np.nonzero((pos[:, 0] == a) & nz)[0]
                if not len(idx):
                    continue
                xs = pos[idx, 1]
                if len(idx) == 1:
                    k0 = k1 = np.zeros(f_, int)
                else:
                    k1 = np.clip(np.searchsorted(xs, c, side="left"), 1, len(idx) - 1)
                    k0 = k1 - 1
                hf[a] = _lerp(c.astype(rdt), xs[k0].astype(rdt), xs[k1].astype(rdt), x[..., i, j, idx[k0]],
                              x[..., i, j, idx[k1]])
            syms = sorted(hf)
            if time_avg:
                avg = sum(hf[a] for a in syms) / len(syms)
                hf = {a: avg for a in syms}
            if len(syms) == 1:
                out[..., i, j, :, :] = hf[syms[0]][..., None, :]
                continue
            t = np.arange(s_)
            k1 = np.clip(np.searchsorted(syms, t, side="left"), 1, len(syms) - 1)
            k0 = k1 - 1
            rows = np.stack([hf[a] for a in syms], axis=-2)           # [..., num pilot symbols, F]
            sy = np.asarray(syms)
            out[..., i, j, :, :] = _lerp(t.astype(rdt)[:, None], sy[k0].astype(rdt)[:, None], sy[k1].astype(rdt)[:, None],
                                         rows[..., k0, :], rows[..., k1, :])
    return out


# ---- LMMSE -----------------------------------------------------------------------------------------------------------
def lmmse_equalizer(y, h, s):
    """mimo/equalization.py:183-233 with whiten_interference=True (mimo/utils.py:343-347, utils/linalg.py:28-32)."""
    l = np.linalg.cholesky(s)
    l_inv = np.linalg.solve(l, np.broadcast_to(np.eye(s.shape[-1]), s.shape))
    y_w = (l_inv @ y[..., None])[..., 0]
    h_w = l_inv @ h
    a = np.conj(np.swapaxes(h_w, -1, -2)) @ h_w + np.eye(h.shape[-1])
    g = np.linalg.solve(a, np.conj(np.swapaxes(h_w, -1, -2)))
    gy = (g @ y_w[..., None])[..., 0]
    d = np.diagonal(g @ h_w, axis1=-2, axis2=-1)
    return gy / d, np.real(1 / d - 1)


def lmmse_equalizer_f32(y, h, s):
    """The same formula sequence evaluated in complex64 / float32 (LAPACK single precision), i.e. with the arithmetic
    precision the reference itself runs at. Not a second oracle: the parity tests use it to MEASURE the reference's own
    fp32 error envelope against the complex128 evaluation above (how far any single-precision evaluation of
    mimo/equalization.py:183-233 sits from the exact result), which is the yardstick the CUDA kernel is held to."""
    y, h, s = y.astype(np.complex64), h.astype(np.complex64), s.astype(np.complex64)
    l = np.linalg.cholesky(s)
    l_inv = np.linalg.solve(l, np.broadcast_to(np.eye(s.shape[-1], dtype=np.complex64), s.shape))
    y_w = (l_inv @ y[..., None])[..., 0]
    h_w = l_inv @ h
    a = np.conj(np.swapaxes(h_w, -1, -2)) @ h_w + np.eye(h.shape[-1], dtype=np.complex64)
    g = np.linalg.solve(a, np.conj(np.swapaxes(h_w, -1, -2)))
    gy = (g @ y_w[..., None])[..., 0]
    d = np.diagonal(g @ h_w, axis1=-2, axis2=-1)
    one = np.float32(1)
    return (gy / d).astype(np.complex64), np.real(one / d - one).astype(np.float32)


def _herm(a):
    return np.conj(np.swapaxes(a, -1, -2))


def _cholesky_solve(a, b):
    """tf.linalg.cholesky_solve(tf.linalg.cholesky(a), b)."""
    l = np.linalg.cholesky(a)
    return np.linalg.solve(_herm(l), np.linalg.solve(l, b))


def inv_cholesky(s):
    """utils/linalg.py:28-32: L^-1 = triangular_solve(chol(s), I). Keeps the precision of s."""
    return np.linalg.solve(np.linalg.cholesky(s), np.broadcast_to(np.eye(s.shape[-1], dtype=s.dtype), s.shape))


def whiten_channel(y, h, s):
    """mimo/utils.py:343-347: (L^-1 y, L^-1 H). Keeps the precision of the inputs."""
    l_inv = inv_cholesky(s)
    return (l_inv @ y[..., None])[..., 0], l_inv @ h


def lmmse_matrix(h, s=None):
    """mimo/equalization.py:76-97: G = (cholesky_solve(H H^H + S, H))^H, or with s None
    G = cholesky_solve(H^H H + I, H^H). Keeps the precision of the inputs."""
    if s is None:
        return _cholesky_solve(_herm(h) @ h + np.eye(h.shape[-1], dtype=h.dtype), _herm(h))
    return _herm(_cholesky_solve(h @ _herm(h) + s, h))


def lmmse_equalizer_cholesky(y, h, s, whiten_interference=True):
    """mimo/equalization.py:183-233 step by step as the reference evaluates it (whitening, then the Cholesky-based
    lmmse_matrix), in the precision of the inputs: complex64 inputs give the reference's own fp32 error envelope."""
    if whiten_interference:
        y, h = whiten_channel(y, h, s)
        g = lmmse_matrix(h)
    else:
        g = lmmse_matrix(h, s)
    d = np.diagonal(g @ h, axis1=-2, axis2=-1)
    one = np.ones((), y.real.dtype)
    return (g @ y[..., None])[..., 0] / d, np.real(one / d - one)


def ofdm_lmmse_equalize(y_eff, h_hat, err_var, no, mask, sm):
    """OFDMEqualizer.call + lmmse_equalizer (ofdm/equalization.py:126-275). y_eff [B, rx, ant, S, F] (effective
    subcarriers), h_hat [B, rx, ant, tx, st, S, F] -> x_hat, no_eff [B, tx, st, num_data]."""
    return _ofdm_lmmse(y_eff, h_hat, err_var, no, mask, sm, np.complex128, np.float64, lmmse_equalizer)


def ofdm_lmmse_equalize_f32(y_eff, h_hat, err_var, no, mask, sm):
    """ofdm_lmmse_equalize with every step in complex64 / float32 (S assembled, then lmmse_equalizer_cholesky): the
    reference's own single-precision error envelope."""
    return _ofdm_lmmse(y_eff, h_hat, err_var, no, mask, sm, np.complex64, np.float32, lmmse_equalizer_cholesky)


def _ofdm_lmmse(y_eff, h_hat, err_var, no, mask, sm, cdt, rdt, equalizer):
    y_eff, h_hat, err_var = y_eff.astype(cdt), h_hat.astype(cdt), np.asarray(err_var).astype(rdt)
    b, rx, ant, s_, f_ = y_eff.shape
    tx, st = h_hat.shape[3:5]
    y_dt = np.transpose(y_eff, [0, 1, 3, 4, 2])
    ev = np.broadcast_to(err_var, h_hat.shape)
    ev = np.transpose(ev, [0, 1, 5, 6, 2, 3, 4]).reshape(b, rx, s_, f_, ant, tx * st)
    h_dt = np.transpose(h_hat, [1, 3, 4, 0, 2, 5, 6]).reshape(rx * tx * st, b, ant, s_, f_)
    hd = h_dt[sm["desired"]].reshape(rx, sm["spr"], b, ant, s_, f_)
    hu = h_dt[sm["undesired"]].reshape(rx, -1, b, ant, s_, f_)
    hd = np.transpose(hd, [2, 0, 4, 5, 3, 1])
    hu = np.transpose(hu, [2, 0, 4, 5, 3, 1])
    no_b = np.broadcast_to(np.asarray(no, rdt).reshape(np.shape(no) + (1,) * (3 - np.ndim(no))), (b, rx, ant))
    no_dt = np.transpose(np.broadcast_to(no_b[..., None, None], (b, rx, ant, s_, f_)), [0, 1, 3, 4, 2])
    s = hu @ np.conj(np.swapaxes(hu, -1, -2))
    idx = np.arange(ant)
    s[..., idx, idx] += no_dt + ev.sum(-1)
    x_hat, no_eff = equalizer(y_dt, hd, s)                             # [B, rx, S, F, K]
    x_hat = np.transpose(x_hat, [1, 4, 2, 3, 0]).reshape(rx * sm["spr"], s_, f_, b)[sm["stream_ind"]]
    no_eff = np.transpose(no_eff, [1, 4, 2, 3, 0]).reshape(rx * sm["spr"], s_, f_, b)[sm["stream_ind"]]
    x_hat = x_hat.reshape(tx, st, s_ * f_, b)
    no_eff = no_eff.reshape(tx, st, s_ * f_, b)
    nd = s_ * f_ - int(mask[0, 0].sum())
    data_ind = np.argsort(mask.reshape(tx, st, -1).astype(int), axis=-1, kind="stable")[..., :nd]
    xo = np.take_along_axis(x_hat, data_ind[..., None], axis=2)
    no_o = np.take_along_axis(no_eff, data_ind[..., None], axis=2)
    return np.transpose(xo, [3, 0, 1, 2]), np.transpose(no_o, [3, 0, 1, 2])


# ---- on-device channel generation (SURVEY.md 8(f3)) ------------------------------------------------------------------
def tdl_sos(doppler, theta, phi, phi0, powers, los_power, los_aoa, num_time_steps, fs, dtype=np.float64):
    """Sum-of-sinusoids tap gains (channel/tr38901/tdl.py:374-456): doppler [B], theta [B, P, Ns], phi [B, A, P, Ns],
    phi0 [B] | None, powers [P] -> a [B, A, P, T], evaluated in the real type ``dtype`` (float64, or float32 for the
    reference's own single-precision evaluation)."""
    rd = np.dtype(dtype).type
    ns = theta.shape[-1]
    t = np.arange(num_time_steps, dtype=rd) / rd(fs)                                    # :374-376
    alpha = rd(2 * np.pi / ns) * np.arange(1, ns + 1, dtype=rd) + theta.astype(rd)      # :286-288, :403
    arg = (doppler.astype(rd)[:, None, None, None, None] * t[None, None, None, :, None]
           * np.cos(alpha)[:, None, :, None, :] + phi.astype(rd)[:, :, :, None, :])               # :415
    h = np.exp(1j * arg).sum(-1) / np.sqrt(rd(ns))                                       # :417-421
    h = np.sqrt(np.asarray(powers, rd))[None, None, :, None] * h                         # :423-424
    if phi0 is not None:                                                                 # :426-448
        spec = np.exp(1j * (doppler.astype(rd)[:, None] * t[None, :] * np.cos(rd(los_aoa))
                            + phi0.astype(rd)[:, None]))
        h[:, :, 0, :] += np.sqrt(rd(los_power)) * spec[:, None, :]
    return h


def _contract(a, e):
    if e.ndim == 2:                                                                      # shared table [P, C]
        return np.einsum("...pt,pf->...tf", a, e)
    return np.einsum("brmtnpl,brtpf->brmtnlf", a, e)                                     # per-link [B, RX, TX, P, C]


def cir_to_ofdm(frequencies, a, tau, dtype=np.complex128):
    """h[..., t, f] = sum_p a[..., p, t] exp(-j 2 pi f tau_p) (channel/utils.py:180-253); a [B, RX, RA, TX, TA, P, T],
    tau [P] or per link [B, RX, TX, P]. In ``dtype``: complex128, or complex64 (the phases still exact in float64 and
    then rounded, as the kernel's table is; the contraction in complex64)."""
    e = np.exp(-2j * np.pi * np.asarray(tau, np.float64)[..., None] * np.asarray(frequencies, np.float64))
    return _contract(np.asarray(a).astype(dtype), e.astype(dtype))


def cir_to_time(bandwidth, a, tau, l_min, l_max, dtype=np.complex128):
    """hm[..., t, l] = sum_p a[..., p, t] sinc(l - tau_p W) (channel/utils.py:320-336); shapes and ``dtype`` as
    cir_to_ofdm."""
    l = np.arange(l_min, l_max + 1, dtype=np.float64)
    g = np.sinc(l - np.asarray(tau, np.float64)[..., None] * bandwidth)                  # [..., P, L]
    return _contract(np.asarray(a).astype(dtype), g.astype(dtype))


def apply_time_channel(x, h, dtype=np.complex128):
    """y[b, r, n] = sum_t sum_l h[b, r, t, n, l] x[b, t, n - l], x zero outside [0, N) (apply_time_channel.py:115-133).
    x [B, Tt, N], h [B, R, Tt, N + L - 1, L] -> [B, R, N + L - 1], in ``dtype``."""
    b, r, tt, no, l_tot = h.shape
    n = x.shape[-1]
    idx = np.arange(no)[:, None] - np.arange(l_tot)[None, :]                             # [NO, L]: n - l
    xp = np.concatenate([np.asarray(x).astype(dtype), np.zeros(x.shape[:-1] + (1,), dtype)], -1)
    xs = xp[..., np.where((idx >= 0) & (idx < n), idx, n)]                              # [B, Tt, NO, L], 0 outside
    return np.einsum("brtnl,btnl->brn", np.asarray(h).astype(dtype), xs)
