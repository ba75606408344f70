"""Oracle: EP and MMSE-PIC MIMO detection. TEST INFRASTRUCTURE (NumPy). Literal restatements of
/root/reference/src/sionna/phy:
  mimo/detection.py:1039-1312 (EPDetector), mimo/utils.py:194-242 (complex2real_channel),
  mapping.py:927-967 (SymbolLogits2LLRs), 1234-1316 (PAM2QAM)                              -> ep_detect
  mimo/detection.py:1314-1643 (MMSEPICDetector), mapping.py:664-691 (Demapper with prior),
  1045-1059 (LLRs2SymbolLogits), 1061-1139 (SymbolLogits2Moments)                         -> mmse_pic_detect
  ofdm/detection.py:20-447, 969-1173 (OFDM wrappers)                                       -> ofdm_ep_detect / ofdm_mmse_pic_detect
with ``np.linalg.inv`` for the reference's ``tf.linalg.inv``. ``dtype=np.complex128`` is the oracle; ``np.complex64``
evaluates the same sequence in single precision, the reference's own fp32 error envelope. The clamps are the
single-precision ones (EP 1e-6, MMSE-PIC 1e-4) in both: the detectors run on fp32 kernels in every precision.
Both also return, per problem, the smallest relative margin of every data-dependent branch: EP's ``lam < 0`` test and its
two ``max(., 1e-6)`` clamps, MMSE-PIC's ``max(1 - v mu, 1e-4)``, and the hard decisions.
"""
import numpy as np

from .kbest import pam2qam
from .mapping import pam
from .mimo import _rdt, _labels, llrs_to_logits, logits_to_llrs, reduce_logsumexp
from .ofdm import whiten_channel, _ofdm_lmmse

EP_PREC = 1e-6
PIC_EPS = 1e-4
TINY = np.finfo(np.float32).tiny


def _rel_gap(a, b):
    return np.abs(b - a) / np.maximum(np.maximum(np.abs(a), np.abs(b)), 1e-300)


def _flat(y, h, s, dtype):
    kk, mm = h.shape[-1], h.shape[-2]
    batch = np.broadcast_shapes(np.shape(y)[:-1], np.shape(h)[:-2], np.shape(s)[:-2])
    y = np.broadcast_to(np.asarray(y).astype(dtype), batch + (mm,)).reshape(-1, mm)
    h = np.broadcast_to(np.asarray(h).astype(dtype), batch + (mm, kk)).reshape(-1, mm, kk)
    s = np.broadcast_to(np.asarray(s).astype(dtype), batch + (mm, mm)).reshape(-1, mm, mm)
    return y, h, s, batch


def _realify(a):
    """complex2real_matrix: [[Re a, -Im a], [Im a, Re a]]."""
    return np.concatenate([np.concatenate([a.real, -a.imag], -1), np.concatenate([a.imag, a.real], -1)], -2)


def _top2_gap(logits):
    srt = np.sort(logits, axis=-1)
    return _rel_gap(srt[..., -1], srt[..., -2])


def ep_levels(num_bits_per_symbol):
    """EPDetector's PAM (detection.py:1156-1161): Constellation("pam", m / 2) / sqrt(2) in float32."""
    return np.real(pam(num_bits_per_symbol // 2) / np.float32(np.sqrt(2.0))).astype(np.float32)


def ep_detect(y, h, s, num_bits_per_symbol, output, hard_out=False, l=10, beta=0.9, dtype=np.complex128):
    """EPDetector.call. y [..., M], h [..., M, K], s [..., M, M]. Returns (out, margin): LLRs / hard bits [..., K, m],
    QAM logits [..., K, 2^m] or int indices [..., K], and margin [...]."""
    rdt = _rdt(dtype)
    m, kk = num_bits_per_symbol, h.shape[-1]
    y, h, s, batch = _flat(y, h, s, dtype)
    n = y.shape[0]
    yw, hw = whiten_channel(y, h, s)
    yr = np.concatenate([yw.real, yw.imag], -1)
    hr = _realify(hw)
    pts = ep_levels(m).astype(rdt)
    es = np.var(pts)
    no = rdt(0.5)
    prec = rdt(EP_PREC)
    hth = np.swapaxes(hr, -1, -2) @ hr
    hty = (np.swapaxes(hr, -1, -2) @ yr[..., None])[..., 0]
    lam = np.ones((n, 2 * kk), rdt) / es
    gam = np.zeros((n, 2 * kk), rdt)
    margin = np.full(n, np.inf)
    eye = np.eye(2 * kk, dtype=rdt)
    for it in range(l):
        sigma = np.linalg.inv(hth + no * lam[:, None, :] * eye)                                # (28), (29)
        mu = (sigma @ (hty + no * gam)[..., None])[..., 0]
        sig = no * np.diagonal(sigma, axis1=-2, axis2=-1)
        vo = 1 / (1 / sig - lam)                                                               # (31), (32)
        margin = np.minimum(margin, _rel_gap(vo, prec).min(-1))
        v_obs = np.maximum(vo, prec)
        x_obs = v_obs * (mu / sig - gam)
        logits = -(x_obs[..., None] - pts) ** 2 / (2 * v_obs[..., None])                       # (33)
        if it == l - 1:                                                                        # the last update is unused
            break
        z = logits - logits.max(-1, keepdims=True)
        pmf = np.exp(z) / np.exp(z).sum(-1, keepdims=True)
        x = np.sum(pts * pmf, -1, keepdims=True)
        vv = np.sum((pts - x) ** 2 * pmf, -1)
        margin = np.minimum(margin, _rel_gap(vv, prec).min(-1))
        v = np.maximum(vv, prec)
        x = x[..., 0]
        lam_n = 1 / v - 1 / v_obs                                                              # (35) - (38)
        gam_n = x / v - x_obs / v_obs
        margin = np.minimum(margin, (np.abs(lam_n) / np.maximum(1 / v, 1 / v_obs)).min(-1))
        neg = lam_n < 0
        lam_new, gam_new = np.where(neg, lam, lam_n), np.where(neg, gam, gam_n)
        lam = ((1 - beta) * lam_new + beta * lam).astype(rdt)
        gam = ((1 - beta) * gam_new + beta * gam).astype(rdt)
    p1, p2 = logits[:, :kk], logits[:, kk:]
    hb = m // 2
    if output == "symbol" and hard_out:
        margin = np.minimum(margin, np.minimum(_top2_gap(p1), _top2_gap(p2)).min(-1))
        out = pam2qam(np.argmax(p1, -1), np.argmax(p2, -1), hb)
        return out.reshape(batch + (kk,)), margin.reshape(batch)
    if output == "symbol":
        nl = 2 ** hb
        flat = (p1[..., :, None] + p2[..., None, :]).reshape(n, kk, nl * nl)
        i, j = np.meshgrid(np.arange(nl), np.arange(nl), indexing="ij")
        gather = pam2qam(i, j, hb).reshape(-1)                                                 # tf.gather(flat, qam_ind)
        return flat[..., gather].reshape(batch + (kk, nl * nl)), margin.reshape(batch)
    lab = _labels(hb)
    l1 = np.stack([np.max(np.where(lab[:, u] == 1, p, -np.inf), -1) for p in (p1, p2) for u in range(hb)], -1)
    l0 = np.stack([np.max(np.where(lab[:, u] == 0, p, -np.inf), -1) for p in (p1, p2) for u in range(hb)], -1)
    llr = (l1 - l0).reshape(n, kk, 2, hb)
    llr = np.swapaxes(llr, -1, -2).reshape(n, kk, m)                                           # stack([llr1, llr2], -1)
    if hard_out:
        margin = np.minimum(margin, _rel_gap(l1, l0).min(-1).min(-1))
        llr = (llr > 0).astype(rdt)
    return llr.reshape(batch + (kk, m)), margin.reshape(batch)


def demap_with_prior(x, no, points, llr_a, method):
    """Demapper(method, with_prior=True).call: x [..., K], no [..., K], llr_a [..., K, m] -> (LLRs [..., K, m], the
    larger magnitude of the two reduced exponents per bit)."""
    m = llr_a.shape[-1]
    no = np.maximum(no, np.asarray(TINY, no.dtype))
    ex = -np.abs(x[..., None] - points) ** 2 / no[..., None] + llrs_to_logits(llr_a, m)
    red = reduce_logsumexp if method == "app" else (lambda v, axis: np.max(v, axis=axis))
    lab = _labels(m)
    l1 = np.stack([red(ex[..., lab[:, i] == 1], -1) for i in range(m)], -1)
    l0 = np.stack([red(ex[..., lab[:, i] == 0], -1) for i in range(m)], -1)
    return l1 - l0, np.maximum(np.abs(l1), np.abs(l0))


def mmse_pic_detect(y, h, s, prior, points, output, method="maxlog", num_iter=1, hard_out=False, dtype=np.complex128):
    """MMSEPICDetector.call. prior: bit LLRs [..., K, m] (output "bit") or point logits [..., K, |C|] (output "symbol");
    None is a zero prior.
    Returns (out, margin): extrinsic LLRs / hard bits [..., K, m], logits [..., K, |C|] or int indices [..., K], and
    margin [...]."""
    rdt = _rdt(dtype)
    points = np.asarray(points).astype(dtype)
    npts, kk = len(points), h.shape[-1]
    m = int(np.log2(npts))
    y, h, s, batch = _flat(y, h, s, dtype)
    n = y.shape[0]
    if prior is None:
        prior = np.zeros((), rdt)
    prior = np.broadcast_to(np.asarray(prior).astype(rdt), batch + (kk, m if output == "bit" else npts))
    prior = prior.reshape(n, kk, -1)
    yw, hw = whiten_channel(y, h, s)
    hh = np.conj(np.swapaxes(hw, -1, -2))
    y_mf = (hh @ yw[..., None])[..., 0]
    g = hh @ hw
    hr = _realify(hw)
    gr = np.swapaxes(hr, -1, -2) @ hr
    llr_a = logits_to_llrs(prior, m, method) if output == "symbol" else prior
    llr_d = llr_a
    margin = np.full(n, np.inf)
    eye = np.eye(2 * kk, dtype=rdt)
    for _ in range(num_iter):
        llr_a = llr_d
        z = llrs_to_logits(llr_a, m)                                                           # SymbolLogits2Moments
        z = z - z.max(-1, keepdims=True)
        p = np.exp(z) / np.exp(z).sum(-1, keepdims=True)
        x_hat = np.sum(p * points, -1)
        var = np.sum(p * np.abs(points - x_hat[..., None]) ** 2, -1).astype(rdt)
        y_pic = y_mf[..., :, None] + g * x_hat[..., None, :] - (g @ x_hat[..., None])           # [n, K, K]
        var2 = np.concatenate([var, var], -1)
        a_inv = np.linalg.inv(gr * var2[..., None, :] + eye)
        mu = np.sum(a_inv * np.swapaxes(gr, -1, -2), -1)
        yt = np.swapaxes(y_pic, -1, -2)
        yt = np.concatenate([yt.real, yt.imag], -1)
        yt = np.concatenate([yt, yt], -2)
        xr = np.sum(a_inv * yt, -1) / mu
        x_t = xr[..., :kk] + 1j * xr[..., kk:]
        d = 1 - var2 * mu
        margin = np.minimum(margin, _rel_gap(d, rdt(PIC_EPS)).min(-1))
        var_x = (mu / np.maximum(d, rdt(PIC_EPS)))[..., :kk]
        llr_d, scale = demap_with_prior(x_t.astype(dtype), (1 / var_x).astype(rdt), points, llr_a, method)
    llr_e = llr_d - llr_a
    if output == "symbol":
        logits = llrs_to_logits(llr_e, m)
        if hard_out:
            margin = np.minimum(margin, _top2_gap(logits).min(-1))
            return np.argmax(logits, -1).reshape(batch + (kk,)), margin.reshape(batch)
        return logits.reshape(batch + (kk, npts)), margin.reshape(batch)
    if hard_out:
        margin = np.minimum(margin, (np.abs(llr_e) / np.maximum(np.maximum(scale, np.abs(llr_a)), 1e-300)).min(-1).min(-1))
        llr_e = (llr_e > 0).astype(rdt)
    return llr_e.reshape(batch + (kk, m)), margin.reshape(batch)


def _ofdm(y_eff, h_hat, err_var, no, mask, sm, dtype, detect, width, prior=None):
    """An OFDM detector through the LMMSE oracle's pre- and post-processing (``_ofdm_lmmse``: S assembly, stream
    re-ordering, data-symbol gather), with ``detect(y, h, s, prior) -> (out [..., K, width] or [..., K], margin)`` as
    the per-element detector; each output column and the margin travel through it as one "x_hat". prior (the
    reference's tiling, one receiver detecting every stream): [B, tx, st, nd, w]. Returns (out [B, tx, st, nd, width],
    margin [B, tx, st, nd])."""
    rdt = _rdt(dtype)
    b, rx, ant, s_, f_ = y_eff.shape
    tx, st = h_hat.shape[3:5]
    nd = s_ * f_ - int(mask[0, 0].sum())
    prior_dt = None
    if prior is not None:
        assert rx == 1 and sm["spr"] == tx * st, "the reference's prior tiling needs one receiver detecting every stream"
        w = prior.shape[-1]
        pr = np.asarray(prior).astype(rdt).reshape(b, tx * st, nd, w)
        grid = np.zeros((b, tx * st, s_ * f_, w), rdt)
        data_ind = np.argsort(mask.reshape(tx * st, -1).astype(int), axis=-1, kind="stable")[:, :nd]
        for t in range(tx * st):
            grid[:, t, data_ind[t]] = pr[:, t]
        prior_dt = np.transpose(grid.reshape(b, tx * st, s_, f_, w), [0, 2, 3, 1, 4])[:, None]     # [B, 1, S, F, K, w]
    res = {}

    def detector(y_dt, hd, s):
        if "z" not in res:
            z, g = detect(y_dt, hd, s, prior_dt)
            z = z if z.ndim == 6 else z[..., None]                                              # [B, rx, S, F, K, L]
            g = np.broadcast_to(g[..., None, None], z.shape[:-1] + (1,))
            res["z"] = np.concatenate([z.astype(np.float64), g], -1)
        z = res["z"][..., res["col"]]
        return z, np.zeros(z.shape, rdt)

    cols = []
    for col in list(range(width)) + [width]:
        res["col"] = col
        cols.append(np.real(_ofdm_lmmse(y_eff, h_hat, err_var, no, mask, sm, dtype, rdt, detector)[0]))
    return np.stack(cols[:-1], -1), cols[-1]


def _ofdm_out(out, margin, output, hard_out, width):
    b, tx, st, nd = margin.shape
    if output == "bit":
        return out.reshape(b, tx, st, nd * width), margin
    return (out[..., 0].astype(np.int64), margin) if hard_out else (out, margin)


def ofdm_ep_detect(y_eff, h_hat, err_var, no, mask, sm, num_bits_per_symbol, output, hard_out=False, l=10, beta=0.9,
                   dtype=np.complex128):
    """OFDM EPDetector.call. Returns ([B, tx, st, nd * m], [B, tx, st, nd, 2^m] or [B, tx, st, nd], margin
    [B, tx, st, nd])."""
    m = num_bits_per_symbol
    width = m if output == "bit" else (1 if hard_out else 2 ** m)
    out, margin = _ofdm(y_eff, h_hat, err_var, no, mask, sm, dtype,
                        lambda y, h, s, _: ep_detect(y, h, s, m, output, hard_out, l, beta, dtype), width)
    return _ofdm_out(out, margin, output, hard_out, width)


def ofdm_mmse_pic_detect(y_eff, h_hat, err_var, no, mask, sm, prior, points, output, method="maxlog", num_iter=1,
                         hard_out=False, dtype=np.complex128):
    """OFDM MMSEPICDetector.call; prior: bit LLRs [B, tx, st, nd * m] or logits [B, tx, st, nd, |C|], or None (a zero
    prior, for any stream management)."""
    m = int(np.log2(len(points)))
    b, tx, st = h_hat.shape[0], h_hat.shape[3], h_hat.shape[4]
    nd = y_eff.shape[3] * y_eff.shape[4] - int(mask[0, 0].sum())
    pr = None if prior is None else np.asarray(prior).reshape(b, tx, st, nd, m if output == "bit" else len(points))
    width = m if output == "bit" else (1 if hard_out else len(points))
    out, margin = _ofdm(y_eff, h_hat, err_var, no, mask, sm, dtype,
                        lambda y, h, s, p: mmse_pic_detect(y, h, s, p, points, output, method, num_iter, hard_out,
                                                           dtype), width, pr)
    return _ofdm_out(out, margin, output, hard_out, width)
