"""Oracle: K-Best MIMO detection. TEST INFRASTRUCTURE (NumPy). Literal restatement of
/root/reference/src/sionna/phy:
  mimo/detection.py:539-1037 (KBestDetector), mimo/utils.py:194-242 (complex2real_channel), 420-577 (List2LLRSimple),
  mapping.py:1234-1320 (PAM2QAM)                                                        -> kbest_detect
  ofdm/detection.py:20-317, 849-967 (OFDM wrapper)                                      -> ofdm_kbest_detect
with ``np.linalg.qr`` (Householder, as TF) and stable sorts. ``dtype=np.complex128`` is the oracle; ``np.complex64``
evaluates the same sequence in single precision, the reference's own fp32 error envelope. Both also return, per problem,
the smallest relative gap that decided anything: between adjacent sorted column norms, between the k-th and (k+1)-th
child metric of every pruning layer, and between the two best final paths (the hard decision).
"""
import numpy as np

from .mapping import pam
from .mimo import _rdt
from .ofdm import whiten_channel, _ofdm_lmmse


def pam_points(num_bits):
    """The real-valued representation's constellation (detection.py:728-734): unnormalised PAM scaled to energy 0.5
    (in float64 here, so that ``qam_from_pam`` gives exactly its QAM)."""
    c = pam(num_bits, normalize=False).astype(np.complex128)
    return np.real(c / (np.std(c) * np.sqrt(2)))


def pam2qam(re, im, num_bits_per_dim):
    """PAM2QAM (mapping.py:1274-1302): QAM index whose even label bits (MSB first) are re's and odd ones im's."""
    out = np.zeros(np.shape(re), np.int64)
    m = 2 * num_bits_per_dim
    for t in range(num_bits_per_dim):
        out |= ((re >> (num_bits_per_dim - 1 - t)) & 1) << (m - 1 - 2 * t)
        out |= ((im >> (num_bits_per_dim - 1 - t)) & 1) << (m - 2 - 2 * t)
    return out


def qam_from_pam(num_bits):
    """The unit-energy QAM whose real and imaginary parts are pam_points(num_bits // 2), by label (float64)."""
    n = num_bits // 2
    p = pam_points(n)
    re, im = np.meshgrid(np.arange(2 ** n), np.arange(2 ** n), indexing="ij")
    q = np.zeros(2 ** num_bits, np.complex128)
    q[pam2qam(re, im, n)] = p[re] + 1j * p[im]
    return q


def _rel_gap(a, b):
    return np.abs(b - a) / np.maximum(np.maximum(np.abs(a), np.abs(b)), 1e-300)


def kbest_detect(y, h, s, points, k, output, hard_out=False, real_rep=False, llr_clip=20.0, dtype=np.complex128):
    """KBestDetector.call. y [..., M], h [..., M, K], s [..., M, M]; points: the complex constellation (its size sets the
    output bits m; with real_rep its PAM companion is used). Returns (out, gap): LLRs / hard bits [..., K, m], int
    indices [..., K] (output "symbol", hard_out), and gap [...]."""
    rdt = _rdt(dtype)
    points = np.asarray(points).astype(dtype)
    m = int(np.log2(len(points)))
    kk = h.shape[-1]
    mm = h.shape[-2]
    batch = np.broadcast_shapes(np.shape(y)[:-1], np.shape(h)[:-2], np.shape(s)[:-2])
    y = np.broadcast_to(np.asarray(y).astype(dtype), batch + (mm,)).reshape(-1, mm)
    h = np.broadcast_to(np.asarray(h).astype(dtype), batch + (mm, kk)).reshape(-1, mm, kk)
    s = np.broadcast_to(np.asarray(s).astype(dtype), batch + (mm, mm)).reshape(-1, mm, mm)
    n = y.shape[0]
    if real_rep:                                            # complex2real_channel
        y = np.concatenate([y.real, y.imag], -1)
        h = np.concatenate([np.concatenate([h.real, -h.imag], -1), np.concatenate([h.imag, h.real], -1)], -2)
        s = np.concatenate([np.concatenate([s.real, -s.imag], -1), np.concatenate([s.imag, s.real], -1)], -2) / 2
        pts = pam_points(m // 2).astype(rdt)
        md = m // 2
    else:
        pts = points
        md = m
    S = h.shape[-1]
    npts = len(pts)
    yw, hw = whiten_channel(y, h, s)
    norms = np.sum(np.abs(hw) ** 2, axis=-2)                # [n, S]
    if real_rep:                                            # one norm per complex column: k sorts before K + k
        norms[:, kk:] = norms[:, :kk]
    order = np.argsort(-norms, axis=-1, kind="stable")
    sn = np.take_along_axis(norms, order, -1)
    gap = np.full(n, np.inf)
    if real_rep:
        sc = -np.sort(-norms[:, :kk], axis=-1)
        if kk > 1:
            gap = np.minimum(gap, _rel_gap(sc[:, :-1], sc[:, 1:]).min(-1))
    elif S > 1:
        gap = np.minimum(gap, _rel_gap(sn[:, :-1], sn[:, 1:]).min(-1))
    hs = np.take_along_axis(hw, order[:, None, :], -1)
    q, r = np.linalg.qr(hs)
    yb = np.einsum("nms,nm->ns", np.conj(q), yw)
    k = min(k, npts ** S)
    paths = np.zeros((n, 1, S), np.int64)
    dists = np.zeros((n, 1), rdt)
    ar = np.arange(n)[:, None]
    for i in range(S - 1, -1, -1):                          # streams processed last row first
        npar = paths.shape[1]
        b = yb[:, i, None] - np.sum(r[:, i, None, i + 1:] * pts[paths[:, :, i + 1:]], -1)          # [n, npar]
        d = dists[..., None] + np.abs(b[..., None] - r[:, i, i, None, None] * pts) ** 2           # [n, npar, |C|]
        d = d.reshape(n, npar * npts).astype(rdt)
        srt = np.argsort(d, axis=-1, kind="stable")         # (metric, candidate index): top_k's order
        need = min(k, npar * npts)
        ds = np.take_along_axis(d, srt, -1)
        if need < npar * npts:
            gap = np.minimum(gap, _rel_gap(ds[:, need - 1], ds[:, need]))
        sel = srt[:, :need]
        par, pt = sel // npts, sel % npts
        paths = paths[ar, par]
        paths[:, :, i] = pt
        dists = ds[:, :need]
    if dists.shape[1] > 1:
        gap = np.minimum(gap, _rel_gap(dists[:, 0], dists[:, 1]))
    unsort = np.argsort(order, axis=-1)
    if hard_out:
        x = np.take_along_axis(paths[:, 0], unsort, -1)   # [n, S] detection-domain indices in stream order
        if real_rep:
            x = pam2qam(x[:, :kk], x[:, kk:], md)
        if output == "bit":
            out = ((x[..., None] >> np.arange(m - 1, -1, -1)) & 1).astype(rdt)
            return out.reshape(batch + (kk, m)), gap.reshape(batch)
        return x.reshape(batch + (kk,)), gap.reshape(batch)
    if real_rep:
        dists = dists / 2
    bits = (paths[..., None] >> np.arange(md - 1, -1, -1)) & 1                                      # [n, k, S, md]
    dd = dists[:, :, None, None]
    l0 = np.min(np.where(bits == 0, dd, np.inf), axis=1)
    l1 = np.min(np.where(bits == 1, dd, np.inf), axis=1)
    llr = np.clip(l0 - l1, -llr_clip, llr_clip).astype(rdt)                                         # [n, S, md]
    llr = np.take_along_axis(llr, unsort[..., None], 1)
    if real_rep:
        llr = np.stack([llr[:, :kk], llr[:, kk:]], -1).reshape(n, kk, m)
    return llr.reshape(batch + (kk, m)), gap.reshape(batch)


def ofdm_kbest_detect(y_eff, h_hat, err_var, no, mask, sm, points, k, output, hard_out=False, real_rep=False,
                      llr_clip=20.0, dtype=np.complex128):
    """OFDM KBestDetector.call through the LMMSE oracle's pre- and post-processing (``_ofdm_lmmse``: S assembly, stream
    re-ordering, data-symbol gather), with ``kbest_detect`` as the per-element detector; each output column travels
    through it as one "x_hat", the element's gap as one more. Returns ([B, tx, st, nd * m] or [B, tx, st, nd],
    gap [B, tx, st, nd])."""
    rdt = _rdt(dtype)
    b, rx, ant, s_, f_ = y_eff.shape
    tx, st = h_hat.shape[3:5]
    m = int(np.log2(len(points)))
    nd = s_ * f_ - int(mask[0, 0].sum())
    res = {}

    def detector(y_dt, hd, s):
        if "z" not in res:
            z, g = kbest_detect(y_dt, hd, s, points, k, output, hard_out, real_rep, llr_clip, dtype)
            z = z if z.ndim == 6 else z[..., None]                                                  # [B, rx, S, F, K, L]
            g = np.broadcast_to(g[..., None, None], z.shape[:-1] + (1,))
            res["z"] = np.concatenate([z.astype(np.float64), g], -1)
        z = res["z"][..., res["col"]]
        return z, np.zeros(z.shape, rdt)

    width = m if output == "bit" else 1
    cols = []
    for col in list(range(width)) + [width]:
        res["col"] = col
        cols.append(_ofdm_lmmse(y_eff, h_hat, err_var, no, mask, sm, dtype, rdt, detector)[0])       # [B, tx, st, nd]
    out = np.real(np.stack(cols[:-1], -1))
    gap = np.real(cols[-1])
    if output == "bit":
        return out.reshape(b, tx, st, nd * m), gap
    return out[..., 0].astype(np.int64), gap
