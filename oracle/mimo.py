"""Oracle: maximum-likelihood MIMO detection. TEST INFRASTRUCTURE (NumPy). Literal restatements of
/root/reference/src/sionna/phy:
  mimo/detection.py:389-471 (_build_vecs), 473-537 (MaximumLikelihoodDetector.call)   -> build_vecs / ml_detect
  mapping.py:927-967 (SymbolLogits2LLRs), 1045-1059 (LLRs2SymbolLogits)                -> logits_to_llrs / llrs_to_logits
  ofdm/detection.py:126-317, 448-738 (OFDM detector pre- and post-processing)          -> ofdm_ml_detect
``dtype=np.complex128`` is the oracle; ``np.complex64`` evaluates the same sequence in single precision, the reference's
own fp32 error envelope (as ``lmmse_equalizer_f32`` does for the LMMSE tests). Candidates are processed in chunks of
problems so that 65 536-candidate cases fit in host memory.
"""
import numpy as np

from .ofdm import whiten_channel, _ofdm_lmmse


def _rdt(cdt):
    return np.float64 if np.dtype(cdt) == np.complex128 else np.float32


def build_vecs(points, num_streams):
    """_build_vecs (detection.py:389-471): vecs [|C|^K, K] (stream 0 varies slowest), vecs_ind [|C|^K, K] point
    indices, c [|C|^(K-1), K, |C|]: c[:, k, s] = rows of vecs whose stream k carries point s."""
    points = np.asarray(points)
    n = len(points)
    vecs_ind = np.zeros((1, 0), np.int64)
    for _ in range(num_streams):
        vecs_ind = np.concatenate([np.concatenate([np.full((len(vecs_ind), 1), i), vecs_ind], 1) for i in range(n)], 0)
    vecs = points[vecs_ind]
    c = np.stack([np.stack([np.where(vecs_ind[:, j] == i)[0] for j in range(num_streams)], -1) for i in range(n)], -1)
    return vecs, vecs_ind, c


def reduce_logsumexp(x, axis):
    """tf.reduce_logsumexp: log(sum(exp(x - max))) + max, the max replaced by 0 where it is not finite."""
    m = np.max(x, axis=axis, keepdims=True)
    m = np.where(np.isfinite(m), m, np.zeros((), x.dtype))
    with np.errstate(divide="ignore"):
        return (np.log(np.sum(np.exp(x - m), axis=axis, keepdims=True)) + m).squeeze(axis)


def _labels(m):
    return (np.arange(2 ** m)[:, None] >> np.arange(m - 1, -1, -1)) & 1


def llrs_to_logits(llrs, m):
    """LLRs2SymbolLogits (mapping.py:1045-1059): [..., m] -> [..., 2^m], sum_i log_sigmoid(a_ci llr_i)."""
    a = (2 * _labels(m) - 1).astype(llrs.dtype)
    z = llrs[..., None, :] * a
    return np.sum(np.minimum(z, 0) - np.log1p(np.exp(-np.abs(z))), axis=-1)      # log_sigmoid


def logits_to_llrs(logits, m, method):
    """SymbolLogits2LLRs (mapping.py:927-967): LLR_i = reduce over points with label bit i = 1 minus over bit i = 0."""
    red = reduce_logsumexp if method == "app" else (lambda x, axis: np.max(x, axis=axis))
    lab = _labels(m)
    out = [red(logits[..., lab[:, i] == 1], -1) - red(logits[..., lab[:, i] == 0], -1) for i in range(m)]
    return np.stack(out, -1)


def ml_detect(y, h, s, points, method, output, prior=None, hard_out=False, dtype=np.complex128, chunk_bytes=1 << 27):
    """MaximumLikelihoodDetector.call (detection.py:473-537). y [..., M], h [..., M, K], s [..., M, M]; prior: bit LLRs
    [..., K, m] (output "bit") or point logits [..., K, |C|] (output "symbol"). Returns LLRs [..., K, m] (hard: 0/1),
    logits [..., K, |C|] or int indices [..., K]."""
    rdt = _rdt(dtype)
    points = np.asarray(points).astype(dtype)
    npts = len(points)
    m = int(np.log2(npts))
    k = h.shape[-1]
    batch = np.broadcast_shapes(np.shape(y)[:-1], np.shape(h)[:-2], np.shape(s)[:-2])
    mm = h.shape[-2]
    y = np.broadcast_to(np.asarray(y).astype(dtype), batch + (mm,)).reshape(-1, mm)
    h = np.broadcast_to(np.asarray(h).astype(dtype), batch + (mm, k)).reshape(-1, mm, k)
    s = np.broadcast_to(np.asarray(s).astype(dtype), batch + (mm, mm)).reshape(-1, mm, mm)
    if prior is not None:
        prior = np.asarray(prior).astype(rdt)
        if output == "bit":
            prior = llrs_to_logits(prior, m)
        prior = np.broadcast_to(prior, batch + (k, npts)).reshape(-1, k, npts)
    vecs, vecs_ind, c = build_vecs(points, k)
    n = y.shape[0]
    step = max(1, chunk_bytes // (len(vecs) * mm * np.dtype(dtype).itemsize))
    logits = np.empty((n, k, npts), rdt)
    for a in range(0, n, step):
        yw, hw = whiten_channel(y[a:a + step], h[a:a + step], s[a:a + step])
        diff = yw[:, None, :] - np.einsum("nmk,vk->nvm", hw, vecs)
        ex = -np.sum(np.square(np.abs(diff)), axis=-1).astype(rdt)                        # [n, |C|^K]
        if prior is not None:
            ex = ex + np.sum(prior[a:a + step][:, np.arange(k)[None, :], vecs_ind], axis=-1)
        g = ex[:, c]                                                                       # [n, |C|^(K-1), K, |C|]
        logits[a:a + step] = reduce_logsumexp(g, 1) if method == "app" else np.max(g, axis=1)
    if output == "bit":
        llr = logits_to_llrs(logits, m, method)
        out = (llr > 0).astype(rdt) if hard_out else llr
        return out.reshape(batch + (k, m))
    if hard_out:
        return np.argmax(logits, axis=-1).reshape(batch + (k,))
    return logits.reshape(batch + (k, npts))


def ofdm_ml_detect(y_eff, h_hat, err_var, no, mask, sm, points, method, output, prior=None, hard_out=False,
                   dtype=np.complex128):
    """OFDM MaximumLikelihoodDetector(WithPrior).call through the LMMSE oracle's pre- and post-processing
    (``_ofdm_lmmse``: S assembly, stream re-ordering, data-symbol gather), with ``ml_detect`` as the per-element
    detector; each output column travels through it as one "x_hat". prior (the reference's tiling,
    ofdm/detection.py:476-510, is defined for one receiver detecting every stream): bit LLRs [B, tx, st, nd * m] or
    logits [B, tx, st, nd, |C|]. Returns [B, tx, st, nd * m], [B, tx, st, nd, |C|] or [B, tx, st, nd]."""
    rdt = _rdt(dtype)
    b, rx, ant, s_, f_ = y_eff.shape
    tx, st = h_hat.shape[3:5]
    npts = len(points)
    m = int(np.log2(npts))
    nd = s_ * f_ - int(mask[0, 0].sum())
    prior_dt = None
    if prior is not None:
        assert rx == 1 and sm["spr"] == tx * st, "the reference's prior tiling needs one receiver detecting every stream"
        width = m if output == "bit" else npts                           # bit LLRs stay LLRs: ml_detect converts them
        pr = np.asarray(prior).astype(rdt).reshape(b, tx * st, nd, width)
        grid = np.zeros((b, tx * st, s_ * f_, width), rdt)
        data_ind = np.argsort(mask.reshape(tx * st, -1).astype(int), axis=-1, kind="stable")[:, :nd]
        for t in range(tx * st):
            grid[:, t, data_ind[t]] = pr[:, t]
        prior_dt = np.transpose(grid.reshape(b, tx * st, s_, f_, width), [0, 2, 3, 1, 4])[:, None]  # [B, 1, S, F, K, w]
    res = {}

    def detector(y_dt, hd, s):
        if "z" not in res:
            z = ml_detect(y_dt, hd, s, points, method, output, prior_dt, hard_out, dtype)
            res["z"] = z if z.ndim == 6 else z[..., None]                                   # [B, rx, S, F, K, L]
        z = res["z"][..., res["col"]]
        return z, np.zeros(z.shape, rdt)

    cols = []
    width = m if output == "bit" else (1 if hard_out else npts)
    for col in range(width):
        res["col"] = col
        cols.append(_ofdm_lmmse(y_eff, h_hat, err_var, no, mask, sm, dtype, rdt, detector)[0])   # [B, tx, st, nd]
    out = np.stack(cols, -1)
    if output == "bit":
        return out.reshape(b, tx, st, nd * m)
    return out[..., 0] if hard_out else out
