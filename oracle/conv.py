"""NumPy restatement of the convolutional codes (reference fec/conv/{utils,encoding,decoding}.py), test infrastructure.

`trellis` builds the reference's tables from its construction rules. `encode` runs the shift register serially.
`viterbi` is the reference's add-compare-select in the given dtype: with float32 it performs the kernel's operations in
the kernel's order (branch metric summed over j = 0 ... n - 1, one add per branch, strict < picks the second
predecessor), so `csrc/conv.cu` must equal it bit for bit. `bcjr` in float64 is the reference's formulation ("map" in
the probability domain with per-step normalisation, "log" with logsumexp, "maxlog" with max); in float32 it is the
single-precision evaluation of the same function that `parity.envelope` measures the kernel against ("map" in the log
domain there, where it cannot overflow)."""
import numpy as np


def trellis(gen_poly, rsc=False):
    """dict of int arrays: to_nodes, from_nodes, op_by_tonode, ip_by_tonode, op_by_fromnode ([ns, 2]), and ns, conv_n,
    mu, polys (integers, first character = MSB)."""
    K, n = len(gen_poly[0]), len(gen_poly)
    mu, ns = K - 1, 1 << (K - 1)
    polys = [int(p, 2) for p in gen_poly]
    fb = polys[0] & (ns - 1)
    t = {name: np.full((ns, 2), -1, np.int64) for name in
         ("to_nodes", "from_nodes", "op_by_tonode", "ip_by_tonode", "op_by_fromnode")}
    cnt = np.zeros(ns, np.int64)
    for b in range(2):
        for s in range(ns):
            new = b ^ (bin(s & fb).count("1") & 1) if rsc else b
            reg = (new << mu) | s
            nxt = reg >> 1
            op = 0
            for p in polys:
                op = (op << 1) | (bin(reg & p).count("1") & 1)
            t["to_nodes"][s, b] = nxt
            t["op_by_fromnode"][s, b] = op
            t["from_nodes"][nxt, cnt[nxt]] = s
            t["op_by_tonode"][nxt, cnt[nxt]] = op
            t["ip_by_tonode"][nxt, cnt[nxt]] = b
            cnt[nxt] += 1
    t.update(ns=ns, conv_n=n, mu=mu, polys=polys)
    return t


def _sym_bits(op, n):
    """[..., n] bits of output symbols, most significant first."""
    return (np.asarray(op)[..., None] >> np.arange(n - 1, -1, -1)) & 1


def encode(u, gen_poly, rsc=False, terminate=False):
    """Codewords [B, (k + mu * terminate) * n] (float64) of bits u [B, k]."""
    tr = trellis(gen_poly, rsc)
    u = np.asarray(u).astype(np.int64).reshape(-1, np.shape(u)[-1])
    B, k = u.shape
    fb = tr["polys"][0] & (tr["ns"] - 1)
    st = np.zeros(B, np.int64)
    out = []
    for t in range(k + (tr["mu"] if terminate else 0)):
        if t < k:
            b = u[:, t] & 1
        elif rsc:
            b = np.array([bin(s & fb).count("1") & 1 for s in st])
        else:
            b = np.zeros(B, np.int64)
        out.append(_sym_bits(tr["op_by_fromnode"][st, b], tr["conv_n"]))
        st = tr["to_nodes"][st, b]
    return np.concatenate(out, axis=1).astype(np.float64)


def _branch_metrics(y, n, mode, dtype):
    """[B, T, 2^n] metrics of every output symbol, summed over the n bits in order, in `dtype`."""
    B = y.shape[0]
    y = y.reshape(B, -1, n).astype(dtype)
    bits = _sym_bits(np.arange(1 << n), n)                       # [2^n, n]
    acc = None
    for j in range(n):
        v = y[:, :, j][:, :, None]
        if mode == "soft_llr":
            term = np.where(bits[:, j] == 1, -v, v)
        elif mode == "hard":
            yb = np.mod(np.abs(np.round(v)), dtype(2))           # np.round: half to even, as tf.math.round
            term = np.abs(yb - bits[:, j].astype(dtype))
        else:                                                    # BCJR: 0.5 (-llr) (1 - 2 b)
            h = dtype(0.5) * v
            term = np.where(bits[:, j] == 1, h, -h)
        acc = term if acc is None else (acc + term).astype(dtype)
    return acc.astype(dtype)


def viterbi(llr, gen_poly, rsc=False, terminate=False, method="soft_llr", return_info_bits=True, dtype=np.float64):
    """Viterbi decoding of logits [B, n] (decoding.py:236-453) in `dtype`; info bits [B, k] or codeword [B, n]."""
    tr = trellis(gen_poly, rsc)
    ns, n, mu = tr["ns"], tr["conv_n"], tr["mu"]
    llr = np.asarray(llr).reshape(-1, np.shape(llr)[-1])
    B, T = llr.shape[0], llr.shape[1] // n
    bm = _branch_metrics(llr, n, method, dtype)
    pm = np.full((B, ns), dtype(2.0 ** 20), dtype)
    pm[:, 0] = 0
    fr, opt = tr["from_nodes"], tr["op_by_tonode"]
    dec = np.zeros((T, B, ns), bool)
    for t in range(T):
        m0 = (pm[:, fr[:, 0]] + bm[:, t, opt[:, 0]]).astype(dtype)
        m1 = (pm[:, fr[:, 1]] + bm[:, t, opt[:, 1]]).astype(dtype)
        dec[t] = m1 < m0
        pm = np.where(dec[t], m1, m0)
    s = np.zeros(B, np.int64) if terminate else np.argmin(pm, axis=1)
    ip = np.zeros((B, T), np.int64)
    op = np.zeros((B, T), np.int64)
    rows = np.arange(B)
    for t in range(T - 1, -1, -1):
        slot = dec[t, rows, s].astype(np.int64)
        ip[:, t] = tr["ip_by_tonode"][s, slot]
        op[:, t] = opt[s, slot]
        s = fr[s, slot]
    if return_info_bits:
        return ip[:, :T - (mu if terminate else 0)].astype(np.float64)
    return _sym_bits(op, n).reshape(B, T * n).astype(np.float64)


def _lse(a, b, maxlog):
    if maxlog:
        return np.maximum(a, b)
    with np.errstate(invalid="ignore"):
        return np.logaddexp(a, b)


def _lse_axis(x, maxlog):
    m = np.max(x, axis=-1)
    if maxlog:
        return m
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ms = np.where(np.isfinite(m), m, 0)
        return ms + np.log(np.sum(np.exp(x - ms[..., None]), axis=-1))


def bcjr(llr_ch, gen_poly, rsc=False, terminate=False, algorithm="map", llr_a=None, dtype=np.float64):
    """APP logits (Sionna's sign) of the input bits of all T steps [B, T] (decoding.py:694-943) in `dtype`."""
    tr = trellis(gen_poly, rsc)
    ns, n = tr["ns"], tr["conv_n"]
    llr_ch = np.asarray(llr_ch).reshape(-1, np.shape(llr_ch)[-1])
    B, T = llr_ch.shape[0], llr_ch.shape[1] // n
    la = np.zeros((B, T), dtype) if llr_a is None else np.asarray(llr_a).reshape(B, T).astype(dtype)
    bm = _branch_metrics(llr_ch, n, "bcjr", dtype)               # [B, T, 2^n]
    ha = (dtype(0.5) * -la).astype(dtype)                        # internal sign: log p(0) / p(1)
    sign = np.array([1, -1], dtype)
    to, opf = tr["to_nodes"], tr["op_by_fromnode"]
    # gamma[t][:, j, b] = 0.5 la_t (1 - 2 b) + bm_t[op(j, b)]
    if algorithm == "map" and dtype == np.float64:
        with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
            eb = np.exp(bm)
            alpha = np.zeros((T + 1, B, ns), dtype)
            alpha[0, :, 0] = 1
            for t in range(T):
                g = np.exp(ha[:, t, None, None] * sign) * eb[:, t][:, opf]
                nxt = np.zeros((B, ns), dtype)
                for b in range(2):
                    np.add.at(nxt.T, to[:, b], (alpha[t] * g[:, :, b]).T)
                alpha[t + 1] = nxt / nxt.sum(axis=1, keepdims=True)
            beta = np.zeros((B, ns), dtype)
            if terminate:
                beta[:, 0] = 1
            else:
                beta[:] = 1.0 / ns
            out = np.zeros((B, T), dtype)
            for t in range(T - 1, -1, -1):
                g = np.exp(ha[:, t, None, None] * sign) * eb[:, t][:, opf]
                bn = beta[:, to]                                 # [B, ns, 2]
                p = alpha[t][:, :, None] * g * bn
                out[:, t] = -np.log(p[:, :, 0].sum(1) / p[:, :, 1].sum(1))
                nb = (g * bn).sum(axis=2)
                beta = nb / nb.sum(axis=1, keepdims=True)
        return out
    maxlog = algorithm == "maxlog"
    alpha = np.full((T + 1, B, ns), -np.inf, dtype)
    alpha[0, :, 0] = 0
    fr, ipt = tr["from_nodes"], tr["ip_by_tonode"]
    for t in range(T):
        g = (ha[:, t, None, None] * sign + bm[:, t][:, opf]).astype(dtype)        # [B, ns(from), 2]
        a0 = (alpha[t][:, fr[:, 0]] + g[:, fr[:, 0], ipt[:, 0]]).astype(dtype)
        a1 = (alpha[t][:, fr[:, 1]] + g[:, fr[:, 1], ipt[:, 1]]).astype(dtype)
        alpha[t + 1] = _lse(a0, a1, maxlog).astype(dtype)
    beta = np.full((B, ns), -np.inf if terminate else np.log(1.0 / ns), dtype)
    if terminate:
        beta[:, 0] = 0
    out = np.zeros((B, T), dtype)
    for t in range(T - 1, -1, -1):
        g = (ha[:, t, None, None] * sign + bm[:, t][:, opf]).astype(dtype)
        bn = beta[:, to]
        e = (g + bn).astype(dtype)
        p = (alpha[t][:, :, None] + e).astype(dtype)
        with np.errstate(invalid="ignore"):
            out[:, t] = (_lse_axis(p[:, :, 1], maxlog) - _lse_axis(p[:, :, 0], maxlog)).astype(dtype)
        beta = _lse(e[:, :, 0], e[:, :, 1], maxlog).astype(dtype)
    return out
