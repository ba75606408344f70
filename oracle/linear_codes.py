"""NumPy restatement of sionna.phy.fec.linear and the matrix utilities it uses (fec/utils.py:650-1113,
fec/linear/encoding.py, fec/linear/decoding.py): the reference's OSD step by step (float32 softplus metric, row-wise
pivot rule), a float64 discrepancy form of the same decoder, and brute-force ML decoding for small k."""
import itertools

import numpy as np


def alist2mat(alist):
    n, m = alist[0][0], alist[0][1]
    pcm = np.zeros((m, n), int)
    for v in range(n):
        for i in range(alist[2][v]):
            pcm[alist[4 + v][i] - 1, v] = 1
    return pcm, n - m, n, (n - m) / n


def make_systematic(mat, is_pcm=False):
    """Loop form of fec/utils.py:797-906; returns (mat_sys, column_swaps), ValueError if not of full rank."""
    mat = np.array(mat, dtype=bool)
    m, n = mat.shape
    swaps = []
    for c in range(m):
        ok = bool(mat[c, c])
        if not ok:
            for r in range(c + 1, m):
                if mat[r, c]:
                    mat[[c, r]] = mat[[r, c]]
                    ok = True
                    break
        if not ok:
            for cc in range(c + 1, n):
                if mat[c, cc]:
                    mat[:, [c, cc]] = mat[:, [cc, c]]
                    swaps.append([c, cc])
                    ok = True
                    break
        if not ok:
            raise ValueError("not full rank")
        for r in range(c + 1, m):
            if mat[r, c]:
                mat[r] ^= mat[c]
    for c in range(m - 1, -1, -1):
        for r in range(c - 1, -1, -1):
            if mat[r, c]:
                mat[r] ^= mat[c]
    if is_pcm:
        for i in range(n - 1, n - 1 - m, -1):
            j = i - (n - m)
            mat[:, [i, j]] = mat[:, [j, i]]
            swaps.append([i, j])
    return mat.astype(int), swaps


def pcm2gm(pcm):
    n = pcm.shape[1]
    k = n - pcm.shape[0]
    s, swaps = make_systematic(pcm, is_pcm=True)
    gm = np.concatenate([np.eye(k, dtype=int), s[:, :k].T], axis=1)
    for a, b in swaps[::-1]:
        gm[:, [a, b]] = gm[:, [b, a]]
    return gm


def gm2pcm(gm):
    k, n = gm.shape
    s, swaps = make_systematic(gm)
    pcm = np.concatenate([s[:, k:].T, np.eye(n - k, dtype=int)], axis=1)
    for a, b in swaps[::-1]:
        pcm[:, [a, b]] = pcm[:, [b, a]]
    return pcm


def encode(u, gm):
    """c = u G mod 2 over the last axis."""
    return (np.asarray(u, np.int64) @ np.asarray(gm, np.int64)) % 2


def gf2_rank(mat):
    a = np.array(mat, dtype=bool)
    r = 0
    for c in range(a.shape[1]):
        rows = np.flatnonzero(a[r:, c])
        if rows.size == 0:
            continue
        p = r + rows[0]
        a[[r, p]] = a[[p, r]]
        others = np.flatnonzero(a[:, c])
        others = others[others != r]
        a[others] ^= a[r]
        r += 1
        if r == a.shape[0]:
            break
    return r


def mrb_row_pivot(gm_sorted):
    """The reference's _find_mrb pivot rule (decoding.py:318-398): row c's pivot is its first 1, eliminated from every
    other row. Returns (pivot columns in row order, systematic matrix)."""
    g = np.array(gm_sorted, dtype=bool)
    k = g.shape[0]
    piv = []
    for c in range(k):
        p = int(np.argmax(g[c]))
        piv.append(p)
        rows = np.flatnonzero(g[:, p])
        rows = rows[rows != c]
        g[rows] ^= g[c]
    return piv, g


def mrb_greedy(gm_sorted):
    """Columns kept by walking the sorted columns and keeping each one independent of those kept so far."""
    k, n = gm_sorted.shape
    keep, basis = [], []                                   # basis: reduced column vectors as ints with pivot bits
    for j in range(n):
        v = int("".join(str(int(b)) for b in gm_sorted[:, j]), 2)
        for b, top in basis:
            if v >> top & 1:
                v ^= b
        if v:
            basis.append((v, v.bit_length() - 1))
            keep.append(j)
            if len(keep) == k:
                break
    return keep


def _softplus32(x):
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore"):
        return np.log(np.float32(1) + np.exp(x)).astype(np.float32)


def osd_literal(llr, gm, t):
    """The reference's OSD (decoding.py:253-478) for one codeword: float32 clip, stable sort, row-pivot MRB, float32
    softplus mean metric, strict improvement across orders and the first minimum within one. Returns the codeword."""
    gm = np.asarray(gm, np.int64)
    k, n = gm.shape
    l = np.clip(np.asarray(llr, np.float32), -100, 100).astype(np.float32)
    idx = np.argsort(-np.abs(l), kind="stable")
    piv, g = mrb_row_pivot(gm[:, idx])
    par = [j for j in range(n) if j not in set(piv)]
    order = np.array(piv + par)
    idx = idx[order]
    g = g[:, order].astype(np.int64)
    ls = l[idx]
    u = (ls[:k] > 0).astype(np.int64)
    c = u @ g % 2

    def dist(cands):
        return np.mean(_softplus32(ls[None, :] * (1 - 2 * cands).astype(np.float32)), axis=1, dtype=np.float32)
    best_c, best_d = c, dist(c[None])[0]
    for ti in range(1, min(t, k) + 1):
        ep = np.array(list(itertools.combinations(range(k), ti)))
        cands = (c[None] + g[ep].sum(axis=1)) % 2
        d = dist(cands)
        i = int(np.argmin(d))
        if d[i] < best_d:
            best_d, best_c = d[i], cands[i]
    out = np.empty(n, np.int64)
    out[idx] = best_c
    return out


def _popw(words, weights):
    """sum of weights over the set bits of packed uint8 rows [..., nb]."""
    bits = np.unpackbits(words, axis=-1, bitorder="little")[..., :len(weights)]
    return bits @ weights


def osd_discrepancy(llr, gm, t, return_gap=False):
    """Float64 discrepancy form of the same decoder: greedy MRB in stable |llr| order, candidates in (order,
    itertools.combinations rank over the MRB positions in reliability order), D = sum of |llr| where the candidate
    differs from the hard decisions, first minimum kept. Returns the codeword (and the best D and the runner-up's)."""
    gm = np.asarray(gm, np.int64)
    k, n = gm.shape
    l = np.clip(np.asarray(llr, np.float32), -100, 100).astype(np.float64)
    a = np.abs(l)
    hd = (l > 0).astype(np.uint8)
    idx = np.argsort(-a, kind="stable")
    mrb = mrb_greedy(gm[:, idx])
    par = [j for j in range(n) if j not in set(mrb)]
    gs = gm[:, idx]
    sub = gs[:, mrb]
    # rows of the systematic generator on the MRB: inverse(sub) @ gs over GF(2)
    aug = np.concatenate([sub.T, np.eye(k, dtype=np.int64)], axis=1).astype(bool)   # solve sub^T x = e
    for c in range(k):
        p = c + int(np.flatnonzero(aug[c:, c])[0])
        aug[[c, p]] = aug[[p, c]]
        rows = np.flatnonzero(aug[:, c])
        rows = rows[rows != c]
        aug[rows] ^= aug[c]
    inv = aug[:, k:].astype(np.int64).T                    # inv @ sub = I
    sysm = inv @ gs % 2
    P = sysm[:, par].astype(np.uint8)                      # [k, n-k], row i = MRB position i (reliability order)
    a_m, a_p = a[idx][mrb], a[idx][par]
    hd_m, hd_p = hd[idx][mrb], hd[idx][par]
    r0 = (hd_m.astype(np.int64) @ P % 2).astype(np.uint8) ^ hd_p
    Pk = np.packbits(P, axis=1, bitorder="little")
    r0k = np.packbits(r0, bitorder="little")
    ds, pats = [np.array([_popw(r0k, a_p)])], [()]
    for ti in range(1, min(t, k) + 1):
        ep = np.array(list(itertools.combinations(range(k), ti)))
        res = np.bitwise_xor.reduce(Pk[ep], axis=1) ^ r0k[None]
        ds.append(a_m[ep].sum(axis=1) + _popw(res, a_p))
        pats += [tuple(e) for e in ep]
    d = np.concatenate(ds)
    i = int(np.argmin(d))
    flip = np.zeros(k, np.uint8)
    flip[list(pats[i])] = 1
    cm = hd_m ^ flip
    cp = (cm.astype(np.int64) @ P % 2).astype(np.uint8)
    cs = np.empty(n, np.int64)
    cs[mrb] = cm
    cs[par] = cp
    out = np.empty(n, np.int64)
    out[idx] = cs
    if not return_gap:
        return out
    d2 = np.partition(d, 1)[1] if d.size > 1 else np.inf
    return out, d[i], d2


def ml_bruteforce(llr, gm, return_gap=False):
    """Maximum-likelihood codeword over all 2^k codewords: the minimum float64 discrepancy."""
    gm = np.asarray(gm, np.int64)
    k, n = gm.shape
    l = np.clip(np.asarray(llr, np.float32), -100, 100).astype(np.float64)
    u = (np.arange(2 ** k)[:, None] >> np.arange(k)[None]) & 1
    cw = u @ gm % 2
    d = ((cw != (l > 0)[None]) * np.abs(l)[None]).sum(axis=1)
    i = int(np.argmin(d))
    if not return_gap:
        return cw[i]
    d2 = np.partition(d, 1)[1]
    return cw[i], d[i], d2
