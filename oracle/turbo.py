"""NumPy restatement of the turbo code (reference fec/turbo/{encoding,decoding,utils}.py, fec/interleaving.py), test
infrastructure.

`qpp_perm` is the 3GPP interleaver computed from the QPP table. `encode` runs two `conv.encode` RSC passes and
multiplexes (x1, z1, z2) symbols, the termination bits of encoder 1 then encoder 2 with zero padding, and the puncturing
pattern row by row. `depuncture` inverts the puncturing with zeros and splits the stream into the two component
codewords (decoding.py:254-312). `decode` is the reference's loop (decoding.py:357-435) over `conv.bcjr` in `dtype`: in
float64 the reference's formulation, in float32 the single-precision evaluation that `parity.envelope` measures the
kernel against."""
import math

import numpy as np

from . import conv

PATTERNS = {1 / 3: np.array([[1, 1, 1]], bool), 1 / 2: np.array([[1, 1, 0], [1, 0, 1]], bool)}


def qpp_perm(k, table):
    """pi [k] of the QPP interleaver with table {K: (f1, f2)}: the next K >= k, entries >= k dropped."""
    K = min(x for x in table if x >= k)
    f1, f2 = table[K]
    i = np.arange(K, dtype=np.int64)
    p = (f1 * i + f2 * i * i) % K
    return p[p < k]


def _keep(rows, rate):
    pat = PATTERNS[rate]
    return np.tile(pat, (math.ceil(rows / len(pat)), 1))[:rows].reshape(-1)


def encode(u, gen_poly, perm, rate=1 / 3, terminate=False):
    """Turbo codewords [B, n] (float64) of bits u [B, k] with interleaver perm (u2[i] = u[perm[i]])."""
    u = np.asarray(u).astype(np.int64)
    B, k = u.shape
    mu = len(gen_poly[0]) - 1
    c1 = conv.encode(u, gen_poly, True, terminate)
    c2 = conv.encode(u[:, perm], gen_poly, True, terminate)
    body = np.stack([c1[:, 0:2 * k:2], c1[:, 1:2 * k:2], c2[:, 1:2 * k:2]], -1).reshape(B, -1)
    if terminate:
        term = np.concatenate([c1[:, 2 * k:], c2[:, 2 * k:]], 1)
        pad = 3 * math.ceil(4 * mu / 3) - term.shape[1]
        body = np.concatenate([body, term, np.zeros((B, pad))], 1)
    return body[:, _keep(body.shape[1] // 3, rate)]


def depuncture(y, k, mu, perm, rate=1 / 3, terminate=False):
    """The two component codewords [B, 2 T] of turbo logits y [B, n] (punctured positions 0)."""
    y = np.asarray(y)
    B = y.shape[0]
    rows = k + (math.ceil(4 * mu / 3) if terminate else 0)
    full = np.zeros((B, 3 * rows), y.dtype)
    full[:, _keep(rows, rate)] = y
    body = full[:, :3 * k].reshape(B, k, 3)
    y1 = body[:, :, :2].reshape(B, -1)
    y2 = np.stack([body[:, perm, 0], body[:, :, 2]], -1).reshape(B, -1)
    if terminate:
        t = full[:, 3 * k:]
        y1 = np.concatenate([y1, t[:, :2 * mu]], 1)
        y2 = np.concatenate([y2, t[:, 2 * mu:4 * mu]], 1)
    return y1, y2


def decode(y, gen_poly, perm, rate=1 / 3, terminate=False, num_iter=6, algorithm="map", dtype=np.float64,
           return_llr=True, return_peak_ext=False):
    """APP logits [B, k] (or hard bits) of turbo logits y [B, n], the reference's iteration in `dtype`. With
    return_peak_ext also the largest |extrinsic LLR| [B] before the +-20 clip among those passed on to the other
    decoder (decoder 1's of every iteration, decoder 2's of all but the last), which shows whether the clip bound."""
    mu = len(gen_poly[0]) - 1
    k = len(perm)
    pinv = np.argsort(perm)
    y1, y2 = (a.astype(dtype) for a in depuncture(np.asarray(y, dtype), k, mu, perm, rate, terminate))
    B = y1.shape[0]
    tz = mu if terminate else 0
    lch, lch2 = y1[:, 0:2 * k:2], y2[:, 0:2 * k:2]
    l1e = np.zeros((B, k + tz), dtype)
    l2i = np.zeros((B, k), dtype)
    peak = np.zeros(B)
    for i in range(num_iter):
        l1i = conv.bcjr(y1, gen_poly, True, terminate, algorithm, l1e, dtype)[:, :k]
        ex = ((l1i - lch).astype(dtype) - l1e[:, :k]).astype(dtype)
        peak = np.maximum(peak, np.abs(ex).max(axis=1))
        l2e = np.concatenate([np.clip(ex[:, perm], -20, 20), np.zeros((B, tz), dtype)], 1).astype(dtype)
        l2i = conv.bcjr(y2, gen_poly, True, terminate, algorithm, l2e, dtype)[:, :k]
        ex = ((l2i - l2e[:, :k]).astype(dtype) - lch2).astype(dtype)
        if i + 1 < num_iter:
            peak = np.maximum(peak, np.abs(ex).max(axis=1))
        l1e = np.concatenate([np.clip(ex[:, pinv], -20, 20), np.zeros((B, tz), dtype)], 1).astype(dtype)
    out = l2i[:, pinv]
    out = out if return_llr else (out > 0).astype(np.float64)
    return (out, peak) if return_peak_ext else out
