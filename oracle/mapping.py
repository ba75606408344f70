"""Oracle: constellations, mapping, demapping, AWGN helpers (NumPy + oracle/mapping_ref.c). TEST INFRASTRUCTURE.

Follows /root/reference/src/sionna/phy/mapping.py: pam_gray :15-42, qam :44-118, pam :120-193 (38.211 5.1 closed
forms, checked against the formulas of /root/reference/test/unit/mapping/test_constellation.py:11-62),
Mapper.call :497-519, Demapper.call :664-691 + SymbolLogits2LLRs.call :927-967; utils/misc.py: ebnodb2no :171-251,
hard_decisions :254-271.
"""
import ctypes as C
import numpy as np

from . import ldpc as _l


def _lib():
    h = _l.lib()
    if not getattr(h, "_map_ready", False):
        h.sbo_demap.restype = None
        h.sbo_demap.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_int]
        h.sbo_demap_qam.restype = None
        h.sbo_demap_qam.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                    C.c_void_p, C.c_int64, C.c_int]
        h._map_ready = True
    return h


def pam_gray(b):                                                   # mapping.py:40-42
    if len(b) > 1:
        return (1 - 2 * b[0]) * (2 ** len(b[1:]) - pam_gray(b[1:]))
    return 1 - 2 * b[0]


def qam(m, normalize=True):                                        # mapping.py:104-117
    c = np.zeros(2 ** m, np.complex64)
    for i in range(2 ** m):
        b = np.array(list(np.binary_repr(i, m)), dtype=np.int32)
        c[i] = pam_gray(b[0::2]) + 1j * pam_gray(b[1::2])
    if normalize:
        n = m // 2
        qam_var = 1 / (2 ** (n - 2)) * np.sum(np.linspace(1, 2 ** n - 1, 2 ** (n - 1), dtype=np.float32) ** 2)
        c /= np.sqrt(qam_var)
    return c


def pam(m, normalize=True):                                        # mapping.py:180-192
    c = np.zeros(2 ** m, np.complex64)
    for i in range(2 ** m):
        c[i] = pam_gray(np.array(list(np.binary_repr(i, m)), dtype=np.int32))
    if normalize:
        pam_var = 1 / (2 ** (m - 1)) * np.sum(np.linspace(1, 2 ** m - 1, 2 ** (m - 1), dtype=np.float32) ** 2)
        c /= np.sqrt(pam_var)
    return c


def mapper(bits, points):                                          # mapping.py:497-514
    m = int(np.log2(len(points)))
    b = np.asarray(bits).astype(np.int32)
    b = b.reshape(b.shape[:-1] + (b.shape[-1] // m, m))
    idx = np.sum(b << np.arange(m - 1, -1, -1), axis=-1)
    return points[idx], idx


def separable_levels(points):
    """(levels_re, levels_im) if points[j] = levels_re[even label bits of j] + 1j * levels_im[odd label bits of j]
    exactly (every square QAM of mapping.py:104-117), else None. Bits are counted MSB first."""
    pts = np.asarray(points)
    m = int(np.log2(len(pts)))
    if m < 2 or m % 2 or m > 10:
        return None
    h = m // 2
    j = np.arange(len(pts))
    bits = (j[:, None] >> np.arange(m - 1, -1, -1)) & 1                # [2^m, m] MSB first
    w = 1 << np.arange(h - 1, -1, -1)
    jr, ji = bits[:, 0::2] @ w, bits[:, 1::2] @ w
    lev_re = np.zeros(1 << h, np.float32)
    lev_im = np.zeros(1 << h, np.float32)
    lev_re[jr[ji == 0]] = pts.real[ji == 0]
    lev_im[ji[jr == 0]] = pts.imag[jr == 0]
    if np.array_equal(lev_re[jr].astype(np.float32), pts.real.astype(np.float32)) and \
            np.array_equal(lev_im[ji].astype(np.float32), pts.imag.astype(np.float32)):
        return lev_re, lev_im
    return None


def demapper(y, no, points, method="app", prior=None, hard_out=False, math_mode=0):
    """y [..., S] complex64, no scalar or broadcastable to y, prior None | [m] | [..., S, m] -> llr [..., S*m].
    math_mode 0: the reference's 2-D formula with libm; math_mode 1: what the CUDA kernels evaluate (the separable form
    for square QAM without prior, the 2-D formula with sb_math.h otherwise)."""
    y = np.ascontiguousarray(y, np.complex64)
    m = int(np.log2(len(points)))
    pts = np.ascontiguousarray(points, np.complex64)
    n_sym = y.size
    no_b = np.ascontiguousarray(np.broadcast_to(np.asarray(no, np.float32).reshape(
        np.shape(no) + (1,) * (y.ndim - np.ndim(no))), y.shape), np.float32)
    sep = separable_levels(pts) if (math_mode == 1 and prior is None) else None
    if sep is not None:
        llr = np.empty(y.shape[:-1] + (y.shape[-1] * m,), np.float32)
        lr, li = np.ascontiguousarray(sep[0]), np.ascontiguousarray(sep[1])
        _lib().sbo_demap_qam(y.ctypes.data, no_b.ctypes.data, 1, lr.ctypes.data, li.ctypes.data, m,
                             0 if method == "app" else 1, llr.ctypes.data, n_sym, int(hard_out))
        return llr
    pr = None
    inner = 1
    if prior is not None:
        prior = np.asarray(prior, np.float32)
        if prior.ndim == 1:
            pr, inner = np.ascontiguousarray(prior), max(n_sym, 1)
        else:
            pr = np.ascontiguousarray(np.broadcast_to(prior, y.shape + (m,)), np.float32)
    llr = np.empty(y.shape[:-1] + (y.shape[-1] * m,), np.float32)
    _lib().sbo_demap(y.ctypes.data, no_b.ctypes.data, 1, pts.ctypes.data, m, 0 if method == "app" else 1,
                     None if pr is None else pr.ctypes.data, inner, llr.ctypes.data, n_sym, int(hard_out), math_mode)
    return llr


def demapper_f64(y, no, points, method="app", prior=None):
    """The reference's 2-D demapping formula in float64 (mapping.py:664-691, 915-967), plain NumPy / SciPy: exponents
    -|y - c|^2 / max(no, float32 tiny) (+ sum_k log_sigmoid(+-prior_k)), then logsumexp ("app") or max ("maxlog") over
    the points with label bit i = 1 minus the same over bit i = 0, each group relative to its own maximum. Inputs as
    `demapper`, evaluated at their float32 / complex64 values; -> llr [..., S*m] float64."""
    from scipy.special import logsumexp
    y = np.asarray(y, np.complex64).astype(np.complex128)
    pts = np.asarray(points, np.complex64).astype(np.complex128)
    m = int(np.log2(len(pts)))
    no = np.asarray(no, np.float32).astype(np.float64)
    no = np.broadcast_to(no.reshape(no.shape + (1,) * (y.ndim - no.ndim)), y.shape)
    tiny = float(np.finfo(np.float32).tiny)
    e = -np.abs(y[..., None] - pts) ** 2 / np.maximum(no, tiny)[..., None]          # [..., S, 2^m]
    lab = (np.arange(2 ** m)[:, None] >> np.arange(m - 1, -1, -1)) & 1               # [2^m, m] label bits, MSB first
    if prior is not None:
        p = np.broadcast_to(np.asarray(prior, np.float32).astype(np.float64), y.shape + (m,))
        s = 2.0 * lab - 1.0                                                          # bit 1 -> +prior, 0 -> -prior
        for k in range(m):
            e = e - np.logaddexp(0.0, -s[:, k] * p[..., k, None])                    # log_sigmoid(s * prior_k)
    e = e.reshape(-1, 2 ** m)
    out = np.empty((e.shape[0], m))
    for i in range(m):
        g = e.reshape(-1, 2 ** i, 2, 2 ** (m - 1 - i))                               # [.., higher bits, bit i, lower]
        red = (lambda a: logsumexp(a, axis=(1, 2))) if method == "app" else (lambda a: np.max(a, axis=(1, 2)))
        out[:, i] = red(g[:, :, 1, :]) - red(g[:, :, 0, :])
    return out.reshape(y.shape[:-1] + (y.shape[-1] * m,))


def ebnodb2no(ebno_db, num_bits_per_symbol, coderate):             # utils/misc.py:233-251 (no resource grid)
    ebno = np.power(np.float32(10), np.float32(ebno_db) / np.float32(10))
    return np.float32(1) / (ebno * np.float32(coderate) * np.float32(num_bits_per_symbol) / np.float32(1.0))


def hard_decisions(llr):                                           # utils/misc.py:270-271
    return (np.asarray(llr) > 0).astype(np.float32)
