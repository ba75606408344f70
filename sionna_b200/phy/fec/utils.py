"""FEC utilities (mirror of parts of sionna/phy/fec/utils.py): LLR sources and information measures for the tests,
the example codes, and the generator / parity-check matrix conversions that linear block codes need (NumPy, one-time
set-up, not on the hot path)."""
import os
import warnings

import numpy as np
import torch

from ..block import Block
from ..config import config
from .._lib_helpers import philox_fill


class GaussianPriorSource(Block):
    """Fake LLRs of an all-zero codeword sent with BPSK over AWGN (fec/utils.py:16-114): logits ~ N(-mu, sigma^2),
    sigma^2 = 4/no, mu = sigma^2/2. ``call(output_shape, no)``."""

    def __init__(self, *, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)

    def __call__(self, output_shape, no=None, mi=None):
        return self._invoke(output_shape, no, mi)

    def call(self, output_shape, no=None, mi=None):
        if no is None:
            if mi is None:
                raise ValueError("Either no or mi must be provided.")
            # mutual-information parametrisation (fec/utils.py:88-96): mu = J^-1(mi), sigma^2 = 2 mu
            mi = float(torch.as_tensor(mi).reshape(-1)[0]) if not isinstance(mi, (int, float)) else float(mi)
            mi = min(max(mi, 1e-7), 1.0)
            mu_llr = float(j_fun_inv(mi))
            sigma_llr = np.sqrt(2 * mu_llr)
        else:
            no = float(torch.as_tensor(no).reshape(-1)[0]) if not isinstance(no, (int, float)) else float(no)
            no = max(no, 1e-7)
            sigma_llr = np.sqrt(4.0 / no)
            mu_llr = sigma_llr ** 2 / 2
        shape = [int(s) for s in output_shape]
        return philox_fill("sb_normal", shape, -mu_llr, sigma_llr, self.device).to(self.rdtype)


def llr2mi(llr, s=None, reduce_dims=True):
    r"""Mutual information estimate :math:`1 - E[\log_2(1 + e^{llr})]` for logits of an all-zero codeword (or of the
    codeword with BPSK signs ``s``), fec/utils.py:116-182. An analysis helper (EXIT charts), not on the hot path."""
    llr = torch.as_tensor(llr)
    if not llr.dtype.is_floating_point:
        raise TypeError("Dtype of llr must be a real-valued float.")
    z = llr if s is None else torch.as_tensor(s).to(llr.dtype) * llr
    z = torch.clamp(z, -100.0, 100.0)
    x = torch.log2(1.0 + torch.exp(z))
    return 1.0 - (x.mean() if reduce_dims else x.mean(dim=-1))


_H1, _H2, _H3 = 0.3073, 0.8935, 1.1064


def j_fun(mu):
    r"""J-function (Brannstrom approximation), fec/utils.py:184-225: mutual information of Gaussian LLRs with mean mu."""
    mu = np.minimum(np.maximum(np.asarray(mu, dtype=np.float64), 1e-10), 1000.0)
    return (1 - 2 ** (-_H1 * (2 * mu) ** _H2)) ** _H3


def j_fun_inv(mi):
    r"""Inverse J-function, fec/utils.py:227-267 (output clipped to 20)."""
    mi = np.minimum(np.maximum(np.asarray(mi, dtype=np.float64), 1e-10), 1.0)
    with np.errstate(divide="ignore"):
        mu = 0.5 * ((-1 / _H1) * np.log2(1 - mi ** (1 / _H3))) ** (1 / _H2)
    return np.minimum(mu, 20.0)


def load_parity_check_examples(pcm_id, verbose=False):
    """Built-in example parity-check matrices (fec/utils.py:478-531): 0 = (7,4) Hamming, 1 = BCH(63,45),
    2 = BCH(127,106), 3 = (3,6)-regular LDPC n=100, 4 = 802.11n LDPC n=648. Returns ``pcm, k, n, coderate``."""
    p = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ldpc", "codes", "example_pcms.npz")
    with np.load(p) as d:
        pcm = np.array(d[f"pcm{int(pcm_id)}"], dtype=np.int64)
    n = int(pcm.shape[1])
    k = int(n - pcm.shape[0])
    coderate = k / n
    if verbose:
        print(f"\nn: {n}, k: {k}, coderate: {coderate:.3f}")
    return pcm, k, n, coderate


def bin2int(arr):
    """Integer of a binary sequence, most significant bit first (fec/utils.py:532-549): ``[1, 0, 1]`` -> 5; None for
    an empty sequence."""
    if len(arr) == 0:
        return None
    return int("".join(str(int(x)) for x in arr), 2)


def int2bin(num, length):
    """The ``length`` least significant bits of ``num``, most significant first (fec/utils.py:576-611):
    ``int2bin(5, 4)`` -> ``[0, 1, 0, 1]``, ``int2bin(12, 3)`` -> ``[1, 0, 0]``."""
    assert num >= 0, "Input integer should be non-negative"
    assert length >= 0, "length should be non-negative"
    bits = format(num, f"0{length}b")
    return [int(x) for x in bits[-length:]] if length else []


def alist2mat(alist, verbose=True):
    """Parity-check matrix of an ``alist`` code description (fec/utils.py:650-762): row 1 ``n m``, row 2 the maximum
    VN and CN degrees, rows 3 and 4 the VN and CN degree profiles, then n rows of each column's 1-based check indices
    and (optionally) m rows of each check's variable indices. Returns ``pcm [m, n], k, n, coderate``."""
    assert len(alist) > 4, "Invalid alist format."
    n, m = alist[0][0], alist[0][1]
    v_max, c_max = alist[1][0], alist[1][1]
    k = n - m
    coderate = k / n
    vn_profile, cn_profile = alist[2], alist[3]
    assert np.sum(vn_profile) == np.sum(cn_profile), "Invalid alist format."
    assert np.max(vn_profile) == v_max, "Invalid alist format."
    assert np.max(cn_profile) == c_max, "Invalid alist format."
    if len(alist) == len(vn_profile) + 4:
        print("Note: .alist does not contain (redundant) CN perspective.")
        print("Recovering parity-check matrix from VN only.")
        print("Please verify the correctness of the results manually.")
        vn_only = True
    else:
        assert len(alist) == len(vn_profile) + len(cn_profile) + 4, "Invalid alist format."
        vn_only = False
    pcm = np.zeros((m, n))
    num_edges = 0
    for idx_v in range(n):
        for idx_i in range(vn_profile[idx_v]):
            pcm[alist[4 + idx_v][idx_i] - 1, idx_v] = 1
            num_edges += 1
    if not vn_only:
        for idx_c in range(m):
            for idx_i in range(cn_profile[idx_c]):
                assert pcm[idx_c, alist[4 + n + idx_c][idx_i] - 1] == 1
    if verbose:
        print("Number of variable nodes (columns): ", n)
        print("Number of check nodes (rows): ", m)
        print("Number of information bits per cw: ", k)
        print("Number edges: ", num_edges)
        print("Max. VN degree: ", v_max)
        print("Max. CN degree: ", c_max)
        print("VN degree: ", vn_profile)
        print("CN degree: ", cn_profile)
    return pcm, k, n, coderate


def load_alist(path):
    """Nested list of the integers of an ``alist`` file, one list per non-empty line (fec/utils.py:764-795)."""
    alist = []
    with open(path, "r") as reader:
        for line in reader:
            row = [int(w) for w in line.split()]
            if row:
                alist.append(row)
    return alist


def make_systematic(mat, is_pcm=False):
    """Systematic form of a binary ``[m, n]`` matrix by GF(2) row operations and column swaps
    (fec/utils.py:797-906): identity in the first m columns, or the last m with ``is_pcm``. Returns ``(mat_sys,
    column_swaps)``, the swaps as ``[i, j]`` pairs in the order they were applied (the same swaps as the reference, so
    ``pcm2gm`` returns the reference's generator). Raises ``ValueError`` if ``mat`` is not of full rank."""
    m, n = mat.shape[0], mat.shape[1]
    assert m <= n, "Invalid matrix dimensions."
    if is_pcm and np.any(np.sum(mat, axis=0) == 0):
        warnings.warn("All-zero column in parity-check matrix detected. "
                      "It seems as if the code contains unprotected nodes.")
    mat = np.array(mat, copy=True).astype(bool)
    column_swaps = []
    for idx_c in range(m):
        success = bool(mat[idx_c, idx_c])
        if not success:
            rows = np.flatnonzero(mat[idx_c + 1:, idx_c])
            if rows.size:
                idx_r = idx_c + 1 + int(rows[0])
                mat[[idx_c, idx_r]] = mat[[idx_r, idx_c]]
                success = True
        if not success:
            cols = np.flatnonzero(mat[idx_c, idx_c + 1:])
            if cols.size:
                idx_cc = idx_c + 1 + int(cols[0])
                mat[:, [idx_c, idx_cc]] = mat[:, [idx_cc, idx_c]]
                column_swaps.append([idx_c, idx_cc])
                success = True
        if not success:
            raise ValueError("Could not succeed; mat is not full rank?")
        below = idx_c + 1 + np.flatnonzero(mat[idx_c + 1:, idx_c])
        mat[below] ^= mat[idx_c]
    for idx_c in range(m - 1, -1, -1):
        above = np.flatnonzero(mat[:idx_c, idx_c])
        mat[above] ^= mat[idx_c]
    assert np.array_equal(mat[:, :m], np.eye(m)), "Internal error, could not find systematic matrix."
    if is_pcm:
        for i in range(n - 1, (n - 1) - m, -1):
            j = i - (n - m)
            mat[:, [i, j]] = mat[:, [j, i]]
            column_swaps.append([i, j])
    return mat.astype(int), column_swaps


def gm2pcm(gm, verify_results=True):
    """Parity-check matrix ``[M^T | I]`` of the generator ``gm = [I | M]`` in systematic form, with
    ``make_systematic``'s column swaps undone (fec/utils.py:908-984). ``gm`` must be of full rank."""
    k, n = gm.shape[0], gm.shape[1]
    assert k < n, "Invalid matrix dimensions."
    gm_sys, c_swaps = make_systematic(gm, is_pcm=False)
    pcm = np.concatenate((np.transpose(gm_sys[:, -(n - k):]), np.eye(n - k)), axis=1)
    for a, b in c_swaps[::-1]:
        pcm[:, [a, b]] = pcm[:, [b, a]]
    if verify_results:
        assert verify_gm_pcm(gm=gm, pcm=pcm), "Resulting parity-check matrix does not match to generator matrix."
    return pcm


def pcm2gm(pcm, verify_results=True):
    """Generator matrix ``[I | M^T]`` of the parity-check matrix ``pcm = [M | I]`` in systematic form, with
    ``make_systematic``'s column swaps undone (fec/utils.py:986-1060). ``pcm`` must be of full rank."""
    n = pcm.shape[1]
    k = n - pcm.shape[0]
    assert k < n, "Invalid matrix dimensions."
    pcm_sys, c_swaps = make_systematic(pcm, is_pcm=True)
    gm = np.concatenate((np.eye(k), np.transpose(pcm_sys[:, :k])), axis=1)
    for a, b in c_swaps[::-1]:
        gm[:, [a, b]] = gm[:, [b, a]]
    if verify_results:
        assert verify_gm_pcm(gm=gm, pcm=pcm), "Resulting parity-check matrix does not match to generator matrix."
    return gm


def verify_gm_pcm(gm, pcm):
    """True iff ``gm [k, n]`` and ``pcm [n - k, n]`` are binary and ``pcm gm^T = 0`` over GF(2)
    (fec/utils.py:1062-1113)."""
    k, n = gm.shape[0], gm.shape[1]
    n_pcm = pcm.shape[1]
    k_pcm = n_pcm - pcm.shape[0]
    assert k == k_pcm, "Inconsistent shape of gm and pcm."
    assert n == n_pcm, "Inconsistent shape of gm and pcm."
    assert ((gm == 0) | (gm == 1)).all(), "gm is not binary."
    assert ((pcm == 0) | (pcm == 1)).all(), "pcm is not binary."
    s = np.mod(np.matmul(np.asarray(pcm, np.int64), np.transpose(np.asarray(gm, np.int64))), 2)
    return bool(np.sum(s) == 0)


def int_mod_2(x):
    """x mod 2 (fec/utils.py:1236-1262): bitwise for integer tensors, ``|round(x)| mod 2`` for floating ones. Takes a
    torch tensor or a NumPy array and returns the same kind."""
    if isinstance(x, np.ndarray):
        if np.issubdtype(x.dtype, np.integer):
            return np.bitwise_and(x, 1)
        return np.mod(np.abs(np.round(x)), 2)
    x = torch.as_tensor(x)
    if not x.dtype.is_floating_point:
        return torch.bitwise_and(x, 1)
    return torch.remainder(torch.abs(torch.round(x)), 2)
