"""Linear-algebra helpers (mirror of /root/reference/src/sionna/phy/utils/linalg.py): inv_cholesky, matrix_pinv."""
import torch

from ..config import config
from ..._lib import lib, check, ptr, current_stream


def inv_cholesky(tensor):
    r"""Inverse ``L^-1`` of the Cholesky factor ``L`` of Hermitian positive-definite matrices ``[..., M, M]``
    (linalg.py:8-32); one kernel, ``sb_mimo_linalg`` mode 0."""
    from ..block import fallback_to_single
    wide = fallback_to_single("inv_cholesky", None)
    dev = config.device
    t = torch.as_tensor(tensor)
    real = not t.is_complex()
    s = t.to(device=dev, dtype=torch.complex64).contiguous()
    m = s.shape[-1]
    out = torch.empty_like(s)
    check(lib().sb_mimo_linalg(0, None, None, ptr(s), ptr(out), None, s.numel() // (m * m), m, m, current_stream()),
          "sb_mimo_linalg")
    if wide:
        out = out.to(torch.complex128)
    return out.real.contiguous() if real else out


def matrix_pinv(tensor):
    r"""Pseudo-inverse ``A^+ = (A^H A)^-1 A^H`` of matrices ``[..., M, K]`` with linearly independent columns
    (linalg.py, ``matrix_pinv``: Cholesky factor of ``A^H A``, then cholesky_solve) -> ``[..., K, M]``; one kernel,
    ``sb_mimo_linalg`` mode 6."""
    from ..block import fallback_to_single
    wide = fallback_to_single("matrix_pinv", None)
    dev = config.device
    t = torch.as_tensor(tensor)
    real = not t.is_complex()
    h = t.to(device=dev, dtype=torch.complex64).contiguous()
    m, k = h.shape[-2], h.shape[-1]
    out = torch.empty(*h.shape[:-2], k, m, dtype=torch.complex64, device=dev)
    check(lib().sb_mimo_linalg(6, None, ptr(h), None, ptr(out), None, h.numel() // (m * k), m, k, current_stream()),
          "sb_mimo_linalg")
    if wide:
        out = out.to(torch.complex128)
    return out.real.contiguous() if real else out
