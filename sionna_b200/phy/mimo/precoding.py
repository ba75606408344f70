"""MIMO transmit precoding (mirror of the reference's src/sionna/phy/mimo/precoding.py:12-245) on ``sb_mimo_precode``:
the precoding matrix ``G = V D`` of every problem is computed by one group of lanes in shared memory and never leaves
the chip unless it is asked for. Complex64 only; ``precision="double"`` falls back to the single-precision kernel
(``PrecisionWarning``) and returns complex128. The DFT grid-of-beams helpers (``grid_of_beams_dft(_ula)``,
``flatten_precoding_mat``, ``normalize_precoding_power``) are not provided."""
import torch

from ..config import config
from ..._lib import lib, check, ptr, current_stream

_RZF, _CBF = 0, 1


def _precode(kind, h, alpha, x, want_g):
    """(g [..., M, K] or None, G x [..., M] or None) from sb_mimo_precode; alpha (RZF) broadcasts like
    ``expand_to_rank(alpha, rank(g), axis=-1)``: its dimensions align with h's leading ones from the left."""
    dev = config.device
    h = torch.as_tensor(h).to(device=dev, dtype=torch.complex64)
    k, m = h.shape[-2], h.shape[-1]
    lead = tuple(h.shape[:-2])
    if x is not None:
        x = torch.as_tensor(x).to(device=dev, dtype=torch.complex64)
        lead = tuple(torch.broadcast_shapes(lead, tuple(x.shape[:-1])))
    al, al_stride = None, 0
    if kind == _RZF:
        al = torch.as_tensor(alpha).to(device=dev, dtype=torch.float32)
        if al.dim() > len(lead):
            raise ValueError("alpha has more dimensions than the batch dimensions of h")
        al = al.reshape(tuple(al.shape) + (1,) * (len(lead) - al.dim()))
        lead = tuple(torch.broadcast_shapes(lead, tuple(al.shape)))
        if al.numel() == 1:
            al = al.reshape(1).contiguous()
        else:
            al, al_stride = al.expand(lead).contiguous(), 1
    h = h.expand(*lead, k, m).contiguous()
    num = h.numel() // (k * m) if k * m else 0
    g = torch.empty(*lead, m, k, dtype=torch.complex64, device=dev) if want_g else None
    gx = None
    if x is not None:
        x = x.expand(*lead, k).contiguous()
        gx = torch.empty(*lead, m, dtype=torch.complex64, device=dev)
    check(lib().sb_mimo_precode(ptr(h), ptr(al), al_stride, ptr(x), ptr(g), ptr(gx), num, k, m, kind,
                                current_stream()), "sb_mimo_precode")
    return g, gx


def _double(name, precision):
    from ..block import fallback_to_single
    return fallback_to_single(name, precision)


def rzf_precoding_matrix(h, alpha=0., precision=None):
    r"""Regularized zero-forcing precoding matrix ``G = V D`` with ``V = H^H (H H^H + alpha I)^-1`` (Cholesky of
    ``H H^H + alpha I``, then ``cholesky_solve`` against H and the adjoint) and ``D`` scaling every column of V to unit
    norm; a zero column stays zero (precoding.py:12-89). h [..., K, M], alpha scalar or [...] -> g [..., M, K].
    alpha = 0 with K > M makes the Gram matrix singular; the result is then not finite."""
    if _double("rzf_precoding_matrix", precision):
        return rzf_precoding_matrix(h, alpha, "single").to(torch.complex128)
    return _precode(_RZF, h, alpha, None, True)[0]


def cbf_precoding_matrix(h, precision=None):
    r"""Conjugate beamforming precoding matrix: ``H^H`` with unit-norm columns (precoding.py:91-155).
    h [..., K, M] -> g [..., M, K]."""
    if _double("cbf_precoding_matrix", precision):
        return cbf_precoding_matrix(h, "single").to(torch.complex128)
    return _precode(_CBF, h, 0., None, True)[0]


def rzf_precoder(x, h, alpha=0., return_precoding_matrix=False, precision=None):
    r"""RZF precoding ``G x`` with ``G = rzf_precoding_matrix(h, alpha)`` (precoding.py:157-245), both from one
    launch. x [..., K], h [..., K, M] -> x_precoded [..., M] (and g [..., M, K] if ``return_precoding_matrix``)."""
    if _double("rzf_precoder", precision):
        out = rzf_precoder(x, h, alpha, return_precoding_matrix, "single")
        return tuple(t.to(torch.complex128) for t in out) if return_precoding_matrix else out.to(torch.complex128)
    g, gx = _precode(_RZF, h, alpha, x, return_precoding_matrix)
    return (gx, g) if return_precoding_matrix else gx
