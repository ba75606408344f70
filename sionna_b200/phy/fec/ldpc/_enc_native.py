"""Owns one ``sb_ldpc5g_encoder`` handle (CSR tables of the RU sub-matrices + transmit gather)."""
import numpy as np
import torch

from ...._lib import Handle, lib, check, ptr, current_stream
from .encoding import _csr_lists


class EncoderHandle(Handle):
    def __init__(self, enc):
        a, b_inv, c1, c2 = enc._ru_submatrices()
        tabs = [np.ascontiguousarray(t, np.int32) for m in (a, b_inv, c1, c2) for t in _csr_lists(m)]
        tabs.append(np.ascontiguousarray(enc._tx_vn(), np.int32))
        super().__init__("ldpc5g_encoder", enc.k, enc.n, enc.k_ldpc, enc.n_ldpc, 4 * enc.z, *(ptr(t) for t in tabs))
        self.k, self.n = enc.k, enc.n

    def encode(self, u):
        if u.dtype != torch.float32:
            raise NotImplementedError("sb_ldpc5g_encode is an fp32 kernel; precision='double' is not available.")
        c = torch.empty((u.shape[0], self.n), dtype=torch.float32, device=u.device)
        check(lib().sb_ldpc5g_encode(self.handle, ptr(u), u.shape[0], ptr(c), current_stream()), "sb_ldpc5g_encode")
        return c
