"""GPU parity of the voting (union-mask) variant of the boxplus-phi QC check-node update against the CPU oracle.

In the voting iterations a row slice evaluates phi only at the positions where some lane of the warp is unsaturated
(the union mask U). The batch below mixes Eb/N0 from 0.5 to 5 dB on the benchmark's code (k = 4224, n = 8448), so
within 20 iterations the codewords switch to the voting variant early, late or not at all, and its row slices meet
every case of the code: |U| = 0 and U = {last edge} (the two-phi rows), other small |U| with both pair and scalar
tails, and |U| = deg (tools/phi_work_model.py counts them). Soft outputs and the final v2c state must equal the
oracle in kernel math and kernel order bit for bit; a kernel that sums P in another order than ascending VN fails.
The mask treats |x| >= 14.7117348 as saturated (SB_PHI_ZERO in ldpc_bp_qc.cu): phi must be +0 for every fp32 value
from there up to the clipping bound 16.635532, in the oracle and on the device.
"""
import numpy as np
import pytest
import torch

from oracle import ldpc as O

PHI_ZERO = np.float32(14.7117348)
PHI_HI = np.float32(16.635532)


def _sweep():
    """Every fp32 value in [PHI_ZERO, PHI_HI], and the one just below PHI_ZERO."""
    lo, hi = int(PHI_ZERO.view(np.uint32)), int(PHI_HI.view(np.uint32))
    return np.arange(lo - 1, hi + 1, dtype=np.uint32).view(np.float32)


def test_phi_zero_bound_oracle():
    x = _sweep()
    phi = np.array([O.phi(v, 1) for v in x])
    assert phi[0] > 0 and np.all(phi[1:] == 0)


@pytest.mark.gpu
def test_phi_zero_bound_device(cuda_device):
    from sionna_b200 import _lib
    x = _sweep()
    x = x[: len(x) // 2 * 2]
    xd = torch.from_numpy(x).to(cuda_device)
    o1, o2 = torch.empty_like(xd), torch.empty_like(xd)
    _lib.check(_lib.lib().sb_debug_phi(_lib.ptr(xd), _lib.ptr(o1), _lib.ptr(o2), len(x), _lib.current_stream()), "sb_debug_phi")
    for o in (o1.cpu().numpy(), o2.cpu().numpy()):
        assert o[0] > 0 and np.all(o[1:].view(np.uint32) == 0)


@pytest.mark.gpu
def test_union_mask_rows_bit_exact_over_snr_mix(cuda_device):
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    from bench import host_cores
    k, n, bs, it = 4224, 8448, 640, 20
    rng = np.random.default_rng(2024)
    enc_r = O.LDPC5GEncoderRef(k, n)
    c = enc_r(rng.integers(0, 2, (bs, k)))
    ebno = np.repeat(np.linspace(0.5, 5.0, 10), bs // 10)
    no = 1.0 / (10 ** (ebno[:, None] / 10) * (k / n))
    y = (2.0 * c - 1.0) + rng.normal(size=c.shape) * np.sqrt(no / 2)
    llr = (4 * y / no).astype(np.float32)
    dec = LDPC5GDecoder(LDPC5GEncoder(k, n), hard_out=False, return_infobits=False, num_iter=it, return_state=True)
    assert dec._graph.is_qc()
    x, st = dec(torch.from_numpy(llr).to(cuda_device))
    ref = O.LDPC5GDecoderRef(enc_r, hard_out=False, return_infobits=False, num_iter=it, return_state=True)
    xr, sr = ref(llr, math_mode=1, order="kernel", num_threads=host_cores()[0])
    assert np.array_equal(x.cpu().numpy(), xr)
    assert np.array_equal(st.cpu().numpy(), sr)
    err = ((xr > 0) != (c > 0)).any(axis=1)
    assert err[: bs // 10].any() and not err[-bs // 10:].any()   # failing and converged codewords in the same launch
