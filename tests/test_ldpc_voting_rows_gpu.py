"""GPU parity of the voting pass of the boxplus-phi QC decoder on graph shapes the benchmark code does not have.

In the voting iterations a warp walks its block rows class-agnostically: a row whose union mask holds no edge but the
last takes two phi, every other row the general 2k + 1 walk, output signs come from a per-lane sign mask, and a lane
outside a row (lane_i >= zrow) must neither read, vote nor store in it. The codes below each bring one shape the
benchmark code (Z = 192, four warp groups of six full block rows) lacks:
  * k = 1000, n = 2000: Z = 104, not a multiple of 32, so the last 32-lane slice of every row is partly empty; the
    pruned graph ends in a partial block row (64 of 104 checks);
  * k = 2000, n = 5000: Z = 208 and a partial last block row (88 checks); warp groups get unequal row counts (6, 6, 5);
  * k = 700, n = 1600: Z = 72, a partial last block row, eight warp groups of which one gets a single row.
Each batch spreads Eb/N0 over -1 ... 5 dB, so within 20 iterations some codewords converge early, some late and some
not at all (the last assertion checks both ends), so the voting rows of a launch meet both paths.
Soft outputs and the final v2c state must equal the oracle in kernel math and kernel order bit for bit.
"""
import numpy as np
import pytest
import torch

from oracle import ldpc as O

# (k, n, Z, checks in the last block row, block rows per warp group)
CODES = [(1000, 2000, 104, 64, [2, 2, 2, 2, 2, 2]),
         (2000, 5000, 208, 88, [6, 6, 5]),
         (700, 1600, 72, 36, [2, 2, 2, 2, 2, 2, 2, 1])]


def _rows_per_group(z, c, n):
    """Block rows dealt to each warp group of the QC kernel (768 threads, one 32-lane slice of a row per warp)."""
    rows, cols = -(-c // z), -(-n // z)
    g = max(1, min(24 // -(-z // 32), max(rows, cols)))
    return [len(range(i, rows, g)) for i in range(g)]


@pytest.mark.parametrize("k, n, z, last, groups", CODES)
def test_codes_have_the_shapes(k, n, z, last, groups):
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    enc = LDPC5GEncoder(k, n)
    dec = LDPC5GDecoder(enc, num_iter=1)
    c = dec._num_cns
    assert enc.z == z and c % z == last
    assert _rows_per_group(z, c, dec._num_vns) == groups


@pytest.mark.gpu
@pytest.mark.parametrize("k, n, z, last, groups", CODES)
def test_voting_rows_bit_exact(cuda_device, k, n, z, last, groups):
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
    from bench import host_cores
    bs, it = 400, 20
    rng = np.random.default_rng(k + n)
    enc_r = O.LDPC5GEncoderRef(k, n)
    c = enc_r(rng.integers(0, 2, (bs, k)))
    ebno = np.repeat(np.linspace(-1.0, 5.0, 10), bs // 10)
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
