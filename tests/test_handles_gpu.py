"""Lifetime and device placement of the library's handles (sb_ldpc_graph, sb_ldpc5g_encoder, sb_turbo_perm,
sb_osd_code): their tables are copied to a device by the first call there and freed by *_destroy, one copy per device.

Lifecycle: repeated create -> one call -> destroy leaves free device memory where it was. Two devices: the same block
gives bit-identical outputs on cuda:0, cuda:1 and cuda:0 again, so every call reads the current device's tables."""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CYCLES = 200
MAX_DRIFT = 32 << 20   # bytes; one leaked table set of the BG1, Z = 384 graph per cycle is about ten times this


def _ldpc_case():
    """5G BG1 at Z = 384 (k = 8448): the largest graph and encoder tables; the decoder takes the QC path."""
    from sionna_b200.phy.fec.ldpc import LDPC5GEncoder
    return LDPC5GEncoder(8448, 16896)


def _turbo_decoder():
    from sionna_b200.phy.fec.turbo import TurboDecoder
    return TurboDecoder(constraint_length=4, rate=1 / 3, terminate=True, num_iter=2)


def _osd_generator(k=64, n=128, seed=3):
    rng = np.random.default_rng(seed)
    return np.concatenate([np.eye(k, dtype=np.int64), rng.integers(0, 2, (k, n - k))], axis=1)


def _cases():
    """name -> (block factory, seeded host input)."""
    from sionna_b200.phy.fec.ldpc import LDPC5GDecoder
    from sionna_b200.phy.fec.linear import OSDecoder
    rng = np.random.default_rng(11)
    enc = _ldpc_case()
    k_turbo = 6144
    n_turbo = 3 * k_turbo + _turbo_decoder()._num_term_bits
    gm = _osd_generator()

    def llr(n):
        return torch.from_numpy(rng.normal(0.0, 3.0, (4, n)).astype(np.float32))

    return {
        "ldpc_graph": (lambda: LDPC5GDecoder(enc, hard_out=False, num_iter=5), llr(enc.n)),
        "ldpc5g_encoder": (_ldpc_case, torch.from_numpy(rng.integers(0, 2, (4, enc.k)).astype(np.float32))),
        "turbo_perm": (_turbo_decoder, llr(n_turbo)),
        "osd_code": (lambda: OSDecoder(gm, t=2), llr(gm.shape[1])),
    }


def _free_bytes():
    torch.cuda.synchronize()
    gc.collect()
    return torch.cuda.mem_get_info()[0]


@pytest.mark.parametrize("kind", ["ldpc_graph", "ldpc5g_encoder", "turbo_perm", "osd_code"])
def test_create_call_destroy_cycles_do_not_leak(kind, cuda_device):
    make, x = _cases()[kind]
    x = x.to(cuda_device)

    def cycle():
        block = make()
        block(x)

    cycle()                                   # module loading, workspaces and the caching allocator settle here
    free = _free_bytes()
    for _ in range(CYCLES):
        cycle()
    drift = free - _free_bytes()
    assert drift <= MAX_DRIFT, f"{kind}: free device memory fell by {drift / 2**20:.1f} MiB over {CYCLES} cycles"


def test_handles_follow_the_current_device(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    from sionna_b200.phy import config
    cases = _cases()
    blocks = {kind: (make(), x) for kind, (make, x) in cases.items() if kind != "ldpc5g_encoder"}
    assert blocks["ldpc_graph"][0]._graph.is_qc()
    saved = config.device
    runs = []
    try:
        for d in (0, 1, 0):
            dev = torch.device("cuda", d)
            config.device = dev
            with torch.cuda.device(dev):
                runs.append({kind: block(x.to(dev)).cpu() for kind, (block, x) in blocks.items()})
    finally:
        config.device = saved
    for kind in blocks:
        for i in (1, 2):
            assert torch.equal(runs[0][kind], runs[i][kind]), f"{kind}: run {i} differs from the first cuda:0 run"
