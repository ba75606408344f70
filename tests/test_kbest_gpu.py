"""K-Best MIMO detection (sb_mimo_kbest / sb_ofdm_kbest) against the NumPy oracle (oracle/kbest.py).

The oracle also returns, per problem, the smallest relative gap that decided anything (column order, every pruning
step, the best path). Problems whose gap is below 1e-4 are excluded; fewer than 1 % may be (EXCLUDED lists the cases
with more pruning layers, which need more). On the rest, hard indices
and bits equal the complex128 oracle exactly, and LLRs are held to the reference's own single-precision envelope: the
kernel's rms and max error against the complex128 oracle stay within 2x (rms) and 4x (max) of the complex64
evaluation's error on the same inputs, errors taken relative to the rms of each stream's reference LLRs."""
import zlib

import numpy as np
import pytest
import torch

from oracle import mapping as MAP
from oracle.kbest import kbest_detect, ofdm_kbest_detect
from oracle.mimo import ml_detect
from oracle.parity import cnormal, constellation, envelope, mimo_problem, ofdm_detection_case

BAR = (2.0, 4.0)
GAP = 1e-4
EXCLUDED = {                                    # cases allowed to exclude more than 1 %, with the oracle's measured share
    "16qam 4x8 k64": 0.05,                      # 4.30 %: 1024 children per layer and 3 pruning layers, dense metrics
    "16qam 4x8 real k64": 0.08,                 # 7.23 %: 8 PAM layers, 5 of them pruned
    "64qam 2x4 real k32": 0.02,                 # 1.37 %
    "256qam 2x4 k64": 0.03,                     # 2.73 %: 16 384 children in the second layer
    "S=16 qpsk 16x16 k32": 0.09,                # 7.81 %: 13 pruning layers
    "S=16 16qam 8x8 real k16": 0.03,            # 2.73 %
    "4x8 mu-mimo": 0.03,                        # 2.08 % of 192 elements
}                                               # (the share depends on the inputs and the oracle only, not the kernel)


def _keep(what, gap):
    keep = gap > GAP
    print(f"{what}: {1 - keep.mean():.3%} of the problems excluded (decision gap <= {GAP})")
    assert 1 - keep.mean() < EXCLUDED.get(what, 0.01), what
    return keep


# (name, streams, constellation type, bits per symbol, antennas, real representation, k, problems, no, LLR clip)
DENSE = [("qpsk 4x4 k16", 4, "qam", 2, 4, False, 16, 2048, 0.1, 20.0),
         ("qpsk 4x4 real k16", 4, "qam", 2, 4, True, 16, 2048, 0.1, np.inf),
         ("16qam 4x8 k64", 4, "qam", 4, 8, False, 64, 1024, 0.05, np.inf),
         ("16qam 4x8 real k64", 4, "qam", 4, 8, True, 64, 1024, 0.05, 20.0),
         ("64qam 2x4 k32", 2, "qam", 6, 4, False, 32, 1024, 0.01, 20.0),
         ("64qam 2x4 real k32", 2, "qam", 6, 4, True, 32, 1024, 0.01, np.inf),
         ("256qam 2x4 k64", 2, "qam", 8, 4, False, 64, 512, 0.002, np.inf),
         ("256qam 2x4 real k8", 2, "qam", 8, 4, True, 8, 512, 0.002, 20.0),
         ("pam8 3x4 k16", 3, "pam", 3, 4, False, 16, 1024, 0.05, np.inf),
         ("custom 8-point 2x3 k8", 2, "custom", 3, 3, False, 8, 1024, 0.05, 20.0),
         ("S=1 16qam k4", 1, "qam", 4, 2, False, 4, 4096, 0.05, np.inf),
         ("S=16 qpsk 16x16 k32", 16, "qam", 2, 16, False, 32, 256, 0.05, np.inf),
         ("S=16 16qam 8x8 real k16", 8, "qam", 4, 8, True, 16, 256, 0.02, np.inf)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", DENSE, ids=[c[0] for c in DENSE])
def test_dense_kbest_against_oracle(cuda_device, case):
    from sionna_b200.phy.mimo import KBestDetector
    name, ns, kind, m, mm, real_rep, k, num, no, clip = case
    const = constellation(kind, m)
    pts = const().cpu().numpy().astype(np.complex64)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    y, h, s = mimo_problem(rng, num, mm, ns, pts, no)
    dev = [torch.from_numpy(v).to(cuda_device) for v in (y, h, s)]
    kw = dict(real_rep=real_rep)
    ref, gap = kbest_detect(y, h, s, pts, k, "bit", llr_clip=clip, **kw)
    f32, _ = kbest_detect(y, h, s, pts, k, "bit", llr_clip=clip, dtype=np.complex64, **kw)
    keep = _keep(name, gap)
    det = KBestDetector("bit", ns, k, constellation=const, use_real_rep=real_rep)
    det.list2llr.llr_clip_val = clip
    got = det(*dev).cpu().numpy()
    assert got.shape == ref.shape == (num, ns, m)
    bad = envelope(f"{name} LLRs", got[keep], f32[keep], ref[keep], BAR)
    for output in ("bit", "symbol"):
        want, _ = kbest_detect(y, h, s, pts, k, output, hard_out=True, **kw)
        hard = KBestDetector(output, ns, k, constellation=const, hard_out=True, use_real_rep=real_rep)(*dev)
        assert hard.dtype == (torch.float32 if output == "bit" else torch.int32)
        hard = hard.cpu().numpy()
        assert hard.shape == want.shape
        assert np.array_equal(hard[keep], want[keep]), f"{name} hard {output}"
    assert not bad, bad


@pytest.mark.gpu
def test_list2llr_clip_is_read_at_every_call(cuda_device):
    from sionna_b200.phy.mimo import KBestDetector
    rng = np.random.default_rng(8)
    pts = MAP.qam(4).astype(np.complex64)
    y, h, s = mimo_problem(rng, 256, 4, 2, pts, 0.01)
    det = KBestDetector("bit", 2, 4, "qam", 4)
    dev = [torch.from_numpy(v).to(cuda_device) for v in (y, h, s)]
    a = det(*dev)
    assert float(a.abs().max()) == 20.0
    det.list2llr.llr_clip_val = 5.0
    assert float(det(*dev).abs().max()) == 5.0
    det.list2llr.llr_clip_val = np.inf
    assert bool(torch.isinf(det(*dev)).any())


# (streams, bits, real representation)
FULL_K = [(2, 4, False), (4, 2, False), (2, 4, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("ns,m,real_rep", FULL_K)
def test_full_k_matches_ml_maxlog(cuda_device, ns, m, real_rep):
    """k = |C|^S and no clipping: K-Best LLRs are the maxlog ML LLRs (the GPU MaximumLikelihoodDetector's and the
    oracle's), within the single-precision envelope."""
    from sionna_b200.phy.mimo import KBestDetector, MaximumLikelihoodDetector
    rng = np.random.default_rng(31 + ns + m + real_rep)
    pts = MAP.qam(m).astype(np.complex64)
    y, h, s = mimo_problem(rng, 1024, 4, ns, pts, 0.1)
    dev = [torch.from_numpy(v).to(cuda_device) for v in (y, h, s)]
    kb = KBestDetector("bit", ns, len(pts) ** ns, "qam", m, use_real_rep=real_rep)
    kb.list2llr.llr_clip_val = np.inf
    got = kb(*dev).cpu().numpy()
    ml = MaximumLikelihoodDetector("bit", "maxlog", ns, "qam", m)(*dev).cpu().numpy()
    ref = ml_detect(y, h, s, pts, "maxlog", "bit")
    f32 = ml_detect(y, h, s, pts, "maxlog", "bit", dtype=np.complex64)
    bad = [envelope(f"full k {ns}x{2 ** m}-QAM real={real_rep} kbest", got, f32, ref, BAR),
           envelope(f"full k {ns}x{2 ** m}-QAM real={real_rep} ML kernel", ml, f32, ref, BAR)]
    assert not any(bad), "\n".join(b for b in bad if b)


ZERO_NOISE = [("qam", b, r, 3, 7, 64) for b in (2, 4, 6, 8) for r in (False, True)] + \
             [("pam", b, False, 4, 8, 16) for b in (1, 2, 3, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,bits,real_rep,ns,ant,k", ZERO_NOISE)
def test_noiseless_problems_have_no_errors(cuda_device, kind, bits, real_rep, ns, ant, k):
    """The reference's own zero-error cases: noiseless y = h x, s = 1e-9 I."""
    from sionna_b200.phy.mimo import KBestDetector
    rng = np.random.default_rng(70 + bits + 5 * real_rep + 11 * (kind == "pam"))
    pts = (MAP.qam(bits) if kind == "qam" else MAP.pam(bits)).astype(np.complex64)
    h = cnormal(rng, (100, ant, ns))
    ind = rng.integers(0, len(pts), (100, ns))
    y = (h @ pts[ind][..., None])[..., 0]
    s = (1e-9 * np.eye(ant)).astype(np.complex64)
    dev = [torch.from_numpy(v).to(cuda_device) for v in (y, h, s)]
    sym = KBestDetector("symbol", ns, k, kind, bits, hard_out=True, use_real_rep=real_rep)(*dev).cpu().numpy()
    assert np.array_equal(sym, ind)
    b = KBestDetector("bit", ns, k, kind, bits, hard_out=True, use_real_rep=real_rep)(*dev).cpu().numpy()
    assert np.array_equal(b, (ind[..., None] >> np.arange(bits - 1, -1, -1)) & 1)


# (name, batch, num_tx, streams per tx, num_rx, rx antennas, bits per symbol, association, k, real representation)
OFDM = [("2 rx interfering", 8, 2, 2, 2, 4, 4, [[1, 0], [0, 1]], 8, False),
        ("2 rx interfering real", 8, 2, 2, 2, 4, 4, [[1, 0], [0, 1]], 8, True),
        ("4x8 mu-mimo", 8, 4, 1, 1, 8, 4, [[1, 1, 1, 1]], 32, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", OFDM, ids=[c[0] for c in OFDM])
def test_ofdm_kbest_against_oracle(cuda_device, cfg):
    from sionna_b200.phy.ofdm import KBestDetector
    rng = np.random.default_rng(zlib.crc32(cfg[0].encode()))
    rg, sm, smr, y, h, ev, no, pts = ofdm_detection_case(cfg, rng, (0.02, 0.06))
    m, k, real_rep = cfg[6], cfg[8], cfg[9]
    ns = sm.num_streams_per_rx
    mask = rg.pilot_pattern.mask.astype(bool)
    args = [torch.as_tensor(v).to(cuda_device) for v in (y, h, ev, no)]
    y64, h64, ev64 = y.astype(np.complex128), h.astype(np.complex128), ev.astype(np.float64)
    ref, gap = ofdm_kbest_detect(y64, h64, ev64, no, mask, smr, pts, k, "bit", real_rep=real_rep)
    f32, _ = ofdm_kbest_detect(y, h, ev, no, mask, smr, pts, k, "bit", real_rep=real_rep, dtype=np.complex64)
    keep = _keep(cfg[0], gap)
    got = KBestDetector("bit", ns, k, rg, sm, "qam", m, use_real_rep=real_rep)(*args).cpu().numpy()
    assert got.shape == ref.shape
    shp = got.shape[:-1] + (-1, m)                              # one stream's LLRs of one RE share a scale
    bad = envelope(f"{cfg[0]} LLRs", got.reshape(shp)[keep], f32.reshape(shp)[keep], ref.reshape(shp)[keep], BAR)
    for output in ("bit", "symbol"):
        want, _ = ofdm_kbest_detect(y64, h64, ev64, no, mask, smr, pts, k, output, hard_out=True, real_rep=real_rep)
        hard = KBestDetector(output, ns, k, rg, sm, "qam", m, hard_out=True, use_real_rep=real_rep)(*args)
        assert hard.dtype == (torch.float32 if output == "bit" else torch.int32)
        hard = hard.cpu().numpy()
        if output == "bit":
            hard, want = hard.reshape(shp), want.reshape(shp)
        assert np.array_equal(hard[keep], want[keep]), f"{cfg[0]} hard {output}"
    assert not bad, bad


def _pusch_cell74(k=32):
    """The PUSCH tutorial's K-Best receiver: two transmitters with 4 antenna ports and 2 codebook-precoded layers each,
    16-QAM, KBestDetector as PUSCHReceiver's MIMO detector."""
    from sionna_b200.phy.nr import PUSCHConfig, PUSCHTransmitter, PUSCHReceiver
    from sionna_b200.phy.ofdm import KBestDetector
    from sionna_b200.phy.mimo import StreamManagement
    pusch_config = PUSCHConfig()
    pusch_config.num_antenna_ports = 4
    pusch_config.num_layers = 2
    pusch_config.dmrs.dmrs_port_set = [0, 1]
    pusch_config.precoding = "codebook"
    pusch_config.tpmi = 7
    pusch_config_1 = pusch_config.clone()
    pusch_config.dmrs.dmrs_port_set = [2, 3]
    pusch_transmitter = PUSCHTransmitter([pusch_config, pusch_config_1])
    rx_tx_association = np.ones([1, pusch_transmitter.resource_grid.num_tx], bool)
    stream_management = StreamManagement(rx_tx_association, pusch_config.num_layers)
    num_streams = pusch_transmitter.resource_grid.num_tx * pusch_transmitter.resource_grid.num_streams_per_tx
    k_best = KBestDetector("bit", num_streams, k, pusch_transmitter.resource_grid, stream_management, "qam",
                           pusch_config.tb.num_bits_per_symbol)
    pusch_receiver = PUSCHReceiver(pusch_transmitter, mimo_detector=k_best, return_tb_crc_status=True)
    return pusch_transmitter, pusch_receiver, stream_management


def _rayleigh(tx, batch, no):
    from sionna_b200.phy.channel import RayleighBlockFading, OFDMChannel
    rayleigh = RayleighBlockFading(num_rx=1, num_rx_ant=16, num_tx=tx.resource_grid.num_tx, num_tx_ant=4)
    channel = OFDMChannel(rayleigh, tx.resource_grid, normalize_channel=True)            # AWGN: call(x, no)
    x, b = tx(batch)
    return channel(x, no), b


@pytest.mark.gpu
def test_pusch_tutorial_receiver_decodes_at_high_snr(cuda_device):
    from sionna_b200.phy import config
    config.seed = 42
    tx, rx, _ = _pusch_cell74()
    y, b = _rayleigh(tx, 16, 0.01)
    b_hat, crc = rx(y, 0.01)
    assert bool(crc.all())
    assert torch.equal(b_hat, b)


@pytest.mark.gpu
def test_pusch_kbest_makes_no_more_hard_bit_errors_than_lmmse(cuda_device):
    """Same received batch and the same LS estimate: K-Best's hard coded bits have no more errors than LinearDetector's
    at the first noise level (of a fixed list, from the noisiest) where LinearDetector makes hundreds of errors, between
    100 and 2 000 (the counts are printed)."""
    from sionna_b200.phy import config
    from sionna_b200.phy.ofdm import KBestDetector, LinearDetector
    tx, rx, sm = _pusch_cell74()
    rg, m = tx.resource_grid, 4
    kb = KBestDetector("bit", rg.num_tx * rg.num_streams_per_tx, 32, rg, sm, "qam", m, hard_out=True)
    lin = LinearDetector("lmmse", "bit", "maxlog", rg, sm, "qam", m, hard_out=True)
    for no in (0.3, 0.2, 0.1, 0.05, 0.02):
        config.seed = 7
        y, b = _rayleigh(tx, 32, no)
        c = tx._tb_encoder(b)                                       # transmitted coded bits [batch, num_tx, n]
        h_hat, ev = rx._channel_estimator(y, no)
        e_kb = int((rx._layer_demapper(kb(y, h_hat, ev, no)) != c).sum())
        e_lin = int((rx._layer_demapper(lin(y, h_hat, ev, no)) != c).sum())
        print(f"no = {no}: hard coded-bit errors on {c.numel()} bits: K-Best {e_kb}, LMMSE {e_lin}")
        if 100 <= e_lin <= 2000:
            break
    assert 100 <= e_lin <= 2000
    assert e_kb <= e_lin


@pytest.mark.gpu
def test_ofdm_num_streams_must_match_stream_management(cuda_device):
    from sionna_b200.phy.ofdm import KBestDetector, ResourceGrid
    from sionna_b200.phy.mimo import StreamManagement
    rg = ResourceGrid(3, 12, 15e3, num_tx=1, num_streams_per_tx=2, pilot_pattern="kronecker",
                      pilot_ofdm_symbol_indices=[1])
    with pytest.raises(ValueError):
        KBestDetector("bit", 3, 16, rg, StreamManagement(np.ones((1, 1), int), 2), "qam", 4)


@pytest.mark.gpu
def test_constructor_errors(cuda_device):
    """The reference's argument assertions (test_kbest_det.py: test_wrong_parameters, test_init_*,
    test_wrong_constellation_for_real_rep, test_too_few_rx_antennas), k clipping, limits and list2llr."""
    from sionna_b200.phy.mimo import KBestDetector, List2LLR, List2LLRSimple
    from sionna_b200.phy.mapping import Constellation
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16)
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16, constellation_type="qam")
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16, num_bits_per_symbol=4)
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16, num_bits_per_symbol=4, constellation=Constellation("pam", 4))
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16, constellation_type="qam", constellation=Constellation("pam", 4))
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16, constellation_type="qam", num_bits_per_symbol=4,
                      constellation=Constellation("pam", 4))
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16, constellation=Constellation("pam", 4, precision="single"), precision="double")
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16, constellation=Constellation("pam", 4, precision="double"))
    with pytest.raises(AssertionError):
        KBestDetector("foo", 4, 16, "qam", 4)
    with pytest.raises(AssertionError):
        KBestDetector("symbol", 4, 16, "qam", 4)                        # soft symbols
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16, constellation_type="pam", use_real_rep=True)
    with pytest.raises(AssertionError):
        KBestDetector("bit", 4, 16, constellation=Constellation("pam", 4), use_real_rep=True)
    d = KBestDetector("bit", 4, 16, constellation_type="qam", num_bits_per_symbol=4)
    assert d._num_streams == 4 and d._num_symbols == 16 and d._k == 16 and np.allclose(np.var(d._constellation), 1.0)
    d = KBestDetector("bit", 4, 16, constellation=Constellation("pam", 4))
    assert d._num_streams == 4 and d._num_symbols == 16 and np.allclose(np.var(d._constellation), 1.0)
    for d in (KBestDetector("bit", 4, 16, "qam", 4, use_real_rep=True),
              KBestDetector("bit", 4, 16, constellation=Constellation("qam", 4), use_real_rep=True)):
        assert d._num_streams == 8 and d._num_symbols == 4 and d._k == 16
        assert np.allclose(np.var(d._constellation), 0.5)
    with pytest.warns(Warning):
        d = KBestDetector("bit", 2, 2 * 16 ** 2, "qam", 4)
    assert d._k == 256
    with pytest.raises(ValueError):
        KBestDetector("bit", 17, 16, "qam", 2)                          # 17 layers
    with pytest.raises(ValueError):
        KBestDetector("bit", 9, 16, "qam", 2, use_real_rep=True)        # 18 layers
    with pytest.raises(ValueError):
        KBestDetector("bit", 2, 128, "qam", 8)                          # 128 x 256 children
    with pytest.raises(AssertionError):
        KBestDetector("bit", 2, 16, "qam", 4, list2llr="simple")
    assert isinstance(KBestDetector("bit", 2, 16, "qam", 4).list2llr, List2LLRSimple)

    class Other(List2LLR):
        pass
    with pytest.raises(NotImplementedError):
        KBestDetector("bit", 2, 16, "qam", 4, list2llr=Other())
    # fewer receive antennas than streams (test_too_few_rx_antennas)
    rng = np.random.default_rng(1)
    pts = MAP.qam(4).astype(np.complex64)
    h = torch.from_numpy(cnormal(rng, (100, 3, 4))).to(cuda_device)
    y = h @ torch.from_numpy(pts[rng.integers(0, 16, (100, 4, 1))]).to(cuda_device)
    s = torch.from_numpy((1e-9 * np.eye(3)).astype(np.complex64)).to(cuda_device)
    for real_rep in (False, True):
        with pytest.raises(AssertionError):
            KBestDetector("symbol", 4, 64, "qam", 4, use_real_rep=real_rep, hard_out=True)(y[..., 0], h, s)


@pytest.mark.gpu
def test_double_precision_falls_back_with_a_warning(cuda_device):
    from sionna_b200.phy.mimo import KBestDetector
    from sionna_b200.phy.block import PrecisionWarning
    rng = np.random.default_rng(5)
    pts = MAP.qam(2).astype(np.complex64)                       # QPSK: the same fp32 points in both precisions
    y, h, s = mimo_problem(rng, 256, 4, 2, pts, 0.1)
    single = KBestDetector("bit", 2, 8, "qam", 2)(*(torch.from_numpy(v).to(cuda_device) for v in (y, h, s)))
    with pytest.warns(PrecisionWarning):
        double = KBestDetector("bit", 2, 8, "qam", 2, precision="double")(
            *(torch.from_numpy(v.astype(np.complex128)).to(cuda_device) for v in (y, h, s)))
    assert double.dtype == torch.float64
    assert torch.equal(double.float(), single)
