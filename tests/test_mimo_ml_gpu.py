"""Maximum-likelihood MIMO detection (sb_mimo_ml / sb_ofdm_ml) against the NumPy oracle (oracle/mimo.py).

Soft outputs are held to the reference's own single-precision envelope: the kernel's rms and max error against the
complex128 oracle stay within 2x (rms) and 4x (max) of the complex64 evaluation's error on the same inputs, errors taken
relative to the rms of the reference output of each stream (logits or LLRs of one stream share a scale). Hard outputs
equal the complex128 oracle wherever its decision margin exceeds that soft-output bound."""
import zlib

import numpy as np
import pytest
import torch

from oracle import mapping as MAP
from oracle.mimo import ml_detect, ofdm_ml_detect
from oracle.parity import constellation, envelope, mimo_problem, ofdm_detection_case

pytestmark = pytest.mark.gpu

BAR = (2.0, 4.0)
BARS = {                                        # (rms, max) bars of the cases that need their own, worst measured ratio
    "K4-16qam M16": (2.6, 4.0),                 # 2.10 / 1.86: whitening and Gram-Schmidt accumulate 16 antennas in
    "4x16 mu-mimo": (2.6, 4.0),                 # 2.46 / 3.06: sequence, LAPACK in blocks (as the LMMSE bars)
    "M<K (1 antenna, 2 streams)": (2.5, 4.0),   # 2.09 / 2.32, bit app with prior
    "custom 8-point": (5.0, 8.0),               # 4.41 / 6.50, bit app without prior: this random constellation's app
}                                               # LLRs are small next to its logits, the difference keeps the kernel's
                                                # independent rounding of each point's exp sum (symbol logits: 1.16 / 1.24)


def _margin_bound(f32, ref, symbol, bar=BAR):
    """Absolute soft-output bound: bar[1] times the complex64 evaluation's largest error, for symbols over the two
    largest logits of each element (the ones the decision compares)."""
    err = np.abs(np.where(np.isfinite(ref), f32 - ref, 0))
    if symbol:
        top2 = np.argsort(ref, axis=-1)[..., -2:]
        err = np.take_along_axis(err, top2, axis=-1)
    return bar[1] * float(err.max())


def _hard_check(what, got, ref_soft, ref_hard, bound, symbol):
    """got == ref_hard wherever the complex128 decision margin exceeds bound; fewer than 1 % excluded."""
    if symbol:
        srt = np.sort(ref_soft, axis=-1)
        margin = srt[..., -1] - srt[..., -2]
    else:
        margin = np.abs(ref_soft)
    keep = margin > bound
    excluded = 1.0 - keep.mean()
    print(f"{what}: hard outputs, {excluded:.3%} excluded (margin <= {bound:.2e})")
    assert excluded < 0.01, what
    assert np.array_equal(got[keep], ref_hard[keep]), what


# (name, K, bits per symbol, M, constellation type, problems, no)
DENSE = [(f"K{k}-{'qpsk' if m == 2 else '16qam'}", k, m, 4, "qam", 128 if m ** k >= 4 ** 4 else 512, 0.1)
         for k in (1, 2, 3, 4) for m in (2, 4)]
DENSE += [("8 streams qpsk", 8, 2, 8, "qam", 64, 0.1),
          ("K4-16qam M16", 4, 4, 16, "qam", 64, 0.1),
          ("2 streams 256qam", 2, 8, 4, "qam", 96, 0.002),
          ("1 stream 1024qam", 1, 10, 2, "qam", 2048, 2e-4),
          ("custom 8-point", 2, 3, 3, "custom", 256, 0.1),
          ("M<K (1 antenna, 2 streams)", 2, 2, 1, "qam", 512, 0.1)]


@pytest.mark.parametrize("case", DENSE, ids=[c[0] for c in DENSE])
def test_dense_ml_against_oracle(cuda_device, case):
    from sionna_b200.phy.mimo import MaximumLikelihoodDetector
    name, k, m, mm, kind, num, no = case
    const = constellation(kind, m)
    pts = const().cpu().numpy().astype(np.complex64)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    y, h, s = mimo_problem(rng, num, mm, k, pts, no)
    dev = [torch.from_numpy(v).to(cuda_device) for v in (y, h, s)]
    bad = []
    for output in ("bit", "symbol"):
        for method in ("app", "maxlog"):
            for with_prior in (False, True):
                prior = None
                if with_prior:
                    prior = rng.normal(size=(num, k, m if output == "bit" else 2 ** m)).astype(np.float32)
                tag = f"{name} {output} {method} prior={with_prior}"
                ref = ml_detect(y, h, s, pts, method, output, prior)
                f32 = ml_detect(y, h, s, pts, method, output, prior, dtype=np.complex64)
                pd = None if prior is None else torch.from_numpy(prior).to(cuda_device)
                det = MaximumLikelihoodDetector(output, method, k, constellation=const)
                got = det(*dev, prior=pd).cpu().numpy()
                assert got.shape == ref.shape, tag
                bad.append(envelope(tag, got, f32, ref, BARS.get(name, BAR)))
                hard = MaximumLikelihoodDetector(output, method, k, constellation=const, hard_out=True)(*dev, prior=pd)
                want = ml_detect(y, h, s, pts, method, output, prior, hard_out=True)
                assert hard.dtype == (torch.float32 if output == "bit" else torch.int32)
                _hard_check(tag, hard.cpu().numpy(), ref, want, _margin_bound(f32, ref, output == "symbol"), output == "symbol")
    assert not any(bad), "\n".join(b for b in bad if b)


def test_dense_ml_leading_batch_dims(cuda_device):
    from sionna_b200.phy.mimo import MaximumLikelihoodDetector
    rng = np.random.default_rng(3)
    pts = MAP.qam(4).astype(np.complex64)
    y, h, s = mimo_problem(rng, 24, 4, 2, pts, 0.1)
    det = MaximumLikelihoodDetector("bit", "app", 2, "qam", 4)
    flat = det(*(torch.from_numpy(v).to(cuda_device) for v in (y, h, s)))
    shaped = det(*(torch.from_numpy(v.reshape((2, 3, 4) + v.shape[1:])).to(cuda_device) for v in (y, h, s)))
    assert shaped.shape == (2, 3, 4, 2, 4)
    assert torch.equal(shaped.reshape(flat.shape), flat)


@pytest.mark.parametrize("output", ["bit", "symbol"])
def test_high_snr_outputs_stay_finite(cuda_device, output):
    """no = 1e-4, 4 streams of 16-QAM: a single global offset would underflow exp() for the points far from the ML
    solution; the per-accumulator offsets keep every output finite where the oracle's is."""
    from sionna_b200.phy.mimo import MaximumLikelihoodDetector
    rng = np.random.default_rng(17)
    pts = MAP.qam(4).astype(np.complex64)
    y, h, s = mimo_problem(rng, 128, 4, 4, pts, 1e-4)
    ref = ml_detect(y, h, s, pts, "app", output)
    f32 = ml_detect(y, h, s, pts, "app", output, dtype=np.complex64)
    got = MaximumLikelihoodDetector(output, "app", 4, "qam", 4)(*(torch.from_numpy(v).to(cuda_device) for v in (y, h, s)))
    got = got.cpu().numpy()
    assert np.all(np.isfinite(got[np.isfinite(ref)]))
    bad = envelope(f"high SNR {output}", got, f32, ref, BAR)
    assert not bad, bad


def test_oversize_configuration_is_rejected_before_launch():
    from sionna_b200.phy.mimo import MaximumLikelihoodDetector
    from sionna_b200.phy.ofdm import MaximumLikelihoodDetector as OFDMML, ResourceGrid
    from sionna_b200.phy.mimo import StreamManagement
    with pytest.raises(ValueError):
        MaximumLikelihoodDetector("bit", "app", 5, "qam", 4)            # 16^5 candidates
    with pytest.raises(ValueError):
        MaximumLikelihoodDetector("bit", "app", 9, "qam", 2)            # 9 streams
    rg = ResourceGrid(2, 12, 15e3, num_tx=1, num_streams_per_tx=3, pilot_pattern="kronecker",
                      pilot_ofdm_symbol_indices=[0])
    with pytest.raises(ValueError):
        OFDMML("bit", "app", rg, StreamManagement(np.ones((1, 1), int), 3), "qam", 8)   # 256^3


# (name, batch, num_tx, streams per tx, num_rx, rx antennas, bits per symbol, association, err_var shape, no shape)
OFDM = [("siso", 16, 1, 1, 1, 1, 4, [[1]], (), ()),
        ("4x16 mu-mimo", 2, 4, 1, 1, 16, 4, [[1, 1, 1, 1]], (2, 1, 16, 4, 1, 3, 12), (2, 1, 16)),
        ("2 rx interfering", 4, 2, 2, 2, 4, 2, [[1, 0], [0, 1]], (4, 2, 4, 2, 2, 3, 12), (4, 2)),
        ("ev per antenna, no per batch", 4, 1, 2, 1, 3, 4, [[1]], (1, 1, 3, 1, 1, 1, 1), (4,)),
        ("ev over time and frequency", 4, 1, 2, 1, 3, 2, [[1]], (3, 12), (4, 1, 3))]


@pytest.mark.parametrize("cfg", OFDM, ids=[c[0] for c in OFDM])
def test_ofdm_ml_against_oracle(cuda_device, cfg):
    from sionna_b200.phy.ofdm import MaximumLikelihoodDetector
    rng = np.random.default_rng(zlib.crc32(cfg[0].encode()))
    rg, sm, smr, y, h, ev, no, pts = ofdm_detection_case(cfg, rng, (0.05, 0.15), cfg[8], cfg[9])
    mask = rg.pilot_pattern.mask.astype(bool)
    m = cfg[6]
    args = [torch.as_tensor(v).to(cuda_device) for v in (y, h, ev, no)]
    bad = []
    for output in ("bit", "symbol"):
        for method in ("app", "maxlog"):
            tag = f"{cfg[0]} {output} {method}"
            ref = ofdm_ml_detect(y.astype(np.complex128), h.astype(np.complex128), np.asarray(ev, np.float64), no, mask,
                                 smr, pts, method, output)
            f32 = ofdm_ml_detect(y, h, ev, no, mask, smr, pts, method, output, dtype=np.complex64)
            got = MaximumLikelihoodDetector(output, method, rg, sm, "qam", m)(*args).cpu().numpy()
            assert got.shape == ref.shape, tag
            if output == "bit":                                     # one stream's LLRs of one RE share a scale
                shp = got.shape[:-1] + (-1, m)
                got, ref, f32 = got.reshape(shp), ref.reshape(shp), f32.reshape(shp)
            bad.append(envelope(tag, got, f32, ref, BARS.get(cfg[0], BAR)))
    for output in ("bit", "symbol"):                                # hard bits and hard symbol indices
        sym = output == "symbol"
        hard = MaximumLikelihoodDetector(output, "maxlog", rg, sm, "qam", m, hard_out=True)(*args).cpu().numpy()
        want = ofdm_ml_detect(y.astype(np.complex128), h.astype(np.complex128), np.asarray(ev, np.float64), no, mask,
                              smr, pts, "maxlog", output, hard_out=True)
        soft = ofdm_ml_detect(y.astype(np.complex128), h.astype(np.complex128), np.asarray(ev, np.float64), no, mask,
                              smr, pts, "maxlog", output)
        soft32 = ofdm_ml_detect(y, h, ev, no, mask, smr, pts, "maxlog", output, dtype=np.complex64)
        assert hard.dtype == (np.int32 if sym else np.float32)
        _hard_check(f"{cfg[0]} {output} hard", hard, soft, want, _margin_bound(soft32, soft, sym), sym)
    assert not any(bad), "\n".join(b for b in bad if b)


@pytest.mark.parametrize("output", ["bit", "symbol"])
@pytest.mark.parametrize("streams", [2, 4])                     # 2 x 16-QAM: thread per element, 4 x: warp
def test_ofdm_ml_with_prior_single_receiver(cuda_device, output, streams):
    from sionna_b200.phy.ofdm import MaximumLikelihoodDetectorWithPrior
    cfg = ("prior", 2, 1, streams, 1, 4, 4, [[1]], (2, 1, 4, 1, streams, 3, 12), (2, 1, 4))
    rng = np.random.default_rng(23 + (output == "bit") + 10 * streams)
    rg, sm, smr, y, h, ev, no, pts = ofdm_detection_case(cfg, rng, (0.05, 0.15), cfg[8], cfg[9])
    mask = rg.pilot_pattern.mask.astype(bool)
    nd = rg.num_data_symbols
    shape = (2, 1, streams, nd * 4) if output == "bit" else (2, 1, streams, nd, 16)
    prior = rng.normal(size=shape).astype(np.float32)
    bad = []
    for method in ("app", "maxlog"):
        ref = ofdm_ml_detect(y.astype(np.complex128), h.astype(np.complex128), np.asarray(ev, np.float64), no, mask,
                             smr, pts, method, output, prior=prior)
        f32 = ofdm_ml_detect(y, h, ev, no, mask, smr, pts, method, output, prior=prior, dtype=np.complex64)
        det = MaximumLikelihoodDetectorWithPrior(output, method, rg, sm, "qam", 4)
        args = [torch.as_tensor(v).to(cuda_device) for v in (y, h, prior, ev, no)]
        got = det(*args).cpu().numpy()
        if output == "bit":
            got, ref, f32 = (v.reshape(v.shape[:-1] + (-1, 4)) for v in (got, ref, f32))
        bad.append(envelope(f"with prior {streams} streams {output} {method}", got, f32, ref, BAR))
    assert not any(bad), "\n".join(b for b in bad if b)


def test_pusch_receiver_with_ml_detector_decodes(cuda_device):
    """PUSCHReceiver takes the OFDM ML detector as mimo_detector and recovers every transport block at high SNR."""
    from sionna_b200.phy.nr import PUSCHConfig, PUSCHTransmitter, PUSCHReceiver
    from sionna_b200.phy.ofdm import MaximumLikelihoodDetector
    from sionna_b200.phy.mimo import StreamManagement
    from sionna_b200.phy.channel import AWGN
    from sionna_b200.phy import config
    config.seed = 11
    pc = PUSCHConfig(num_layers=2, num_antenna_ports=2)
    pc.carrier.n_size_grid = 8
    tx = PUSCHTransmitter(pc)
    sm = StreamManagement(np.ones((1, 1), bool), 2)
    det = MaximumLikelihoodDetector("bit", "maxlog", tx.resource_grid, sm, "qam", pc.tb.num_bits_per_symbol)
    rx = PUSCHReceiver(tx, mimo_detector=det, stream_management=sm, return_tb_crc_status=True)
    x, b = tx(16)                                                   # [16, 1, 2 ports, 14, F]
    g = torch.Generator(device="cpu").manual_seed(5)
    hch = torch.complex(torch.randn(16, 1, 4, 1, 2, 1, 1, generator=g),
                        torch.randn(16, 1, 4, 1, 2, 1, 1, generator=g)).to(cuda_device) / np.sqrt(2)
    y = torch.einsum("brmtp,btpsf->brmsf", hch[..., 0, 0], x)
    y = AWGN()(y, 0.001)
    b_hat, crc = rx(y, 0.001)
    assert bool(crc.all())
    assert torch.equal(b_hat, b)


def test_ml_makes_fewer_uncoded_bit_errors_than_lmmse(cuda_device):
    """4 streams of 16-QAM on 4 receive antennas (perfect CSI, Rayleigh per RE): the ML detector's hard bits have fewer
    errors than LinearDetector's on the same >= 1e5 bits."""
    from sionna_b200.phy.ofdm import MaximumLikelihoodDetector, LinearDetector, ResourceGrid, ResourceGridMapper
    from sionna_b200.phy.mimo import StreamManagement
    from sionna_b200.phy.mapping import Mapper, BinarySource
    from sionna_b200.phy import config
    config.seed = 3
    rg = ResourceGrid(14, 76, 15e3, num_tx=1, num_streams_per_tx=4, pilot_pattern="kronecker",
                      pilot_ofdm_symbol_indices=[2, 11])
    sm = StreamManagement(np.ones((1, 1), int), 4)
    nd, b = rg.num_data_symbols, 24
    bits = BinarySource(seed=1)([b, 1, 4, nd * 4])
    xg = ResourceGridMapper(rg)(Mapper("qam", 4)(bits))                      # [b, 1, 4, 14, 76]
    g = torch.Generator(device="cpu").manual_seed(9)

    def crandn(*shape):
        return (torch.complex(torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)) / np.sqrt(2)).to(cuda_device)

    h = crandn(b, 1, 4, 1, 4, 14, 76)
    no = 0.05
    y = torch.einsum("brmtksf,btksf->brmsf", h, xg) + crandn(b, 1, 4, 14, 76) * np.sqrt(no)
    ml = MaximumLikelihoodDetector("bit", "maxlog", rg, sm, "qam", 4, hard_out=True)(y, h, 0.0, no)
    lin = LinearDetector("lmmse", "bit", "maxlog", rg, sm, "qam", 4, hard_out=True)(y, h, 0.0, no)
    assert bits.numel() >= 1e5
    e_ml, e_lin = int((ml != bits).sum()), int((lin != bits).sum())
    print(f"uncoded bit errors on {bits.numel()} bits: ML {e_ml}, LMMSE {e_lin}")
    assert e_ml < e_lin


def test_double_precision_falls_back_with_a_warning(cuda_device):
    from sionna_b200.phy.mimo import MaximumLikelihoodDetector
    from sionna_b200.phy.block import PrecisionWarning
    rng = np.random.default_rng(5)
    pts = MAP.qam(2).astype(np.complex64)
    y, h, s = mimo_problem(rng, 64, 2, 2, pts, 0.1)
    single = MaximumLikelihoodDetector("bit", "app", 2, "qam", 2)(*(torch.from_numpy(v).to(cuda_device) for v in (y, h, s)))
    with pytest.warns(PrecisionWarning):
        double = MaximumLikelihoodDetector("bit", "app", 2, "qam", 2, precision="double")(
            *(torch.from_numpy(v.astype(np.complex128)).to(cuda_device) for v in (y, h, s)))
    assert double.dtype == torch.float64
    assert torch.equal(double.float(), single)
