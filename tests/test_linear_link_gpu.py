"""The reference's test_all_detectors_in_all_modes (test/integration/test_mimo_ofdm_detectors.py:110-127) for the
linear detectors: mf / zf / lmmse x bit / symbol through a coded CDL link, in single precision.

The model is the reference's OFDMModel: a CDL-A uplink (100 ns, 2.6 GHz, 3 m/s) from a 4-antenna UT (1 x 2 dual-polarised
cross 38.901) to an 8-antenna BS (1 x 4), 4 streams, a 14 x 12 grid without pilots, 16-QAM and rate 1/2 LDPC. The
channel adds no noise and the detector is given no = 1e-4 with perfect CSI (err_var 0). Bit outputs are maxlog LLRs
decoded by LDPC5GDecoder; symbol outputs are hard symbol indices compared with the mapped ones. As in the reference,
the error rate must be 0 for lmmse and zf and below 1 for mf, at batch 4 (the reference's batch)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

FC = 2.6e9


class _OFDMModel:
    def __init__(self, detector, output):
        from sionna_b200.phy.mimo import StreamManagement
        from sionna_b200.phy.ofdm import ResourceGrid, ResourceGridMapper, LinearDetector
        from sionna_b200.phy.channel import AntennaArray, CDL, OFDMChannel
        from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
        from sionna_b200.phy.mapping import Mapper, BinarySource
        self.num_streams = 4
        m = 4
        self.sm = StreamManagement(np.array([[1]]), self.num_streams)
        self.rg = ResourceGrid(num_ofdm_symbols=14, fft_size=12, subcarrier_spacing=15e3, num_tx=1,
                               num_streams_per_tx=self.num_streams)
        self.n = int(self.rg.num_data_symbols * m)
        self.k = int(self.n * 0.5)
        ut = AntennaArray(1, 2, "dual", "cross", "38.901", FC)
        bs = AntennaArray(1, 4, "dual", "cross", "38.901", FC)
        cdl = CDL("A", 100e-9, FC, ut, bs, "uplink", min_speed=3.0)
        self.channel = OFDMChannel(cdl, self.rg, normalize_channel=True, return_channel=True)
        self.source = BinarySource()
        self.encoder = LDPC5GEncoder(self.k, self.n)
        self.decoder = LDPC5GDecoder(self.encoder, hard_out=True)
        self.mapper = Mapper("qam", m, return_indices=True)
        self.rg_mapper = ResourceGridMapper(self.rg)
        self.output = output
        self.detector = LinearDetector(detector, output, "maxlog", self.rg, self.sm, "qam", m,
                                       hard_out=output == "symbol")

    def __call__(self, batch_size):
        b = self.source([batch_size, 1, self.num_streams, self.k])
        x, x_ind = self.mapper(self.encoder(b))
        y, h = self.channel(self.rg_mapper(x))
        z = self.detector(y, h, 0.0, 1e-4)
        if self.output == "symbol":
            return x_ind, z
        return b, self.decoder(z)


@pytest.mark.parametrize("output", ["bit", "symbol"])
@pytest.mark.parametrize("detector", ["mf", "lmmse", "zf"])
def test_all_linear_detectors_cdl_link(cuda_device, detector, output):
    from sionna_b200.phy import config
    config.seed = 41
    ref, est = _OFDMModel(detector, output)(4)
    assert ref.shape == est.shape
    err = float((ref.to(torch.int64) != est.to(torch.int64)).double().mean())
    print(f"{detector} {output}: error rate {err:.3e}")
    if detector == "mf":
        assert err < 1
    else:
        assert err == 0
