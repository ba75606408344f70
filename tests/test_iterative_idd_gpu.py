"""The perfect-CSI half of the iterative detection and decoding (IDD) tutorial as a seeded test: 4 single-antenna UEs,
16 receive antennas, 16-QAM, 14 x 48 grid with pilots on symbols 2 and 11, LDPC5G rate 1/2 (k = 1152, n = 2304),
min-sum with 12 BP iterations per decoding, i.i.d. Rayleigh block fading through OFDMChannel, perfect CSI.

  LMMSE:   LinearDetector -> decoder
  EP:      EPDetector(l = 10) -> decoder
  IDD(I):  LinearDetector -> (stateful decoder -> MMSEPICDetector with the decoder's a-posteriori LLRs as prior)
           x (I - 1) -> stateful decoder (the tutorial's IddModel)

At the first Eb/N0 of a fixed list (from -10 dB up) where LMMSE's BLER lies in 0.1 ... 0.9 on a probe batch, every
receiver runs on the same transmitted frames; IDD with 3 iterations must beat IDD with 2, which must beat LMMSE, and EP
must beat LMMSE, each by more than three standard errors of the difference. Measured on an H100: the probe stops at
-7 dB (LMMSE probe BLER 0.348); block errors of 4096 codewords: LMMSE 1442, EP 1196, IDD I=2 225, IDD I=3 78."""
import numpy as np
import pytest
import torch


class Link:
    def __init__(self):
        from sionna_b200.phy.ofdm import ResourceGrid, ResourceGridMapper, LinearDetector, EPDetector, MMSEPICDetector
        from sionna_b200.phy.mimo import StreamManagement
        from sionna_b200.phy.mapping import Mapper, BinarySource
        from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
        from sionna_b200.phy.channel import RayleighBlockFading, OFDMChannel
        self.m, self.n_ue = 4, 4
        self.rg = rg = ResourceGrid(num_ofdm_symbols=14, pilot_ofdm_symbol_indices=[2, 11], fft_size=48,
                                    num_tx=self.n_ue, pilot_pattern="kronecker", subcarrier_spacing=30e3)
        sm = StreamManagement(np.ones([1, self.n_ue]), 1)
        self.n = 48 * 12 * self.m
        self.k = self.n // 2
        self.enc = LDPC5GEncoder(self.k, self.n, num_bits_per_symbol=self.m)
        self.src, self.mapper, self.rgm = BinarySource(), Mapper("qam", self.m), ResourceGridMapper(rg)
        self.channel = OFDMChannel(RayleighBlockFading(1, 16, self.n_ue, 1), rg, normalize_channel=True,
                                   return_channel=True)
        self.lmmse = LinearDetector("lmmse", "bit", "maxlog", rg, sm, "qam", self.m)
        self.ep = EPDetector("bit", rg, sm, self.m, l=10)
        self.pic = MMSEPICDetector("bit", "maxlog", rg, sm, 1, "qam", self.m)
        self.dec = LDPC5GDecoder(self.enc, return_infobits=True, hard_out=True, num_iter=12, cn_update="minsum")
        self.siso_dec = LDPC5GDecoder(self.enc, return_infobits=False, hard_out=False, num_iter=12,
                                      return_state=True, cn_update="minsum")
        self.final_dec = LDPC5GDecoder(self.enc, return_infobits=True, hard_out=True, num_iter=12, return_state=True,
                                       cn_update="minsum")

    def frames(self, batch, ebno_db):
        from sionna_b200.phy.utils import ebnodb2no
        no = float(ebnodb2no(ebno_db, self.m, 0.5))
        b = self.src([batch, self.n_ue, 1, self.k])
        y, h = self.channel(self.rgm(self.mapper(self.enc(b))), no)
        return b, y, h, no

    def block_errors(self, b, b_hat):
        return int((b != b_hat).any(-1).sum())

    def lmmse_rx(self, y, h, no):
        return self.dec(self.lmmse(y, h, 0.0, no))

    def ep_rx(self, y, h, no):
        return self.dec(self.ep(y, h, 0.0, no))

    def idd_rx(self, y, h, no, num_idd_iter):
        llr_ch = self.lmmse(y, h, 0.0, no)
        msg = None
        for _ in range(num_idd_iter - 1):
            llr_dec, msg = self.siso_dec(llr_ch, msg_v2c=msg)
            llr_ch = self.pic(y, h, llr_dec, 0.0, no)
        b_hat, _ = self.final_dec(llr_ch, msg_v2c=msg)
        return b_hat


@pytest.mark.gpu
def test_idd_tutorial_perfect_csi_bler_ordering(cuda_device):
    from sionna_b200.phy import config
    link = Link()
    for ebno_db in (-10.0, -9.0, -8.0, -7.0, -6.0, -5.0, -4.0, -3.0, -2.0, -1.0, 0.0):
        config.seed = 11
        b, y, h, no = link.frames(64, ebno_db)
        probe = link.block_errors(b, link.lmmse_rx(y, h, no)) / b[..., 0].numel()
        print(f"Eb/N0 = {ebno_db} dB: LMMSE probe BLER {probe:.3f}")
        if 0.1 <= probe <= 0.9:
            break
    assert 0.1 <= probe <= 0.9
    counts = {"LMMSE": 0, "EP l=10": 0, "IDD I=2": 0, "IDD I=3": 0}
    total = 0
    for rep in range(16):
        config.seed = 1000 + rep
        b, y, h, no = link.frames(64, ebno_db)
        total += b[..., 0].numel()
        counts["LMMSE"] += link.block_errors(b, link.lmmse_rx(y, h, no))
        counts["EP l=10"] += link.block_errors(b, link.ep_rx(y, h, no))
        counts["IDD I=2"] += link.block_errors(b, link.idd_rx(y, h, no, 2))
        counts["IDD I=3"] += link.block_errors(b, link.idd_rx(y, h, no, 3))
    print(f"Eb/N0 = {ebno_db} dB, {total} codewords: block errors {counts}")

    def clearly_below(a, c):
        pa, pc = counts[a] / total, counts[c] / total
        se = np.sqrt((pa * (1 - pa) + pc * (1 - pc)) / total)
        return pc - pa > 3 * se
    assert clearly_below("IDD I=3", "IDD I=2"), counts
    assert clearly_below("IDD I=2", "LMMSE"), counts
    assert clearly_below("EP l=10", "LMMSE"), counts
