"""Transmit precoding on the device (sb_mimo_precode, sb_ofdm_precode) against the complex128 oracle
(oracle/precoding.py): the kernel's error stays within 2x (rms) / 4x (max) of the complex64 evaluation's, the bar the
detectors use. Errors below one float32 ulp of the rms (2^-23 rms, 2^-21 max) are not compared: CBF and the identity
precoder are a normalisation and a scale, whose complex64 error is a rounding or two. Then the reference's checks
(zero forcing diagonalises the channel, RZFPrecodedChannel against the literal loop), the consistency of h_eff with
the precoded transmission, the errors and the downlink CDL links."""
import warnings

import numpy as np
import pytest
import torch

from oracle import precoding as P
from oracle.ofdm import eff_sc_ind
from oracle.parity import cnormal, envelope

pytestmark = pytest.mark.gpu

BAR = (2.0, 4.0)
FLOOR = (2.0 ** -23, 2.0 ** -21)
FC = 2.6e9


def _dev(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _check(what, got, f32, ref, axis=None):
    line = envelope(what, got.cpu().numpy().astype(np.complex128), f32.astype(np.complex128), ref, BAR, FLOOR,
                    axis=axis)
    assert not line, line


# ---- dense functions -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", ["zero", "scalar", "tensor"])
@pytest.mark.parametrize("M", ["K", 15, 64])
@pytest.mark.parametrize("K", [1, 2, 4, 10, 16])
def test_dense_precoding_matrices(cuda_device, K, M, alpha):
    from sionna_b200.phy.mimo import rzf_precoding_matrix, cbf_precoding_matrix, rzf_precoder
    m = K if M == "K" else M
    if m < K and alpha == "zero":
        pytest.skip("singular Gram matrix (alpha = 0, K > M): not finite, not tested")
    rng = np.random.default_rng(1000 * K + m)
    num = 512
    h = cnormal(rng, (num, K, m))
    x = cnormal(rng, (num, K))
    al = {"zero": 0.0, "scalar": 0.25, "tensor": rng.uniform(0.01, 1.0, num).astype(np.float32)}[alpha]
    al_d = _dev(al, cuda_device) if alpha == "tensor" else al
    hd = _dev(h, cuda_device)
    g = rzf_precoding_matrix(hd, al_d)
    assert g.shape == (num, m, K) and g.dtype == torch.complex64
    ref = P.rzf_precoding_matrix(h, al)
    _check(f"rzf G K={K} M={m} {alpha}", g, P.rzf_precoding_matrix(h, al, np.complex64), ref, (-2, -1))
    gx, g2 = rzf_precoder(_dev(x, cuda_device), hd, al_d, return_precoding_matrix=True)
    assert torch.equal(g2, g)
    xr, _ = P.rzf_precoder(x, h, al)
    _check(f"rzf Gx K={K} M={m} {alpha}", gx, P.rzf_precoder(x, h, al, np.complex64)[0], xr, -1)
    if alpha == "zero":
        gc = cbf_precoding_matrix(hd)
        _check(f"cbf G K={K} M={m}", gc, P.cbf_precoding_matrix(h, np.complex64), P.cbf_precoding_matrix(h), (-2, -1))


def test_zf_diagonalises_the_channel_on_the_device(cuda_device):
    """The reference's test_rzf_precoder: K = 10, M = 15, alpha = 0."""
    from sionna_b200.phy.mimo import rzf_precoder
    rng = np.random.default_rng(7)
    h = _dev(cnormal(rng, (1000, 10, 15)), cuda_device)
    x = _dev(cnormal(rng, (1000, 10)), cuda_device)
    xp, g = rzf_precoder(x, h, return_precoding_matrix=True)
    hg = h @ g
    off = hg - torch.diag_embed(torch.diagonal(hg, dim1=-2, dim2=-1))
    assert float(off.abs().pow(2).sum().sqrt()) < 1e-4 * float(hg.abs().pow(2).sum().sqrt())
    assert torch.allclose((g.abs() ** 2).sum(-2), torch.ones(1000, 10, device=cuda_device), atol=1e-5)
    assert torch.allclose(xp, (g @ x[..., None])[..., 0], atol=1e-5)


def test_dense_broadcasting_and_double(cuda_device):
    from sionna_b200.phy.mimo import rzf_precoding_matrix
    from sionna_b200.phy import block
    rng = np.random.default_rng(8)
    h = cnormal(rng, (3, 5, 2, 4))
    al = rng.uniform(0.1, 1.0, 3).astype(np.float32)                   # aligned with h's first batch dimension
    g = rzf_precoding_matrix(_dev(h, cuda_device), _dev(al, cuda_device)).cpu().numpy()
    ref = P.rzf_precoding_matrix(h, al)
    assert np.allclose(g, ref, atol=1e-5)
    block._warned_double.discard("rzf_precoding_matrix")
    with pytest.warns(block.PrecisionWarning):
        g2 = rzf_precoding_matrix(_dev(h, cuda_device), 0.5, precision="double")
    assert g2.dtype == torch.complex128


# ---- OFDM blocks -----------------------------------------------------------------------------------------------------
def _case(name):
    """(rg, sm, assoc, num_rx_ant, num_tx_ant, batch)"""
    from sionna_b200.phy.ofdm import ResourceGrid
    from sionna_b200.phy.mimo import StreamManagement
    if name == "tutorial":                        # CDL tutorial downlink: 8-antenna BS to a 4-antenna UT
        assoc, ra, m, b = np.ones((1, 1), np.int32), 4, 8, 16
        rg = ResourceGrid(14, 76, 15e3, num_tx=1, num_streams_per_tx=4, cyclic_prefix_length=6,
                          num_guard_carriers=(5, 6), dc_null=True, pilot_pattern="kronecker",
                          pilot_ofdm_symbol_indices=[2, 11])
    elif name == "multi_user":                    # 2 transmitters, each serving 2 of 4 two-antenna receivers
        assoc, ra, m, b = np.kron(np.eye(2, dtype=np.int32), np.ones((2, 1), np.int32)), 2, 8, 8
        rg = ResourceGrid(4, 24, 15e3, num_tx=2, num_streams_per_tx=4, num_guard_carriers=(2, 1), dc_null=True)
    else:                                         # massive MIMO: M = 64 to 8 two-antenna UTs, K = 16
        assoc, ra, m, b = np.ones((8, 1), np.int32), 2, 64, 2
        rg = ResourceGrid(2, 64, 15e3, num_tx=1, num_streams_per_tx=16, num_guard_carriers=(4, 3), dc_null=True)
    sm = StreamManagement(assoc, rg.num_streams_per_tx)
    return rg, sm, assoc, ra, m, b


def _eff(rg):
    return np.asarray(rg.effective_subcarrier_ind)


@pytest.mark.parametrize("alpha", ["scalar", "tensor"])
@pytest.mark.parametrize("name", ["tutorial", "multi_user", "massive"])
def test_rzf_precoder_against_oracle(cuda_device, name, alpha):
    from sionna_b200.phy.ofdm import RZFPrecoder
    rg, sm, assoc, ra, m, b = _case(name)
    rng = np.random.default_rng(len(name) * 7 + len(alpha))
    rx, tx, k, s_, f_ = assoc.shape[0], assoc.shape[1], sm.num_streams_per_tx, rg.num_ofdm_symbols, rg.fft_size
    h = cnormal(rng, (b, rx, ra, tx, m, s_, f_))
    x = cnormal(rng, (b, tx, k, s_, f_))
    al = 0.1 if alpha == "scalar" else rng.uniform(0.0, 0.5, (b, tx, s_, f_)).astype(np.float32)
    prec = RZFPrecoder(rg, sm, return_effective_channel=True)
    xp, h_eff = prec(_dev(x, cuda_device), _dev(h, cuda_device), al if alpha == "scalar" else _dev(al, cuda_device))
    assert xp.shape == (b, tx, m, s_, f_) and h_eff.shape == (b, rx, ra, tx, k, s_, rg.num_effective_subcarriers)
    pind, eff = sm.precoding_ind, _eff(rg)
    xr, hr = P.ofdm_precode("rzf", h, pind, eff, x=x, alpha=al)
    x32, h32 = P.ofdm_precode("rzf", h, pind, eff, x=x, alpha=al, dtype=np.complex64)
    _check(f"RZFPrecoder x_precoded {name} {alpha}", xp, x32, xr)
    _check(f"RZFPrecoder h_eff {name} {alpha}", h_eff, h32, hr)
    only_x = RZFPrecoder(rg, sm)(_dev(x, cuda_device), _dev(h, cuda_device), al if alpha == "scalar" else _dev(al, cuda_device))
    assert torch.equal(only_x, xp)


def test_effective_channel_is_what_the_receiver_sees(cuda_device):
    """Without noise, ApplyOFDMChannel(x_precoded, h) on the effective subcarriers equals sum_k h_eff[..., k, :] x_k."""
    from sionna_b200.phy.ofdm import RZFPrecoder
    from sionna_b200.phy.channel import ApplyOFDMChannel
    rg, sm, assoc, ra, m, b = _case("multi_user")
    rng = np.random.default_rng(3)
    rx, tx, k, s_, f_ = assoc.shape[0], assoc.shape[1], sm.num_streams_per_tx, rg.num_ofdm_symbols, rg.fft_size
    h = _dev(cnormal(rng, (b, rx, ra, tx, m, s_, f_)), cuda_device)
    x = _dev(cnormal(rng, (b, tx, k, s_, f_)), cuda_device)
    xp, h_eff = RZFPrecoder(rg, sm, return_effective_channel=True)(x, h, 0.05)
    eff = torch.as_tensor(_eff(rg), device=cuda_device)
    y = ApplyOFDMChannel()(xp, h)[..., eff]
    y2 = torch.einsum("bratksf,btksf->brasf", h_eff, x[..., eff])
    assert float((y - y2).abs().max()) < 1e-4 * float(y.abs().pow(2).mean().sqrt())
    # each receiver sees its own streams (zero forcing up to alpha) and, through h_eff, the other transmitter's
    for i in range(rx):
        j = int(np.where(assoc[i])[0][0])
        own = h_eff[:, i, :, j, i % 2 * ra:(i % 2 + 1) * ra]
        assert float(torch.diagonal(own, dim1=1, dim2=2).abs().mean()) > 0.1
    assert float(h_eff[:, 2:, :, 0].abs().mean()) > 0.1


def test_rzf_precoded_channel_against_alternative_implementation(cuda_device):
    """Port of the reference's test_precoded_channel.py: random tx_power and alpha [B, num_tx, 1, 1], the literal
    per-(receiver, transmitter) loop, here evaluated by the float64 oracle, and the fp32 envelope."""
    from sionna_b200.phy.ofdm import ResourceGrid, RZFPrecodedChannel
    from sionna_b200.phy.mimo import StreamManagement
    rpt, spr, tx = 2, 2, 2
    ra, rx, k = spr, rpt * tx, rpt * spr
    assoc = np.zeros((rx, tx), np.int32)
    for j in range(tx):
        assoc[j * rpt:(j + 1) * rpt, j] = 1
    sm = StreamManagement(assoc, k)
    rg = ResourceGrid(14, 64, 15e3, num_tx=tx, num_streams_per_tx=k)
    b, m = 32, 2 * k
    rng = np.random.default_rng(9)
    h = cnormal(rng, (b, rx, ra, tx, m, 14, 64))
    pw = rng.uniform(size=(b, tx, k, 14, 64)).astype(np.float32)
    al = rng.uniform(size=(b, tx, 1, 1)).astype(np.float32)
    h_eff = RZFPrecodedChannel(rg, sm)(_dev(h, cuda_device), tx_power=_dev(pw, cuda_device), alpha=_dev(al, cuda_device))
    eff = _eff(rg)
    q = h_eff.cpu().numpy()
    for j in range(tx):
        rx_ind = np.where(assoc[:, j])[0]
        h_des = np.transpose(h[:, rx_ind][:, :, :, j].reshape(b, -1, m, 14, 64), (0, 3, 4, 1, 2))
        g = P.rzf_precoding_matrix(h_des.astype(np.complex128), al[:, j])
        g = np.sqrt(np.transpose(pw[:, j], (0, 2, 3, 1)))[..., None, :] * g
        for i in range(rx):
            h_ij = np.transpose(h[:, i, :, j], (0, 3, 4, 1, 2))
            assert np.allclose(np.transpose(q[:, i, :, j], (0, 3, 4, 1, 2)), h_ij @ g, atol=1e-5)
    ref = P.ofdm_precode("rzf", h, sm.precoding_ind, eff, alpha=al, alpha_left=True, tx_power=pw)[1]
    f32 = P.ofdm_precode("rzf", h, sm.precoding_ind, eff, alpha=al, alpha_left=True, tx_power=pw,
                         dtype=np.complex64)[1]
    _check("RZFPrecodedChannel", h_eff, f32, ref)
    h_hat = h + 0.1 * cnormal(rng, h.shape)                                # precoder from an imperfect estimate
    got = RZFPrecodedChannel(rg, sm)(_dev(h, cuda_device), _dev(pw[:, :, :, :1, :1], cuda_device),
                                     h_hat=_dev(h_hat, cuda_device), alpha=0.3)
    ref = P.ofdm_precode("rzf", h, sm.precoding_ind, eff, h_hat=h_hat, alpha=0.3, alpha_left=True, tx_power=pw[:, :, :, :1, :1])[1]
    f32 = P.ofdm_precode("rzf", h, sm.precoding_ind, eff, h_hat=h_hat, alpha=0.3, alpha_left=True,
                         tx_power=pw[:, :, :, :1, :1], dtype=np.complex64)[1]
    _check("RZFPrecodedChannel h_hat", got, f32, ref)


@pytest.mark.parametrize("kind", ["cbf", "eye"])
def test_cbf_and_eye_precoded_channels(cuda_device, kind):
    from sionna_b200.phy.ofdm import CBFPrecodedChannel, EyePrecodedChannel
    rg, sm, assoc, ra, m, b = _case("multi_user")
    rng = np.random.default_rng(11)
    rx, tx, s_, f_ = assoc.shape[0], assoc.shape[1], rg.num_ofdm_symbols, rg.fft_size
    k = sm.num_streams_per_tx if kind == "cbf" else m
    h = cnormal(rng, (b, rx, ra, tx, m, s_, f_))
    pw = rng.uniform(0.5, 2.0, (b, tx, k)).astype(np.float32)            # the first three dimensions
    if kind == "cbf":
        got = CBFPrecodedChannel(rg, sm)(_dev(h, cuda_device), _dev(pw, cuda_device))
    else:
        got = EyePrecodedChannel(rg, sm)(_dev(h, cuda_device), _dev(pw, cuda_device))
    assert got.shape == (b, rx, ra, tx, k, s_, rg.num_effective_subcarriers)
    eff = _eff(rg)
    ref = P.ofdm_precode(kind, h, sm.precoding_ind, eff, tx_power=pw)[1]
    f32 = P.ofdm_precode(kind, h, sm.precoding_ind, eff, tx_power=pw, dtype=np.complex64)[1]
    _check(f"{kind} precoded channel", got, f32, ref)


def test_stream_mismatch_and_double(cuda_device):
    from sionna_b200.phy.ofdm import ResourceGrid, RZFPrecoder, RZFPrecodedChannel
    from sionna_b200.phy.mimo import StreamManagement
    from sionna_b200.phy import block
    rg = ResourceGrid(2, 16, 15e3, num_tx=1, num_streams_per_tx=4)
    sm = StreamManagement(np.ones((1, 1), np.int32), 4)
    rng = np.random.default_rng(12)
    h = _dev(cnormal(rng, (2, 1, 2, 1, 8, 2, 16)), cuda_device)             # 1 receiver x 2 antennas != 4 streams
    x = _dev(cnormal(rng, (2, 1, 4, 2, 16)), cuda_device)
    msg = "The required number of streams per transmitter does not match the channel dimensions"
    with pytest.raises(ValueError, match=msg):
        RZFPrecoder(rg, sm)(x, h)
    with pytest.raises(ValueError, match=msg):
        RZFPrecodedChannel(rg, sm)(h, 1.0)
    h4 = _dev(cnormal(rng, (2, 1, 4, 1, 8, 2, 16)), cuda_device)
    block._warned_double.discard("RZFPrecoder")
    with pytest.warns(block.PrecisionWarning):
        xp, h_eff = RZFPrecoder(rg, sm, return_effective_channel=True, precision="double")(x, h4)
    assert xp.dtype == torch.complex128 and h_eff.dtype == torch.complex128
    xs, hs = RZFPrecoder(rg, sm, return_effective_channel=True)(x, h4)
    assert torch.equal(xp.to(torch.complex64), xs) and torch.equal(h_eff.to(torch.complex64), hs)


# ---- downlink links --------------------------------------------------------------------------------------------------
def _arrays():
    from sionna_b200.phy.channel import AntennaArray
    return AntennaArray(1, 2, "dual", "cross", "38.901", FC), AntennaArray(1, 4, "dual", "cross", "38.901", FC)


class _DownlinkFreq:
    """Downlink of the MIMO OFDM CDL tutorial: 8-antenna BS (1 x 4 dual cross 38.901) to a 4-antenna UT, CDL-B 300 ns,
    2.6 GHz, 10 m/s, 14 x 76 grid, QPSK, rate 1/2 LDPC, ZF precoding, perfect CSI h_hat = h_eff, LMMSE."""

    def __init__(self):
        from sionna_b200.phy.ofdm import ResourceGrid, ResourceGridMapper, LinearDetector, RZFPrecoder
        from sionna_b200.phy.mimo import StreamManagement
        from sionna_b200.phy.mapping import Mapper, BinarySource
        from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
        from sionna_b200.phy.channel import CDL, ApplyOFDMChannel, subcarrier_frequencies
        self.rg = ResourceGrid(14, 76, 15e3, num_tx=1, num_streams_per_tx=4, cyclic_prefix_length=6,
                               num_guard_carriers=(5, 6), dc_null=True, pilot_pattern="kronecker",
                               pilot_ofdm_symbol_indices=[2, 11])
        self.sm = StreamManagement(np.array([[1]]), 4)
        self.n = int(self.rg.num_data_symbols * 2)
        self.k = self.n // 2
        ut, bs = _arrays()
        self.cdl = CDL("B", 300e-9, FC, ut, bs, "downlink", min_speed=10.0)
        self.freqs = subcarrier_frequencies(76, 15e3)
        self.chan = ApplyOFDMChannel()
        self.src, self.enc, self.mapper = BinarySource(), LDPC5GEncoder(self.k, self.n), Mapper("qam", 2)
        self.rgm = ResourceGridMapper(self.rg)
        self.prec = RZFPrecoder(self.rg, self.sm, return_effective_channel=True)
        self.det = LinearDetector("lmmse", "bit", "app", self.rg, self.sm, "qam", 2)
        self.dec = LDPC5GDecoder(self.enc, hard_out=True, num_iter=20)

    def __call__(self, batch_size, ebno_db):
        from sionna_b200.phy.utils import ebnodb2no
        from sionna_b200.phy.channel import cir_to_ofdm_channel
        no = ebnodb2no(ebno_db, 2, 0.5, self.rg)
        b = self.src([batch_size, 1, 4, self.k])
        a, tau = self.cdl(batch_size, 14, 1 / self.rg.ofdm_symbol_duration)
        h = cir_to_ofdm_channel(self.freqs, a, tau, normalize=True)
        x, h_eff = self.prec(self.rgm(self.mapper(self.enc(b))), h)
        y = self.chan(x, h, no)
        return b, self.dec(self.det(y, h_eff, 0.0, no))


def test_downlink_cdl_b_frequency_domain_perfect_csi(cuda_device):
    from sionna_b200.phy import config
    config.seed = 31
    link = _DownlinkFreq()
    ber = []
    for ebno in (-10.0, 0.0, 10.0):
        b, b_hat = link(256, ebno)
        ber.append(float((b != b_hat).float().mean()))
    print("downlink CDL-B BER at -10 / 0 / 10 dB:", ber)
    assert np.all(np.isfinite(ber)) and ber[0] > 1e-2 and ber[0] > ber[1] >= ber[2] and ber[2] < 1e-3, ber


class _DownlinkTime:
    """The reference's test/integration/test_mimo_ofdm_cdl.py Model with domain "time", direction "downlink": CDL-A
    100 ns, 3 m/s, 14 x 72 grid, cyclic prefix 6, pilots on symbols 2 and 11, LS "nn" estimation, LMMSE, app
    demapping. The precoder sees the channel sampled at the OFDM symbol rate."""

    def __init__(self):
        from sionna_b200.phy.ofdm import (ResourceGrid, ResourceGridMapper, RZFPrecoder, LSChannelEstimator,
                                          LMMSEEqualizer, OFDMModulator, OFDMDemodulator)
        from sionna_b200.phy.mimo import StreamManagement
        from sionna_b200.phy.mapping import Mapper, Demapper, BinarySource
        from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
        from sionna_b200.phy.channel import CDL, ApplyTimeChannel, subcarrier_frequencies, time_lag_discrete_time_channel
        self.rg = ResourceGrid(14, 72, 15e3, num_tx=1, num_streams_per_tx=4, cyclic_prefix_length=6,
                               num_guard_carriers=(5, 6), dc_null=True, pilot_pattern="kronecker",
                               pilot_ofdm_symbol_indices=[2, 11])
        self.sm = StreamManagement(np.array([[1]]), 4)
        self.n = int(self.rg.num_data_symbols * 2)
        self.k = int(self.n * 0.5)
        ut, bs = _arrays()
        self.cdl = CDL("A", 100e-9, FC, ut, bs, "downlink", min_speed=3.0)
        self.freqs = subcarrier_frequencies(72, 15e3)
        self.l_min, self.l_max = time_lag_discrete_time_channel(self.rg.bandwidth)
        self.l_tot = self.l_max - self.l_min + 1
        self.chan = ApplyTimeChannel(self.rg.num_time_samples, self.l_tot)
        self.mod, self.demod = OFDMModulator(6), OFDMDemodulator(72, self.l_min, 6)
        self.src, self.enc, self.mapper = BinarySource(), LDPC5GEncoder(self.k, self.n), Mapper("qam", 2)
        self.rgm = ResourceGridMapper(self.rg)
        self.prec = RZFPrecoder(self.rg, self.sm, return_effective_channel=True)
        self.est, self.eq = LSChannelEstimator(self.rg, "nn"), LMMSEEqualizer(self.rg, self.sm)
        self.demapper = Demapper("app", "qam", 2)
        self.dec = LDPC5GDecoder(self.enc, hard_out=True)

    def __call__(self, batch_size, ebno_db):
        from sionna_b200.phy.utils import ebnodb2no
        from sionna_b200.phy.channel import cir_to_ofdm_channel, cir_to_time_channel
        no = ebnodb2no(ebno_db, 2, 0.5, self.rg)
        b = self.src([batch_size, 1, 4, self.k])
        x_rg = self.rgm(self.mapper(self.enc(b)))
        bw, cp, fft = self.rg.bandwidth, 6, 72
        a, tau = self.cdl(batch_size, self.rg.num_time_samples + self.l_tot - 1, bw)
        h_time = cir_to_time_channel(bw, a, tau, self.l_min, self.l_max, normalize=True)
        a_freq = a[..., cp:-1:(fft + cp)][..., :self.rg.num_ofdm_symbols]
        h_freq = cir_to_ofdm_channel(self.freqs, a_freq, tau, normalize=True)
        x_rg, _ = self.prec(x_rg, h_freq)
        y = self.demod(self.chan(self.mod(x_rg), h_time, no))
        h_hat, err_var = self.est(y, no)
        x_hat, no_eff = self.eq(y, h_hat, err_var, no)
        return b, self.dec(self.demapper(x_hat, no_eff))


def test_downlink_time_domain_cdl_a_ls_estimation(cuda_device):
    """The reference's test_dl_time, ported: sim_ber at 0, 10, 20 dB, batch 64, max_mc_iter 10."""
    from sionna_b200.phy.utils import sim_ber
    from sionna_b200.phy import config
    config.seed = 32
    ber, bler = sim_ber(_DownlinkTime(), [0.0, 10.0, 20.0], batch_size=64, max_mc_iter=10, verbose=False)
    ber, bler = np.asarray(ber.cpu()), np.asarray(bler.cpu())
    print("downlink time-domain CDL-A BER / BLER at 0 / 10 / 20 dB:", ber, bler)
    assert np.all(np.isfinite(ber)) and np.all(np.isfinite(bler))
    assert ber[2] < ber[0]
