"""CDL channel model on the device (sb_cdl_coefficients): parity with the NumPy oracle on identical draws, and the
statistics TR 38.901 prescribes, each checked against values computed from the cluster tables alone: power delay
profile and K-factor, cross-polarization ratio, spatial covariance of a uniform linear array, Doppler autocorrelation.
Then links: OFDM + LMMSE + LDPC with perfect CSI, time/frequency equivalence, EP detection."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

FC = 2.6e9
LAM = 299792458.0 / FC
OFFSETS = np.array([0.0447, -0.0447, 0.1413, -0.1413, 0.2492, -0.2492, 0.3715, -0.3715, 0.5129, -0.5129,
                    0.6797, -0.6797, 0.8844, -0.8844, 1.1481, -1.1481, 1.5195, -1.5195, 2.1551, -2.1551])


def _arrays(kind):
    from sionna_b200.phy.channel import AntennaArray
    if kind == "omni_v":
        return (AntennaArray(1, 2, "single", "V", "omni", FC), AntennaArray(2, 2, "single", "V", "omni", FC))
    return (AntennaArray(1, 2, "dual", "cross", "38.901", FC), AntennaArray(1, 4, "dual", "cross", "38.901", FC))


def _np(draws):
    return [d.cpu().numpy() for d in draws]


@pytest.mark.parametrize("speed", [0.0, 30.0])
@pytest.mark.parametrize("arrays", ["omni_v", "cross_38901"])
@pytest.mark.parametrize("direction", ["uplink", "downlink"])
@pytest.mark.parametrize("model", ["A", "B", "C", "D", "E"])
def test_coefficients_equal_oracle_on_identical_draws(cuda_device, model, direction, arrays, speed):
    """The kernel's error against the float64 oracle is at most 2x (rms) / 4x (max) the float32 oracle's."""
    from sionna_b200.phy.channel import CDL
    from sionna_b200.phy import config
    from oracle import cdl as OC
    config.seed = 11
    ut, bs = _arrays(arrays)
    kw = {}
    if arrays == "cross_38901" and speed > 0:
        kw = dict(ut_orientation=[0.4, -0.3, 0.2], bs_orientation=[-0.7, 0.15, 0.1])
    cdl = CDL(model, 300e-9, FC, ut, bs, direction, min_speed=speed, max_speed=speed * 1.2 if speed else None, **kw)
    t_steps, fs = 21, 14e3                                                  # two time tiles, the second partial
    draws = cdl.draws(3)
    a = cdl.synthesize(draws, t_steps, fs).cpu().numpy().astype(np.complex128)
    d = _np(draws)
    ref = OC.cdl_coefficients(cdl, *d, t_steps, fs)
    r32 = OC.cdl_coefficients(cdl, *d, t_steps, fs, dtype=np.float32).astype(np.complex128)
    nr, nt = cdl.rx_array.num_ant, cdl.tx_array.num_ant
    assert a.shape == ref.shape == (3, nr, nt, cdl.num_clusters, t_steps)
    e_k, e_32 = np.abs(a - ref), np.abs(r32 - ref)
    rms = lambda e: float(np.sqrt(np.mean(e ** 2)))
    assert rms(e_k) <= 2 * rms(e_32), (rms(e_k), rms(e_32))
    assert e_k.max() <= 4 * e_32.max(), (e_k.max(), e_32.max())
    if speed == 0.0:
        assert np.allclose(a, a[..., :1], atol=1e-6)


def _single(model, direction="downlink", polarization=("single", "V"), **kw):
    from sionna_b200.phy.channel import CDL, Antenna
    ant = Antenna(*polarization, "omni", FC)
    return CDL(model, 100e-9, FC, ant, ant, direction, **kw)


@pytest.mark.parametrize("model", ["A", "B", "C", "D", "E"])
def test_power_delay_profile_and_k_factor(cuda_device, model):
    from sionna_b200.phy import config
    config.seed = 5
    cdl = _single(model, min_speed=3.0)
    a, tau = cdl(4096, 2, 14e3)
    assert list(a.shape) == [4096, 1, 1, 1, 1, cdl.num_clusters, 2] and a.dtype == torch.complex64
    assert list(tau.shape) == [4096, 1, 1, cdl.num_clusters] and tau.stride(0) == 0
    order = np.argsort(cdl.delays.numpy(), kind="stable")
    assert np.allclose(tau[0, 0, 0].cpu().numpy(), cdl.delays.numpy()[order])
    pw = (a.abs() ** 2).mean(dim=(0, 1, 2, 3, 4, 6)).cpu().numpy()
    expect = cdl.powers.numpy()[order]
    assert np.allclose(pw, expect, rtol=0.08), (pw, expect)
    assert abs(pw.sum() - 1.0) < 0.03
    if cdl.los:
        k, p0 = cdl.k_factor * float(cdl._nlos_powers[0]), float(cdl._nlos_powers[0])
        assert np.isclose(expect[0], (k + p0) / (k + 1), rtol=1e-5)
        assert abs(pw[0] / ((k + p0) / (k + 1)) - 1) < 0.08
    cdl.delay_spread = 300e-9                                              # the tau row is rebuilt
    _, tau3 = cdl(2, 1, 14e3)
    assert np.allclose(tau3[1, 0, 0].cpu().numpy(), 3 * tau[0, 0, 0].cpu().numpy(), rtol=1e-6)


@pytest.mark.parametrize("model", ["A", "C", "D", "E"])
def test_cross_polarization_ratio(cuda_device, model):
    """VH omni arrays at both ends: per cluster, power(H <- V) / power(V <- V) = 1 / XPR; the specular part of the LoS
    models' zero-delay cluster has no cross-polar component."""
    from sionna_b200.phy import config
    config.seed = 6
    cdl = _single(model, polarization=("dual", "VH"))
    a, _ = cdl(4096, 1, 14e3)
    p = (a[:, 0, :, 0, :, :, 0].abs() ** 2).mean(0).cpu().numpy()         # [rx ant, tx ant, cluster]
    ratio = p[1, 0] / p[0, 0]
    inv_xpr = 1.0 / cdl._xpr
    first = 1 if cdl.los else 0
    assert np.allclose(ratio[first:], inv_xpr, rtol=0.1), ratio
    assert np.allclose(p[0, 1, first:] / p[1, 1, first:], inv_xpr, rtol=0.1)
    if cdl.los:
        k, p0 = cdl._k, float(cdl._nlos_powers[0])
        assert abs(ratio[0] / (inv_xpr * p0 / (k + p0)) - 1) < 0.1


def _table_rays(model, zen_key, azi_key, zs_key, as_key):
    from sionna_b200.phy.channel.cdl import cdl_table
    d = cdl_table(model)
    los = int(d["los"])
    zen = d[zen_key][los:][:, None] + float(d[zs_key]) * OFFSETS
    azi = d[azi_key][los:][:, None] + float(d[as_key]) * OFFSETS
    delays = d["delays"][los:]
    return np.deg2rad(zen), np.deg2rad(azi), np.argsort(delays, kind="stable")


@pytest.mark.parametrize("model", ["B", "C"])
def test_spatial_covariance_closed_form(cuda_device, model):
    """Uplink to a 4-element V-pol omni BS row from one UT antenna: E[a_u conj(a_v)] = (P_c / 400) sum_i sum_j
    exp(j 2 pi / lambda r(zoa_j, aoa_i) . (d_u - d_v)), arrival angles = the table's ZoD / AoD rays."""
    from sionna_b200.phy.channel import CDL, Antenna, AntennaArray
    from sionna_b200.phy import config
    config.seed = 8
    bs = AntennaArray(1, 4, "single", "V", "omni", FC)
    cdl = CDL(model, 100e-9, FC, Antenna("single", "V", "omni", FC), bs, "uplink")
    a, _ = cdl(4096, 1, 14e3)
    x = a[:, 0, :, 0, 0, :, 0]                                             # [B, 4, C]
    est = torch.einsum("buc,bvc->cuv", x, x.conj()).cpu().numpy() / x.shape[0]
    zen, azi, order = _table_rays(model, "zod", "aod", "cZSD", "cASD")
    r = np.stack([np.sin(zen)[:, :, None] * np.cos(azi)[:, None, :], np.sin(zen)[:, :, None] * np.sin(azi)[:, None, :],
                  np.broadcast_to(np.cos(zen)[:, :, None], (zen.shape[0], 20, 20))], -1)     # [C, j, i, 3]
    d = bs.ant_pos
    diff = d[:, None, :] - d[None, :, :]                                   # [u, v, 3]
    ph = np.exp(1j * 2 * np.pi / LAM * np.einsum("cjik,uvk->cjiuv", r, diff)).mean(axis=(1, 2))
    p = cdl.powers.numpy()
    expect = (p[:, None, None] * ph)[order]
    for c in range(cdl.num_clusters):
        pc = p[order][c]
        assert np.abs(est[c] - expect[c]).max() < 0.08 * pc, (c, est[c], expect[c])


def test_doppler_constant_at_rest_and_autocorrelation(cuda_device):
    """Zero speed: constant over time. 30 m/s: the autocorrelation summed over clusters equals
    sum_c (P_c / 400) sum_ij E_v[exp(j k r_ij . v tau)] with v = 30 m/s in a direction of azimuth U[0, 2 pi) and zenith
    U[0, pi) (quadrature in float64)."""
    from sionna_b200.phy import config
    config.seed = 12
    rest = _single("B")
    a0, _ = rest(64, 8, 14e3)
    assert torch.allclose(a0, a0[..., :1].expand_as(a0), atol=1e-6)
    cdl = _single("A", min_speed=30.0)
    fs, t_steps = 4e3, 17
    a, _ = cdl(4096, t_steps, fs)
    x = a[:, 0, 0, 0, 0].cpu().numpy().astype(np.complex128)                # [B, C, T]
    lags = np.array([1, 2, 4, 8])
    est = np.array([(x[..., lag:] * x[..., :-lag].conj()).mean(axis=(0, 2)).sum() for lag in lags])
    zen, azi, _ = _table_rays("A", "zoa", "aoa", "cZSA", "cASA")
    r = np.stack([np.sin(zen)[:, :, None] * np.cos(azi)[:, None, :], np.sin(zen)[:, :, None] * np.sin(azi)[:, None, :],
                  np.broadcast_to(np.cos(zen)[:, :, None], (zen.shape[0], 20, 20))], -1).reshape(zen.shape[0], 400, 3)
    n = 256
    vphi = (np.arange(n) + 0.5) * 2 * np.pi / n
    vth = (np.arange(n) + 0.5) * np.pi / n
    v = np.stack([np.cos(vphi)[:, None] * np.sin(vth)[None], np.sin(vphi)[:, None] * np.sin(vth)[None],
                  np.broadcast_to(np.cos(vth)[None], (n, n))], -1).reshape(-1, 3)            # uniform in (phi, theta)
    k = 2 * np.pi / LAM * 30.0
    p = cdl.powers.numpy()
    proj = np.einsum("cjk,vk->cjv", r, v)                                  # [C, 400, n*n]
    expect = np.array([(p[:, None, None] * np.exp(1j * k * proj * lag / fs)).mean(axis=(1, 2)).sum() for lag in lags])
    assert np.allclose(est, expect, atol=0.03), (est, expect)
    assert abs(est[-1]) < 0.9                                               # the lags span real decorrelation


class _Link:
    """Uplink of the reference's MIMO OFDM CDL tutorial: 4-antenna UT (1 x 2 dual cross 38.901) to an 8-antenna BS
    (1 x 4), CDL-B 300 ns, 2.6 GHz, 10 m/s, 14 x 76 grid at 15 kHz, QPSK, rate 1/2 LDPC, perfect CSI."""

    def __init__(self, detector="lmmse"):
        from sionna_b200.phy.ofdm import ResourceGrid, ResourceGridMapper, RemoveNulledSubcarriers, LinearDetector, EPDetector
        from sionna_b200.phy.mimo import StreamManagement
        from sionna_b200.phy.mapping import Mapper, BinarySource
        from sionna_b200.phy.fec.ldpc import LDPC5GEncoder, LDPC5GDecoder
        from sionna_b200.phy.channel import CDL, OFDMChannel, AntennaArray
        self.rg = ResourceGrid(14, 76, 15e3, num_tx=1, num_streams_per_tx=4, cyclic_prefix_length=6,
                               num_guard_carriers=(5, 6), dc_null=True, pilot_pattern="kronecker",
                               pilot_ofdm_symbol_indices=[2, 11])
        self.sm = StreamManagement(np.array([[1]]), 4)
        self.n = int(self.rg.num_data_symbols * 2)
        self.k = self.n // 2
        ut = AntennaArray(1, 2, "dual", "cross", "38.901", FC)
        bs = AntennaArray(1, 4, "dual", "cross", "38.901", FC)
        self.cdl = CDL("B", 300e-9, FC, ut, bs, "uplink", min_speed=10.0)
        self.chan = OFDMChannel(self.cdl, self.rg, normalize_channel=True, return_channel=True)
        self.src, self.enc, self.mapper = BinarySource(), LDPC5GEncoder(self.k, self.n), Mapper("qam", 2)
        self.rgm, self.rm = ResourceGridMapper(self.rg), RemoveNulledSubcarriers(self.rg)
        if detector == "lmmse":
            self.det = LinearDetector("lmmse", "bit", "app", self.rg, self.sm, "qam", 2)
        else:
            self.det = EPDetector("bit", self.rg, self.sm, num_bits_per_symbol=2)
        self.dec = LDPC5GDecoder(self.enc, hard_out=True, num_iter=20)

    def __call__(self, batch_size, ebno_db):
        from sionna_b200.phy.utils import ebnodb2no
        no = ebnodb2no(ebno_db, 2, 0.5, self.rg)
        b = self.src([batch_size, 1, 4, self.k])
        y, h = self.chan(self.rgm(self.mapper(self.enc(b))), no)
        llr = self.det(y, self.rm(h), 0.0, no)
        return b, self.dec(llr)


def test_ofdm_link_lmmse_ldpc_perfect_csi(cuda_device):
    from sionna_b200.phy import config
    config.seed = 21
    link = _Link("lmmse")
    ber = []
    for ebno in (-10.0, 0.0, 10.0):
        b, b_hat = link(256, ebno)
        ber.append(float((b != b_hat).float().mean()))
    assert np.all(np.isfinite(ber)) and ber[0] > 1e-2 and ber[0] > ber[1] >= ber[2] and ber[2] < 1e-3, ber


def test_ofdm_link_ep_detector(cuda_device):
    from sionna_b200.phy import config
    config.seed = 22
    link = _Link("ep")
    b, b_hat = link(128, 10.0)
    assert float((b != b_hat).float().mean()) < 1e-3
    b, b_hat = link(128, -10.0)
    assert float((b != b_hat).float().mean()) > 1e-2


def test_time_channel_matches_ofdm_channel_at_rest(cuda_device):
    """Zero speed: TimeChannel(CDL) + OFDMDemodulator reproduces OFDMChannel(CDL) on the same draws (up to the sinc
    truncation at l_min = -6)."""
    from sionna_b200.phy.channel import CDL, TimeChannel, OFDMChannel, AntennaArray, time_lag_discrete_time_channel
    from sionna_b200.phy.ofdm import OFDMModulator, OFDMDemodulator, ResourceGrid
    from sionna_b200.phy.utils import complex_normal
    from sionna_b200.phy import config
    fft, cp, nsym, scs = 64, 16, 4, 30e3
    bw = fft * scs
    ut = AntennaArray(1, 1, "dual", "cross", "38.901", FC)
    bs = AntennaArray(1, 2, "dual", "cross", "38.901", FC)
    cdl = CDL("C", 100e-9, FC, ut, bs, "uplink")
    l_min, l_max = time_lag_discrete_time_channel(bw)
    n_time = nsym * (fft + cp)
    config.seed = 9
    x = complex_normal([6, 1, 2, nsym, fft])
    rg = ResourceGrid(nsym, fft, scs, num_tx=1, num_streams_per_tx=2, cyclic_prefix_length=cp)
    config.seed = 10
    yf = OFDMChannel(cdl, rg)(x)
    config.seed = 10
    yt = TimeChannel(cdl, bw, n_time, l_min=l_min, l_max=l_max)(OFDMModulator(cp)(x))
    y = OFDMDemodulator(fft, l_min, cp)(yt)
    assert list(y.shape) == list(yf.shape) == [6, 1, 4, nsym, fft]
    err = float(((y - yf).abs() ** 2).mean() / (yf.abs() ** 2).mean())
    assert err < 1e-2
