"""TDL channel models (sum-of-sinusoids time evolution) and CIR -> OFDM channel conversion: on-device channel generation
of SURVEY.md section 8(f3); mirror of /root/reference/src/sionna/phy/channel/tr38901/tdl.py:20-590 and of
channel/utils.py:180-253, 1010-1060. Power delay profiles: TR 38.901 Tables 7.7.2-1..5 and TS 38.104 Annex G
(``tdl_models.npz``, tools/make_code_tables.py). Random draws (``sb_uniform``), tap synthesis (``sb_tdl_sos``) and the
frequency response (``sb_phase_table``, ``sb_cir_gram``, ``sb_cir_link_scale``, ``sb_cir_apply``) are hand-written kernels."""
import os
import numpy as np
import torch

from ..block import Block
from ..config import config
from .._lib_helpers import philox_fill
from ..._lib import lib, check, ptr, current_stream

_MODELS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tdl_models.npz")


def subcarrier_frequencies(num_subcarriers, subcarrier_spacing, precision=None):
    """Baseband frequencies of the subcarriers, DC in the centre (channel/utils.py:1010-1060)."""
    if num_subcarriers % 2 == 0:
        start, limit = -num_subcarriers / 2, num_subcarriers / 2
    else:
        start, limit = -(num_subcarriers - 1) / 2, (num_subcarriers - 1) / 2 + 1
    return torch.arange(start, limit, dtype=torch.float32) * subcarrier_spacing


def _uniform(shape, lo, hi):
    """config.tf_rng.uniform(shape, lo, hi) on the device (``sb_uniform``, Philox4x32-10)."""
    return philox_fill("sb_uniform", shape, lo, hi, config.device)


class _TableCache:
    """Device copies and phase tables keyed by the identity (+ version counter) of the tensors they were built from;
    entries keep their sources alive, so an address can never be mistaken for a newer tensor."""

    def __init__(self, size=16):
        self._size, self._items = size, {}

    def get(self, key_tensors, extra, build):
        key = tuple((id(t), t._version) for t in key_tensors) + tuple(extra)
        hit = self._items.get(key)
        if hit is None:
            if len(self._items) >= self._size:
                self._items.pop(next(iter(self._items)))
            hit = (build(), key_tensors)
            self._items[key] = hit
        return hit[0]


_cache = _TableCache()


def _f32_on(t, dev):
    """float32 contiguous copy of `t` on `dev` (cached per source tensor)."""
    return _cache.get((t,), ("f32", str(dev)), lambda: t.detach().to(device=dev, dtype=torch.float32).contiguous())


def _shared_delays(tau):
    """True if every link uses the same delays, decided from the tensor's layout only (no device read-back): all
    leading dimensions are broadcast (stride 0, as `TDL` returns them) or have size 1."""
    return all(tau.shape[d] == 1 or tau.stride(d) == 0 for d in range(tau.dim() - 1))


def _cir_convert(a, tau, x, mode, scale, normalize, denom):
    """Common body of cir_to_ofdm_channel / cir_to_time_channel: h[..., t, j] = c_link * sum_p a[..., p, t] e[p, j] with
    e from ``sb_phase_table`` (mode 0: exp(-j 2 pi x_j tau_p); mode 1: sinc(x_j - tau_p * scale)), the per-link
    normalisation from ``sb_cir_gram`` + ``sb_cir_link_scale`` and the contraction by ``sb_cir_apply``."""
    if a.dtype == torch.complex128:                          # double precision: single-precision kernels, widened result
        from ..block import fallback_to_single
        fallback_to_single("cir_to_ofdm_channel / cir_to_time_channel", "double")
        return _cir_convert(a.to(torch.complex64), tau, x, mode, scale, normalize, denom).to(torch.complex128)
    if a.dtype != torch.complex64:
        raise TypeError("a must be a complex tensor")
    if a.dim() != 7:
        raise ValueError("a must have shape [batch, num_rx, num_rx_ant, num_tx, num_tx_ant, num_paths, num_time_steps]")
    dev = a.device
    b, rx, ra, tx, ta, p, t = a.shape
    n_col = x.shape[0]
    xd = _f32_on(x, dev)
    shared = _shared_delays(tau)
    if tau.dim() == 6 and not shared:
        raise NotImplementedError("per-antenna path delays are not provided (TDL delays are per link)")

    def build_tables(tau_rows, n_tab):
        e = torch.empty((n_tab, p, n_col), dtype=torch.complex64, device=dev)
        check(lib().sb_phase_table(ptr(tau_rows), ptr(xd), float(scale), mode, ptr(e), n_tab, p, n_col, current_stream()),
              "sb_phase_table")
        g = None
        if normalize:
            g = torch.empty((n_tab, p, p), dtype=torch.complex128, device=dev)
            check(lib().sb_cir_gram(ptr(e), ptr(g), n_tab, p, n_col, current_stream()), "sb_cir_gram")
        return e, g

    if shared:
        base = tau._base if tau._base is not None else tau

        def build_shared():
            t0 = tau.reshape(-1, tau.shape[-1])[:1].to(device=dev, dtype=torch.float32).contiguous()
            return build_tables(t0, 1)
        e, g = _cache.get((base, x), (mode, float(scale), bool(normalize), str(dev), p), build_shared)
        stride_e = stride_g = 0
    else:
        if tuple(tau.shape) != (b, rx, tx, p):
            raise ValueError("tau must have shape [batch, num_rx, num_tx, num_paths]")
        e, g = build_tables(tau.to(device=dev, dtype=torch.float32).contiguous(), b * rx * tx)
        stride_e, stride_g = p * n_col, p * p
    ac = a.contiguous()
    sc = None
    if normalize:
        sc = torch.empty(b * rx * tx, dtype=torch.float32, device=dev)
        check(lib().sb_cir_link_scale(ptr(ac), ptr(g), stride_g, ptr(sc), b, rx, ra, tx, ta, p, t, float(denom),
                                      current_stream()), "sb_cir_link_scale")
    h = torch.empty((b, rx, ra, tx, ta, t, n_col), dtype=torch.complex64, device=dev)
    check(lib().sb_cir_apply(ptr(ac), ptr(e), stride_e, ptr(sc), ptr(h), b, rx, ra, tx, ta, p, t, n_col,
                             current_stream()), "sb_cir_apply")
    return h


def cir_to_ofdm_channel(frequencies, a, tau, normalize=False):
    """h_f[b, rx, rx_ant, tx, tx_ant, t, f] = sum_p a[..., p, t] exp(-j 2 pi f tau_p) (channel/utils.py:180-253);
    ``normalize``: unit average energy per resource element and link (:246-251).

    Three hand-written kernels and no tensor expression: the phase table (built once and cached when all links share
    their delays, which is decided from the layout of ``tau`` without reading it back; one table per link otherwise),
    the per-link normalisation factor from the taps and the table's Gram matrix, and the contraction that writes the
    scaled ``h`` once (csrc/channel.cu)."""
    return _cir_convert(a, tau, frequencies, 0, 0.0, normalize, float(frequencies.shape[0]))


class TDL(Block):
    """TDL(model, delay_spread, carrier_frequency, num_sinusoids=20, los_angle_of_arrival=pi/4, min_speed=0., max_speed=None, num_rx_ant=1, num_tx_ant=1, spatial_corr_mat=None, rx_corr_mat=None, tx_corr_mat=None, precision=None)

    Tapped delay line models "A".."E" of TR 38.901 (delays scaled by ``delay_spread`` [s]) and "A30", "B100", "C300" of
    TS 38.104 (fixed delays). Time evolution by the sum-of-sinusoids model of the reference (tdl.py:372-456): a Doppler
    shift per link drawn in [w(min_speed), w(max_speed)], w = 2 pi v f_c / c, ``num_sinusoids`` arrival angles per path
    and a phase per antenna pair, path and sinusoid; LoS models add a specular term on the first path.

    ``call(batch_size, num_time_steps, sampling_frequency)`` -> ``a [batch, 1, num_rx_ant, 1, num_tx_ant, num_paths,
    num_time_steps]`` complex64, ``tau [batch, 1, 1, num_paths]``. All draws and the tap synthesis run on the device
    (``sb_uniform``, ``sb_tdl_sos``)."""

    def __init__(self, model, delay_spread, carrier_frequency, num_sinusoids=20, los_angle_of_arrival=np.pi / 4,
                 min_speed=0., max_speed=None, num_rx_ant=1, num_tx_ant=1, spatial_corr_mat=None, rx_corr_mat=None,
                 tx_corr_mat=None, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert model in ("A", "B", "C", "D", "E", "A30", "B100", "C300"), "Invalid TDL model"
        fixed = {"A30": 30e-9, "B100": 100e-9, "C300": 300e-9}
        if model in fixed and delay_spread != fixed[model]:
            print(f"Warning: Delay spread is set to {fixed[model] * 1e9:.0f}ns with this model")
            delay_spread = fixed[model]
        with np.load(_MODELS) as d:
            delays, p_db, los = d[f"{model}_delays"], d[f"{model}_powers_db"], int(d[f"{model}_los"])
            self._scale_delays = bool(int(d[f"{model}_scale_delays"]))
        p = 10 ** (p_db / 10)
        self._los = bool(los)
        self._los_power = 0.0
        if self._los:                                          # first entry = specular component sharing the first delay
            self._los_power = float(p[0])
            p, delays = p[1:], delays[1:]
        norm = self._los_power + p.sum()                       # total mean power 1 (tdl.py:583-590)
        self._los_power /= norm
        self._powers = (p / norm).astype(np.float32)
        self._delays_norm = delays.astype(np.float64)
        self._delay_spread = float(delay_spread)
        self._num_rx_ant, self._num_tx_ant = int(num_rx_ant), int(num_tx_ant)
        self._carrier_frequency = float(carrier_frequency)
        self._num_sinusoids = int(num_sinusoids)
        self._los_aoa = float(los_angle_of_arrival)
        self._min_speed = float(min_speed)
        self._max_speed = self._min_speed if max_speed is None else float(max_speed)
        assert self._max_speed >= self._min_speed, "min_speed cannot be larger than max_speed"
        # spatial correlation: ONE lower-triangular factor over the rx_ant * tx_ant antenna pairs (rx antenna major);
        # separate rx / tx matrices R, T mean V' = L_r V L_t^H, i.e. vec(V') = kron(L_r, conj(L_t)) vec(V)
        self._corr_l = None
        if spatial_corr_mat is not None:
            m = torch.as_tensor(np.asarray(spatial_corr_mat), dtype=torch.complex64)
            self._corr_l = torch.linalg.cholesky(m)
        elif rx_corr_mat is not None or tx_corr_mat is not None:
            def chol(m, size):
                if m is None:
                    return torch.eye(size, dtype=torch.complex64)
                return torch.linalg.cholesky(torch.as_tensor(np.asarray(m), dtype=torch.complex64))
            self._corr_l = torch.kron(chol(rx_corr_mat, self._num_rx_ant), chol(tx_corr_mat, self._num_tx_ant).conj())
        self._corr_dev = None
        self._dev_tau = None
        self._dev_powers = None

    def _doppler(self, speed):
        """Maximum radian Doppler 2 pi v f_c / c (tdl.py:504-527)."""
        return 2.0 * np.pi * speed / 299792458.0 * self._carrier_frequency

    num_clusters = property(lambda self: len(self._powers))
    los = property(lambda self: self._los)

    @property
    def k_factor(self):
        assert self._los, "This property is only available for LoS models"
        return self._los_power / float(self._powers[0])

    @property
    def delays(self):
        scale = self._delay_spread if self._scale_delays else 1e-9
        return torch.from_numpy((self._delays_norm * scale).astype(np.float32))

    @property
    def mean_powers(self):
        p = self._powers.copy()
        if self._los:
            p[0] += self._los_power
        return torch.from_numpy(p)

    @property
    def mean_power_los(self):
        assert self._los, "This property is only available for LoS models"
        return self._los_power

    @property
    def delay_spread(self):
        return self._delay_spread

    @delay_spread.setter
    def delay_spread(self, value):
        if self._scale_delays:
            self._delay_spread = float(value)
            self._dev_tau = None
        else:
            print("Warning: The delay spread cannot be set with this model")

    def __call__(self, batch_size, num_time_steps=1, sampling_frequency=1.0):
        return self._invoke(batch_size, num_time_steps, sampling_frequency)

    def draws(self, batch_size):
        """The random draws of one call: (doppler [B], theta [B, P, Ns], phi [B, A, P, Ns], phi0 [B] | None)."""
        n, ns, ap = self.num_clusters, self._num_sinusoids, self._num_rx_ant * self._num_tx_ant
        doppler = _uniform([batch_size], self._doppler(self._min_speed), self._doppler(self._max_speed))
        theta = _uniform([batch_size, n, ns], -np.pi / ns, np.pi / ns)
        phi = _uniform([batch_size, ap, n, ns], -np.pi, np.pi)
        phi0 = _uniform([batch_size], -np.pi, np.pi) if self._los else None
        return doppler, theta, phi, phi0

    def synthesize(self, draws, num_time_steps, sampling_frequency):
        """Tap gains [B, num_rx_ant * num_tx_ant, P, T] from `draws` (kernel ``sb_tdl_sos``)."""
        doppler, theta, phi, phi0 = draws
        dev = doppler.device
        b, n, ns = doppler.shape[0], self.num_clusters, self._num_sinusoids
        ap = self._num_rx_ant * self._num_tx_ant
        if self._dev_powers is None or self._dev_powers.device != dev:
            self._dev_powers = torch.from_numpy(self._powers).to(dev)
        a = torch.empty((b, ap, n, int(num_time_steps)), dtype=torch.complex64, device=dev)
        check(lib().sb_tdl_sos(ptr(doppler), ptr(theta), ptr(phi), ptr(phi0), ptr(self._dev_powers), self._los_power,
                               self._los_aoa, ptr(a), b, ap, n, ns, int(num_time_steps), float(sampling_frequency),
                               current_stream()), "sb_tdl_sos")
        return a

    def call(self, batch_size, num_time_steps=1, sampling_frequency=1.0):
        if self.precision != "single":
            raise NotImplementedError("TDL generates complex64 taps only.")
        batch_size = int(batch_size)
        a = self.synthesize(self.draws(batch_size), num_time_steps, sampling_frequency)   # [B, rx_ant * tx_ant, P, T]
        n, t = self.num_clusters, int(num_time_steps)
        dev = a.device
        if self._corr_l is not None:                            # spatial correlation (tdl.py:466-490): v' = L v
            if self._corr_dev is None or self._corr_dev.device != dev:
                self._corr_dev = self._corr_l.to(dev).contiguous()
            out = torch.empty_like(a)
            check(lib().sb_spatial_corr(ptr(a), ptr(self._corr_dev), ptr(out), batch_size,
                                        self._num_rx_ant * self._num_tx_ant, n * t, current_stream()), "sb_spatial_corr")
            a = out
        a = a.reshape(batch_size, 1, self._num_rx_ant, 1, self._num_tx_ant, n, t)
        if self._dev_tau is None or self._dev_tau.device != dev:
            self._dev_tau = self.delays.to(dev).reshape(1, 1, 1, n)
        # every link has the same delays: a broadcast view (stride 0) says so without any device read-back
        return a, self._dev_tau.expand(batch_size, 1, 1, n)
