"""Clustered delay line (CDL) channel models of TR 38.901 section 7.7.1 with antenna arrays, polarization and element
patterns: mirror of /root/reference/src/sionna/phy/channel/tr38901/cdl.py:20-695 and of the CDL path of
channel_coefficients.py:173-1030 (steps 10 and 11 of section 7.5, without sub-clustering). Cluster tables: TR 38.901
Tables 7.7.1-1..5 (``cdl_models.json``, tools/make_code_tables.py).

Random coupling only permutes the 20 ray angles inside a cluster, and arrays and orientations are fixed per instance, so
every arrival (zenith, azimuth) pair a ray can take is one of 20 x 20 per cluster, and so is every departure pair. The
constructor tabulates, in float64 and then cast to float32, per pair: the GCS field vector of each polarization, the
phase of every antenna (7.5-22) and, on the arrival side, the unit vector used by the Doppler term. A call draws
velocities, coupling normals and initial phases (``sb_uniform``, ``sb_normal``) and the kernel ``sb_cdl_coefficients``
ranks the normals, gathers from the tables, evaluates the Doppler phasors and sums the rays (csrc/channel.cu)."""
import json
import os
import numpy as np
import torch

from ..block import Block
from ..config import config
from .._lib_helpers import philox_fill
from ..._lib import lib, check, ptr, current_stream
from .antenna import SPEED_OF_LIGHT

_MODELS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cdl_models.json")
NUM_RAYS = 20
# TR 38.901 Table 7.5-3: ray offset angles within a cluster (unit rms angle spread)
RAY_OFFSETS = np.array([0.0447, -0.0447, 0.1413, -0.1413, 0.2492, -0.2492, 0.3715, -0.3715, 0.5129, -0.5129,
                        0.6797, -0.6797, 0.8844, -0.8844, 1.1481, -1.1481, 1.5195, -1.5195, 2.1551, -2.1551])


def cdl_table(model):
    """TR 38.901 table of CDL ``model`` in table order: ``los``, ``num_clusters``, float64 arrays ``delays``
    (normalised), ``powers_db``, ``aod``/``aoa``/``zod``/``zoa`` [deg] and scalars ``cASD``/``cASA``/``cZSD``/``cZSA``
    [deg], ``xpr_db``."""
    with open(_MODELS) as f:
        t = json.load(f)[model]
    return {k: np.asarray(v, np.float64) if isinstance(v, list) else v for k, v in t.items()}


def rotation_matrix(orientation):
    """Forward composite rotation matrix (7.1-4) for orientation (alpha, beta, gamma) [rad]."""
    a, b, c = (float(v) for v in orientation)
    return np.array([
        [np.cos(a) * np.cos(b), np.cos(a) * np.sin(b) * np.sin(c) - np.sin(a) * np.cos(c),
         np.cos(a) * np.sin(b) * np.cos(c) + np.sin(a) * np.sin(c)],
        [np.sin(a) * np.cos(b), np.sin(a) * np.sin(b) * np.sin(c) + np.cos(a) * np.cos(c),
         np.sin(a) * np.sin(b) * np.cos(c) - np.cos(a) * np.sin(c)],
        [-np.sin(b), np.cos(b) * np.sin(c), np.cos(b) * np.cos(c)]])


def unit_vector(theta, phi):
    """Unit vector (7.1-6) for zenith ``theta`` and azimuth ``phi``: shape ``theta.shape + (3,)``."""
    return np.stack([np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.cos(theta)], axis=-1)


def gcs_field(element, orientation, theta, phi):
    """GCS field (F_theta, F_phi) of ``element`` mounted with ``orientation`` towards GCS direction (theta, phi): the
    pattern is evaluated at the LCS angles (7.1-7/8; z clipped before arccos, azimuth in (-pi, pi]) and rotated by the
    angle psi of (7.1-15)."""
    r = unit_vector(theta, phi) @ rotation_matrix(orientation)          # R^T rho, row-vector form
    theta_p = np.arccos(np.clip(r[..., 2], -1.0, 1.0))
    phi_p = np.angle(r[..., 0] + 1j * r[..., 1])
    f_th, f_ph = element.field(theta_p, phi_p)
    a, b, c = (float(v) for v in orientation)
    re = np.sin(c) * np.cos(theta) * np.sin(phi - a) + np.cos(c) * (np.cos(b) * np.sin(theta) - np.sin(b) * np.cos(theta)
                                                                      * np.cos(phi - a))
    im = np.sin(c) * np.cos(phi - a) + np.sin(b) * np.cos(c) * np.sin(phi - a)
    psi = np.angle(re + 1j * im)
    return np.cos(psi) * f_th - np.sin(psi) * f_ph, np.sin(psi) * f_th + np.cos(psi) * f_ph


def _side_tables(array, orientation, zen, azi, los_zen, los_azi, wavenumber):
    """Tables of one link end over its (cluster, zenith index j, azimuth index i) pairs, row c * 400 + j * 20 + i, plus
    one last row for the LoS direction: unit vectors [N, 3], fields [N, 4] (pol 1 theta, phi, pol 2 theta, phi) and
    antenna phases exp(j k r.d) [N, num_ant] with d the GCS antenna positions."""
    c = zen.shape[0]
    theta = np.concatenate([np.broadcast_to(zen[:, :, None], (c, NUM_RAYS, NUM_RAYS)).reshape(-1), [los_zen]])
    phi = np.concatenate([np.broadcast_to(azi[:, None, :], (c, NUM_RAYS, NUM_RAYS)).reshape(-1), [los_azi]])
    dirs = unit_vector(theta, phi)
    f1 = gcs_field(array.ant_pol1, orientation, theta, phi)
    f2 = gcs_field(array.ant_pol2, orientation, theta, phi) if array.polarization == "dual" else f1
    fields = np.stack([f1[0], f1[1], f2[0], f2[1]], axis=-1)
    d_gcs = array.ant_pos @ rotation_matrix(orientation).T                  # [num_ant, 3]
    phases = np.exp(1j * wavenumber * (dirs @ d_gcs.T))
    return dirs, fields, phases


class CDL(Block):
    """CDL(model, delay_spread, carrier_frequency, ut_array, bs_array, direction, ut_orientation=None, bs_orientation=None, min_speed=0., max_speed=None, precision=None)

    Clustered delay line models "A".."E" of TR 38.901 (delays scaled by ``delay_spread`` [s]) between a user terminal
    and a base station with `PanelArray` antennas. ``direction`` "uplink" (UT transmits) or "downlink"; orientations
    (alpha, beta, gamma) [rad] default to [pi, 0, 0] for the UT and 0 for the BS. The moving end (the UT) draws a speed
    uniformly in [min_speed, max_speed] and a direction with azimuth in [0, 2 pi) and zenith in [0, pi).

    ``__call__(batch_size, num_time_steps, sampling_frequency)`` -> ``a [batch, 1, num_rx_ant, 1, num_tx_ant,
    num_clusters, num_time_steps]`` complex64 and ``tau [batch, 1, 1, num_clusters]`` float32 [s], clusters in
    ascending order of delay. ``tau`` is a broadcast (stride 0) view of one device row, so the CIR -> channel
    conversions build one shared phase table."""

    def __init__(self, model, delay_spread, carrier_frequency, ut_array, bs_array, direction, ut_orientation=None,
                 bs_orientation=None, min_speed=0., max_speed=None, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert direction in ("uplink", "downlink"), "Invalid link direction"
        assert model in ("A", "B", "C", "D", "E"), "Invalid CDL model"
        self._direction = direction
        ut_orientation = np.array([np.pi, 0.0, 0.0]) if ut_orientation is None else np.asarray(ut_orientation, np.float64)
        bs_orientation = np.zeros(3) if bs_orientation is None else np.asarray(bs_orientation, np.float64)
        if direction == "downlink":
            self._tx_array, self._rx_array = bs_array, ut_array
            tx_orientation, rx_orientation = bs_orientation, ut_orientation
        else:
            self._tx_array, self._rx_array = ut_array, bs_array
            tx_orientation, rx_orientation = ut_orientation, bs_orientation
        self._carrier_frequency = float(carrier_frequency)
        self._delay_spread = float(delay_spread)
        self._min_speed = float(min_speed)
        self._max_speed = self._min_speed if max_speed is None else float(max_speed)
        assert self._max_speed >= self._min_speed, "min_speed cannot be larger than max_speed"

        t = cdl_table(model)
        self._los = bool(int(t["los"]))
        self._num_clusters = int(t["num_clusters"])
        powers = 10.0 ** (t["powers_db"] / 10.0)
        powers = powers / powers.sum()
        delays = t["delays"].copy()
        ang = {k: t[k].copy() for k in ("aod", "aoa", "zod", "zoa")}
        if self._los:                          # row 0 is the specular component (cdl.py:452-486)
            los_power = powers[0]
            los_ang = {k: np.deg2rad(v[0]) for k, v in ang.items()}
            powers, delays = powers[1:], delays[1:]
            ang = {k: v[1:] for k, v in ang.items()}
            norm = powers.sum()
            powers = powers / norm
            self._k = float(los_power / norm)   # K = specular power / total NLoS power
        else:
            los_ang = {k: 0.0 for k in ang}
            self._k = 1.0
        assert len(powers) == self._num_clusters
        spread = {"aod": t["cASD"], "aoa": t["cASA"], "zod": t["cZSD"], "zoa": t["cZSA"]}
        rays = {k: np.deg2rad(v[:, None] + float(spread[k]) * RAY_OFFSETS[None, :]) for k, v in ang.items()}
        if direction == "uplink":              # arrival and departure swap (cdl.py:529-548)
            swap = {"aoa": "aod", "zoa": "zod", "aod": "aoa", "zod": "zoa"}
            rays = {k: rays[swap[k]] for k in rays}
            los_ang = {k: los_ang[swap[k]] for k in los_ang}
        self._nlos_powers = powers
        self._delays_norm = delays
        self._xpr = 10.0 ** (float(t["xpr_db"]) / 10.0)
        self._order = np.argsort(delays, kind="stable").astype(np.int32)   # output cluster o <- table cluster order[o]

        self._wavenumber = 2.0 * np.pi * self._carrier_frequency / SPEED_OF_LIGHT
        rx_dir, rx_field, rx_phase = _side_tables(self._rx_array, rx_orientation, rays["zoa"], rays["aoa"],
                                                  los_ang["zoa"], los_ang["aoa"], self._wavenumber)
        _, tx_field, tx_phase = _side_tables(self._tx_array, tx_orientation, rays["zod"], rays["aod"],
                                             los_ang["zod"], los_ang["aod"], self._wavenumber)
        nlos_scale = np.sqrt(1.0 / (self._k + 1.0)) if self._los else 1.0
        cluster_scale = np.sqrt(powers / NUM_RAYS) * nlos_scale
        los_field = None
        if self._los:                          # phase matrix [[1, 0], [0, -1]] (7.5-29), times sqrt(K / (K + 1))
            fr, ft = rx_field[-1], tx_field[-1]
            los_field = np.array([fr[2 * p] * ft[2 * q] - fr[2 * p + 1] * ft[2 * q + 1] for p in (0, 1) for q in (0, 1)])
            los_field = los_field * np.sqrt(self._k / (self._k + 1.0))
        self._host = {
            "rx_dir": rx_dir.astype(np.float32), "rx_field": rx_field.astype(np.float32),
            "rx_phase": rx_phase.astype(np.complex64), "rx_pol": self._rx_array.ant_pol_index.astype(np.int32),
            "tx_field": tx_field.astype(np.float32), "tx_phase": tx_phase.astype(np.complex64),
            "tx_pol": self._tx_array.ant_pol_index.astype(np.int32),
            "cluster_scale": cluster_scale.astype(np.float32), "order": self._order,
            "los_field": None if los_field is None else los_field.astype(np.float32)}
        self._rays = rays                      # radians after the uplink swap, [clusters, 20], table order
        self._los_angles = los_ang
        self._orientations = (tx_orientation, rx_orientation)
        self._dev = None
        self._dev_tau = None

    num_clusters = property(lambda self: self._num_clusters)
    los = property(lambda self: self._los)
    direction = property(lambda self: self._direction)
    tx_array = property(lambda self: self._tx_array)
    rx_array = property(lambda self: self._rx_array)

    @property
    def k_factor(self):
        """K-factor of the zero-delay cluster (specular over NLoS power of that cluster)."""
        assert self._los, "This property is only available for LoS models"
        return self._k / float(self._nlos_powers[0])

    @property
    def delays(self):
        """Cluster delays [s] in table order."""
        return torch.from_numpy((self._delays_norm * self._delay_spread).astype(np.float32))

    @property
    def powers(self):
        """Cluster powers (linear, sum 1) in table order; for LoS models the first one includes the specular part."""
        p = self._nlos_powers.copy()
        if self._los:
            p[0] += self._k
            p = p / (self._k + 1.0)
        return torch.from_numpy(p.astype(np.float32))

    @property
    def delay_spread(self):
        return self._delay_spread

    @delay_spread.setter
    def delay_spread(self, value):
        self._delay_spread = float(value)
        self._dev_tau = None

    def __call__(self, batch_size, num_time_steps, sampling_frequency):
        return self._invoke(batch_size, num_time_steps, sampling_frequency)

    def draws(self, batch_size):
        """The random draws of one call, from the global Philox stream: speed, velocity azimuth and zenith [B]; coupling
        normals [B, 4, clusters, 20] (arrival azimuth, departure azimuth, arrival zenith, departure zenith; their argsort
        per cluster permutes the rays); initial phases [B, clusters, 20, 4] (step 10)."""
        dev = config.device
        b, c = int(batch_size), self._num_clusters
        speed = philox_fill("sb_uniform", [b], self._min_speed, self._max_speed, dev)
        v_phi = philox_fill("sb_uniform", [b], 0.0, 2 * np.pi, dev)
        v_theta = philox_fill("sb_uniform", [b], 0.0, np.pi, dev)
        coupling = philox_fill("sb_normal", [b, 4, c, NUM_RAYS], 0.0, 1.0, dev)
        phases = philox_fill("sb_uniform", [b, c, NUM_RAYS, 4], -np.pi, np.pi, dev)
        return speed, v_phi, v_theta, coupling, phases

    def _tables(self, dev):
        if self._dev is None or self._dev[0] != dev:
            t = {k: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in self._host.items()}
            self._dev = (dev, t)
        return self._dev[1]

    def synthesize(self, draws, num_time_steps, sampling_frequency):
        """Cluster coefficients [B, num_rx_ant, num_tx_ant, clusters, T] from `draws` (kernel ``sb_cdl_coefficients``)."""
        speed, v_phi, v_theta, coupling, phases = draws
        dev = speed.device
        t = self._tables(dev)
        b, c = speed.shape[0], self._num_clusters
        nr, nt = self._rx_array.num_ant, self._tx_array.num_ant
        a = torch.empty((b, nr, nt, c, int(num_time_steps)), dtype=torch.complex64, device=dev)
        check(lib().sb_cdl_coefficients(
            ptr(speed), ptr(v_phi), ptr(v_theta), ptr(coupling), ptr(phases), ptr(t["rx_dir"]), ptr(t["rx_field"]),
            ptr(t["rx_phase"]), ptr(t["rx_pol"]), ptr(t["tx_field"]), ptr(t["tx_phase"]), ptr(t["tx_pol"]),
            ptr(t["cluster_scale"]), ptr(t["order"]), ptr(t["los_field"]), float(np.sqrt(1.0 / self._xpr)),
            float(self._wavenumber), ptr(a), b, c, nr, nt, int(num_time_steps), float(sampling_frequency),
            current_stream()), "sb_cdl_coefficients")
        return a

    def call(self, batch_size, num_time_steps, sampling_frequency):
        if self.precision != "single":
            raise NotImplementedError("CDL generates complex64 coefficients only.")
        batch_size = int(batch_size)
        a = self.synthesize(self.draws(batch_size), num_time_steps, sampling_frequency)
        nr, nt, c, t = a.shape[1:]
        a = a.reshape(batch_size, 1, nr, 1, nt, c, t)
        dev = a.device
        if self._dev_tau is None or self._dev_tau.device != dev:
            tau = (self._delays_norm[self._order] * self._delay_spread).astype(np.float32)
            self._dev_tau = torch.from_numpy(tau).to(dev).reshape(1, 1, 1, c)
        # every link has the same delays: a broadcast view (stride 0) says so without any device read-back
        return a, self._dev_tau.expand(batch_size, 1, 1, c)
