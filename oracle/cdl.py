"""Oracle: CDL cluster coefficients, TR 38.901 section 7.5 steps 10 and 11 without sub-clustering.
TEST INFRASTRUCTURE (NumPy). Restates the arithmetic of /root/reference/src/sionna/phy/channel/tr38901/
channel_coefficients.py:196-1030 and the random coupling of cdl.py:629-695 ray by ray, directly from the angles (no
tables), in the real type ``dtype``: float64 for the reference value, float32 for the error a single-precision
evaluation makes, which calibrates the tolerance of the kernel.
"""
import numpy as np

_C = 299792458.0


def _rot(o, f):
    a, b, c = (f(v) for v in o)
    cos, sin = np.cos, np.sin
    return np.array([[cos(a) * cos(b), cos(a) * sin(b) * sin(c) - sin(a) * cos(c), cos(a) * sin(b) * cos(c) + sin(a) * sin(c)],
                     [sin(a) * cos(b), sin(a) * sin(b) * sin(c) + cos(a) * cos(c), sin(a) * sin(b) * cos(c) - cos(a) * sin(c)],
                     [-sin(b), cos(b) * sin(c), cos(b) * cos(c)]], dtype=type(f(0)))


def _unit(theta, phi):
    return np.stack([np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.cos(theta)], axis=-1)


def _pattern(name, theta, phi, f):
    if name == "omni":
        return np.ones_like(theta)
    t3 = f(65.0 / 180.0 * np.pi)
    a_v = -np.minimum(f(12) * ((theta - f(np.pi / 2)) / t3) ** 2, f(30))
    a_h = -np.minimum(f(12) * (phi / t3) ** 2, f(30))
    a_db = -np.minimum(-(a_v + a_h), f(30)) + f(8)
    return f(10) ** (a_db / f(10))


def _field(element, o, theta, phi, f):
    """GCS field (7.1-11) of ``element`` with orientation ``o``: [..., 2] (theta, phi components)."""
    r = np.einsum("ji,...j->...i", _rot(o, f), _unit(theta, phi))        # R^T rho (7.1-7/8)
    th_p = np.arccos(np.clip(r[..., 2], f(-1), f(1)))
    ph_p = np.angle(r[..., 0] + 1j * r[..., 1]).astype(f)
    amp = np.sqrt(_pattern(element.pattern, th_p, ph_p, f))
    f_th, f_ph = amp * f(np.cos(element.slant_angle)), amp * f(np.sin(element.slant_angle))
    a, b, c = (f(v) for v in o)
    re = np.sin(c) * np.cos(theta) * np.sin(phi - a) + np.cos(c) * (np.cos(b) * np.sin(theta) - np.sin(b) * np.cos(theta)
                                                                     * np.cos(phi - a))
    im = np.sin(c) * np.cos(phi - a) + np.sin(b) * np.cos(c) * np.sin(phi - a)
    psi = np.angle(re + 1j * im).astype(f)                               # (7.1-15)
    return np.stack([np.cos(psi) * f_th - np.sin(psi) * f_ph, np.sin(psi) * f_th + np.cos(psi) * f_ph], axis=-1)


def _ant_fields(array, o, theta, phi, f):
    """[num_ant, ..., 2]: every antenna's GCS field (the second polarization where ``ant_ind_pol2`` says so)."""
    f1 = _field(array.ant_pol1, o, theta, phi, f)
    out = np.repeat(f1[None], array.num_ant, axis=0)
    if array.polarization == "dual":
        out[array.ant_ind_pol2] = _field(array.ant_pol2, o, theta, phi, f)
    return out


def _array_phase(array, o, theta, phi, wavenumber, f):
    """exp(j k r.d) with d the GCS antenna positions: [..., num_ant]."""
    d = np.asarray(array.ant_pos, f) @ _rot(o, f).T
    return np.exp(1j * (wavenumber * (_unit(theta, phi) @ d.T)))


def cdl_coefficients(cdl, speed, v_phi, v_theta, coupling, phases, num_time_steps, fs, dtype=np.float64):
    """a [B, num_rx_ant, num_tx_ant, clusters, T] of ``cdl`` (a `sionna_b200.phy.channel.CDL`) from its draws
    (`CDL.draws`), clusters in ascending delay."""
    f = np.dtype(dtype).type
    ctype = np.complex128 if f is np.float64 else np.complex64
    tx_o, rx_o = cdl._orientations
    txa, rxa = cdl.tx_array, cdl.rx_array
    k = f(2 * np.pi * cdl._carrier_frequency / _C)
    perm = np.argsort(coupling, axis=-1, kind="stable")                  # [B, 4, C, 20] (cdl.py:648-651)
    sh = {name: np.take_along_axis(np.broadcast_to(cdl._rays[name].astype(f), perm[:, 0].shape), perm[:, i], -1)
          for i, name in enumerate(("aoa", "aod", "zoa", "zod"))}     # [B, C, 20]
    f_rx = _ant_fields(rxa, rx_o, sh["zoa"], sh["aoa"], f)                # [Nr, B, C, 20, 2]
    f_tx = _ant_fields(txa, tx_o, sh["zod"], sh["aod"], f)                # [Nt, B, C, 20, 2]
    e = np.exp(1j * phases.astype(f)).astype(ctype)                      # [B, C, 20, 4]
    x = f(np.sqrt(1.0 / cdl._xpr))
    m = np.stack([np.stack([e[..., 0], x * e[..., 1]], -1), np.stack([x * e[..., 2], e[..., 3]], -1)], -2)
    h_field = np.einsum("ubcrp,bcrpq,vbcrq->bcruv", f_rx.astype(ctype), m, f_tx.astype(ctype))   # (7.5-22)
    h_array = (_array_phase(rxa, rx_o, sh["zoa"], sh["aoa"], k, f)[..., :, None]
               * _array_phase(txa, tx_o, sh["zod"], sh["aod"], k, f)[..., None, :])
    vel = np.stack([speed * np.cos(v_phi) * np.sin(v_theta), speed * np.sin(v_phi) * np.sin(v_theta),
                    speed * np.cos(v_theta)], -1).astype(f)              # [B, 3]
    t = np.arange(num_time_steps, dtype=f) / f(fs)
    r_rx = _unit(sh["zoa"], sh["aoa"])                                   # Doppler uses the arrival direction (:517-573)
    dop = np.exp(1j * (k * np.einsum("bcri,bi->bcr", r_rx, vel)[..., None] * t)).astype(ctype)   # [B, C, 20, T]
    p = cdl._nlos_powers.astype(f)
    scale = np.sqrt(p / f(20))
    if cdl.los:
        scale = scale * np.sqrt(f(1) / (f(cdl._k) + f(1)))
    h = np.einsum("bcruv,bcrt->buvct", (h_field * h_array).astype(ctype), dop) * scale[None, None, None, :, None]
    h = h[:, :, :, cdl._order]                                           # ascending delay, stable (:908-915)
    if cdl.los:                                                          # (7.5-29), added to the zero-delay cluster
        la = {n: f(v) for n, v in cdl._los_angles.items()}
        fr = _ant_fields(rxa, rx_o, la["zoa"], la["aoa"], f)             # [Nr, 2]
        ft = _ant_fields(txa, tx_o, la["zod"], la["aod"], f)
        g = fr[:, None, 0] * ft[None, :, 0] - fr[:, None, 1] * ft[None, :, 1]
        arr = (_array_phase(rxa, rx_o, la["zoa"], la["aoa"], k, f)[:, None]
               * _array_phase(txa, tx_o, la["zod"], la["aod"], k, f)[None, :])
        w = k * (vel @ _unit(la["zoa"], la["aoa"]))                       # [B]
        d = np.exp(1j * (w[:, None] * t[None, :]))                       # [B, T]
        los = np.sqrt(f(cdl._k) / (f(cdl._k) + f(1))) * (g * arr)[None, :, :, None] * d[:, None, None, :]
        h[:, :, :, 0] += los.astype(ctype)
    return h
