"""TR 38.901 antenna elements and panel arrays (host only, float64 NumPy): mirror of
/root/reference/src/sionna/phy/channel/tr38901/antenna.py:17-743 without the plotting and gain-integration helpers.
`CDL` tabulates the element fields and array phases from these objects once per instance (cdl.py)."""
import numpy as np

SPEED_OF_LIGHT = 299792458.0


class AntennaElement:
    """Element with radiation pattern ``"omni"`` or ``"38.901"`` (Table 7.3-1) and polarization slant angle [rad]."""

    def __init__(self, pattern, slant_angle=0.0, precision=None):
        assert pattern in ("omni", "38.901"), "The radiation_pattern must be one of [\"omni\", \"38.901\"]."
        self._pattern = pattern
        self._slant_angle = float(slant_angle)

    pattern = property(lambda self: self._pattern)
    slant_angle = property(lambda self: self._slant_angle)

    def radiation_pattern(self, theta, phi):
        """Linear power pattern at LCS zenith ``theta`` in [0, pi] and azimuth ``phi`` in (-pi, pi]."""
        theta, phi = np.asarray(theta, np.float64), np.asarray(phi, np.float64)
        if self._pattern == "omni":
            return np.ones(np.broadcast(theta, phi).shape)
        theta_3db = phi_3db = 65.0 / 180.0 * np.pi
        a_max = sla_v = 30.0
        a_v = -np.minimum(12.0 * ((theta - np.pi / 2) / theta_3db) ** 2, sla_v)
        a_h = -np.minimum(12.0 * (phi / phi_3db) ** 2, a_max)
        a_db = -np.minimum(-(a_v + a_h), a_max) + 8.0                     # G_E,max = 8 dBi
        return 10.0 ** (a_db / 10.0)

    def field(self, theta, phi):
        """(F_theta, F_phi) in the LCS (7.3-4/5)."""
        a = np.sqrt(self.radiation_pattern(theta, phi))
        return a * np.cos(self._slant_angle), a * np.sin(self._slant_angle)


def _panel_positions(num_rows, num_cols, polarization, vertical_spacing, horizontal_spacing):
    """Element positions of one panel in wavelengths: element i + j * rows at (0, j dh, -i dv), centred; with dual
    polarization the second half repeats the first."""
    p = 1 if polarization == "single" else 2
    pos = np.zeros([num_rows * num_cols * p, 3])
    for i in range(num_rows):
        for j in range(num_cols):
            pos[i + j * num_rows] = [0.0, j * horizontal_spacing, -i * vertical_spacing]
    pos += [0.0, -(num_cols - 1) * horizontal_spacing / 2, (num_rows - 1) * vertical_spacing / 2]
    if polarization == "dual":
        pos[num_rows * num_cols:] = pos[:num_rows * num_cols]
    return pos


class PanelArray:
    """PanelArray(num_rows_per_panel, num_cols_per_panel, polarization, polarization_type, antenna_pattern, carrier_frequency, num_rows=1, num_cols=1, panel_vertical_spacing=None, panel_horizontal_spacing=None, element_vertical_spacing=None, element_horizontal_spacing=None, precision=None)

    Uniform rectangular panels of antenna elements on the y-z plane of the LCS. ``polarization`` "single" (type "V" or
    "H") or "dual" (type "VH" or "cross"); spacings in wavelengths (elements 0.5 by default, panels the panel size +
    0.5). Panels are placed column-major and the whole array is centred and scaled by the wavelength: ``ant_pos`` is in
    metres. Within a panel the first half of the elements carries the first polarization and the second half the
    second one."""

    def __init__(self, num_rows_per_panel, num_cols_per_panel, polarization, polarization_type, antenna_pattern,
                 carrier_frequency, num_rows=1, num_cols=1, panel_vertical_spacing=None, panel_horizontal_spacing=None,
                 element_vertical_spacing=None, element_horizontal_spacing=None, precision=None):
        assert polarization in ("single", "dual"), "polarization must be either 'single' or 'dual'"
        assert precision in (None, "single", "double"), "precision must be None, 'single' or 'double'"
        ev = 0.5 if element_vertical_spacing is None else float(element_vertical_spacing)
        eh = 0.5 if element_horizontal_spacing is None else float(element_horizontal_spacing)
        pv = (num_rows_per_panel - 1) * ev + 0.5 if panel_vertical_spacing is None else float(panel_vertical_spacing)
        ph = (num_cols_per_panel - 1) * eh + 0.5 if panel_horizontal_spacing is None else float(panel_horizontal_spacing)
        assert ph > (num_cols_per_panel - 1) * eh, "Pannel horizontal spacing must be larger than the panel width"
        assert pv > (num_rows_per_panel - 1) * ev, "Pannel vertical spacing must be larger than panel height"
        self._num_rows, self._num_cols = int(num_rows), int(num_cols)
        self._num_rows_per_panel, self._num_cols_per_panel = int(num_rows_per_panel), int(num_cols_per_panel)
        self._polarization, self._polarization_type = polarization, polarization_type
        self._panel_vertical_spacing, self._panel_horizontal_spacing = pv, ph
        self._element_vertical_spacing, self._element_horizontal_spacing = ev, eh
        p = 1 if polarization == "single" else 2
        self._num_panels = self._num_rows * self._num_cols
        self._num_panel_ant = self._num_rows_per_panel * self._num_cols_per_panel * p
        self._num_ant = self._num_panels * self._num_panel_ant
        self._lambda_0 = SPEED_OF_LIGHT / float(carrier_frequency)
        if polarization == "single":
            assert polarization_type in ("V", "H"), "For single polarization, polarization_type must be 'V' or 'H'"
            slant = 0.0 if polarization_type == "V" else np.pi / 2
            self._ant_pol1, self._ant_pol2 = AntennaElement(antenna_pattern, slant), None
        else:
            assert polarization_type in ("VH", "cross"), "For dual polarization, polarization_type must be 'VH' or 'cross'"
            slant = 0.0 if polarization_type == "VH" else -np.pi / 4
            self._ant_pol1 = AntennaElement(antenna_pattern, slant)
            self._ant_pol2 = AntennaElement(antenna_pattern, slant + np.pi / 2)
        panel = _panel_positions(self._num_rows_per_panel, self._num_cols_per_panel, polarization, ev, eh)
        pos = np.zeros([self._num_ant, 3])
        count = 0
        for j in range(self._num_cols):
            for i in range(self._num_rows):
                pos[count * self._num_panel_ant:(count + 1) * self._num_panel_ant] = panel + [0.0, j * ph, -i * pv]
                count += 1
        pos += [0.0, -(self._num_cols - 1) * ph / 2, (self._num_rows - 1) * pv / 2]
        self._ant_pos = pos * self._lambda_0
        ind = np.arange(self._num_ant).reshape(self._num_panels * p, -1)
        self._ant_ind_pol1 = ind[::p].reshape(-1).astype(np.int32)
        self._ant_ind_pol2 = (ind[1::2].reshape(-1) if p == 2 else np.zeros([0])).astype(np.int32)

    num_rows = property(lambda self: self._num_rows)
    num_cols = property(lambda self: self._num_cols)
    num_rows_per_panel = property(lambda self: self._num_rows_per_panel)
    num_cols_per_panel = property(lambda self: self._num_cols_per_panel)
    polarization = property(lambda self: self._polarization)
    polarization_type = property(lambda self: self._polarization_type)
    panel_vertical_spacing = property(lambda self: self._panel_vertical_spacing)
    panel_horizontal_spacing = property(lambda self: self._panel_horizontal_spacing)
    element_vertical_spacing = property(lambda self: self._element_vertical_spacing)
    element_horizontal_spacing = property(lambda self: self._element_horizontal_spacing)
    num_panels = property(lambda self: self._num_panels)
    num_panels_ant = property(lambda self: self._num_panel_ant)
    num_ant = property(lambda self: self._num_ant)
    ant_pol1 = property(lambda self: self._ant_pol1)
    ant_pos = property(lambda self: self._ant_pos)
    ant_ind_pol1 = property(lambda self: self._ant_ind_pol1)
    ant_pos_pol1 = property(lambda self: self._ant_pos[self._ant_ind_pol1])

    @property
    def ant_pol2(self):
        assert self._polarization == "dual", "This property is not defined with single polarization"
        return self._ant_pol2

    @property
    def ant_ind_pol2(self):
        assert self._polarization == "dual", "This property is not defined with single polarization"
        return self._ant_ind_pol2

    @property
    def ant_pos_pol2(self):
        assert self._polarization == "dual", "This property is not defined with single polarization"
        return self._ant_pos[self._ant_ind_pol2]

    @property
    def ant_pol_index(self):
        """Polarization (0: first, 1: second) of every antenna; single-polarized arrays are all 0."""
        idx = np.zeros(self._num_ant, np.int32)
        idx[self._ant_ind_pol2] = 1
        return idx


class Antenna(PanelArray):
    """Antenna(polarization, polarization_type, antenna_pattern, carrier_frequency, precision=None): one element (two
    co-located ones with dual polarization)."""

    def __init__(self, polarization, polarization_type, antenna_pattern, carrier_frequency, precision=None):
        super().__init__(1, 1, polarization, polarization_type, antenna_pattern, carrier_frequency, precision=precision)


class AntennaArray(PanelArray):
    """AntennaArray(num_rows, num_cols, polarization, polarization_type, antenna_pattern, carrier_frequency, vertical_spacing=None, horizontal_spacing=None, precision=None):
    one panel of ``num_rows`` x ``num_cols`` elements."""

    def __init__(self, num_rows, num_cols, polarization, polarization_type, antenna_pattern, carrier_frequency,
                 vertical_spacing=None, horizontal_spacing=None, precision=None):
        super().__init__(num_rows, num_cols, polarization, polarization_type, antenna_pattern, carrier_frequency,
                         element_vertical_spacing=vertical_spacing, element_horizontal_spacing=horizontal_spacing,
                         precision=precision)
