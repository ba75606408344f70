"""CDL host side (no GPU): TR 38.901 antenna arrays and element patterns, the CDL cluster tables with the LoS split and
delay ordering, and the empty-batch / bad-argument behaviour of sb_cdl_coefficients."""
import ctypes as C
import numpy as np
import pytest

FC = 3.0e9
LAM = 299792458.0 / FC


def test_single_antenna():
    from sionna_b200.phy.channel import Antenna
    a = Antenna("single", "V", "omni", FC)
    assert a.num_ant == 1 and a.polarization == "single" and a.polarization_type == "V"
    assert np.array_equal(a.ant_pos, np.zeros((1, 3))) and list(a.ant_ind_pol1) == [0]
    assert a.ant_pol1.slant_angle == 0.0
    with pytest.raises(AssertionError):
        a.ant_ind_pol2
    h = Antenna("single", "H", "omni", FC)
    assert np.isclose(h.ant_pol1.slant_angle, np.pi / 2)
    d = Antenna("dual", "VH", "omni", FC)
    assert d.num_ant == 2 and list(d.ant_ind_pol1) == [0] and list(d.ant_ind_pol2) == [1]
    assert np.array_equal(d.ant_pos, np.zeros((2, 3)))


def test_uniform_linear_cross_polarized_array():
    from sionna_b200.phy.channel import AntennaArray
    a = AntennaArray(1, 4, "dual", "cross", "38.901", FC)
    assert a.num_ant == 8
    y = np.array([-0.75, -0.25, 0.25, 0.75]) * LAM
    expect = np.zeros((8, 3))
    expect[:4, 1] = y
    expect[4:, 1] = y                                                   # second polarization: same positions
    assert np.allclose(a.ant_pos, expect, atol=1e-15)
    assert list(a.ant_ind_pol1) == [0, 1, 2, 3] and list(a.ant_ind_pol2) == [4, 5, 6, 7]
    assert np.allclose(a.ant_pos_pol2, expect[4:])
    assert np.isclose(a.ant_pol1.slant_angle, -np.pi / 4) and np.isclose(a.ant_pol2.slant_angle, np.pi / 4)
    assert list(a.ant_pol_index) == [0, 0, 0, 0, 1, 1, 1, 1]
    assert a.element_horizontal_spacing == 0.5 and a.num_rows_per_panel == 1 and a.num_cols_per_panel == 4


def test_two_by_two_panel_array():
    """2 x 2 panels of 2 x 2 dual-polarized elements: elements i + 2 j inside a panel, panels column-major, panel
    spacing 1 wavelength (panel size + 0.5), the whole array centred."""
    from sionna_b200.phy.channel import PanelArray
    a = PanelArray(2, 2, "dual", "VH", "omni", FC, num_rows=2, num_cols=2)
    assert a.num_ant == 32 and a.num_panels == 4 and a.num_panels_ant == 8
    assert a.panel_vertical_spacing == 1.0 and a.panel_horizontal_spacing == 1.0
    pos = a.ant_pos / LAM
    assert np.allclose(pos[0], [0, -0.75, 0.75])                        # panel (row 0, col 0), element (0, 0)
    assert np.allclose(pos[1], [0, -0.75, 0.25])                        # element (row 1, col 0)
    assert np.allclose(pos[2], [0, -0.25, 0.75])                        # element (row 0, col 1)
    assert np.allclose(pos[4], pos[0]) and np.allclose(pos[7], pos[3])  # second polarization
    assert np.allclose(pos[8], [0, -0.75, -0.25])                       # panel (row 1, col 0)
    assert np.allclose(pos[16], [0, 0.25, 0.75])                        # panel (row 0, col 1)
    assert np.allclose(pos[31], [0, 0.75, -0.75])
    assert np.allclose(pos.mean(0), 0.0)
    assert list(a.ant_ind_pol1) == [0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 19, 24, 25, 26, 27]
    assert list(a.ant_ind_pol2) == [i + 4 for i in a.ant_ind_pol1]
    with pytest.raises(AssertionError):
        PanelArray(2, 2, "dual", "VH", "omni", FC, num_cols=2, panel_horizontal_spacing=0.5)


def test_38901_element_pattern():
    from sionna_b200.phy.channel import AntennaElement
    e = AntennaElement("38.901")
    assert np.isclose(10 * np.log10(e.radiation_pattern(np.pi / 2, 0.0)), 8.0)            # boresight: 8 dBi
    assert np.isclose(10 * np.log10(e.radiation_pattern(np.pi / 2, np.pi)), 8.0 - 30.0)   # 30 dB floor
    assert np.isclose(10 * np.log10(e.radiation_pattern(0.0, 0.0)), 8.0 - 12 * (90 / 65) ** 2)
    assert np.isclose(10 * np.log10(e.radiation_pattern(np.pi, np.pi / 2)), 8.0 - 30.0)
    f_th, f_ph = AntennaElement("38.901", -np.pi / 4).field(np.pi / 2, 0.0)
    assert np.isclose(f_th, 10 ** 0.4 / np.sqrt(2)) and np.isclose(f_ph, -10 ** 0.4 / np.sqrt(2))
    assert np.allclose(AntennaElement("omni").radiation_pattern(np.array([0.1, 2.0]), np.array([3.0, -1.0])), 1.0)


def _cdl(model, direction="downlink"):
    from sionna_b200.phy.channel import CDL, Antenna
    ant = Antenna("single", "V", "omni", FC)
    return CDL(model, 100e-9, FC, ant, ant, direction)


def test_cdl_tables_round_trip():
    """The text tables hold TR 38.901 Tables 7.7.1-1..5 (spot values) in table order."""
    from sionna_b200.phy.channel.cdl import cdl_table
    d = {m: cdl_table(m) for m in "ABCDE"}
    assert [int(d[m]["num_clusters"]) for m in "ABCDE"] == [23, 23, 24, 13, 14]
    assert [len(d[m]["delays"]) for m in "ABCDE"] == [23, 23, 24, 14, 15]
    assert [int(d[m]["los"]) for m in "ABCDE"] == [0, 0, 0, 1, 1]
    assert [float(d[m]["xpr_db"]) for m in "ABCDE"] == [10.0, 8.0, 7.0, 11.0, 8.0]
    a, e = d["A"], d["E"]
    assert np.allclose(a["delays"][:3], [0.0, 0.3819, 0.4025]) and np.allclose(a["powers_db"][:3], [-13.4, 0, -2.2])
    assert (a["aod"][0], a["aoa"][0], a["zod"][0], a["zoa"][0]) == (-178.1, 51.3, 50.2, 125.4)
    assert (a["cASD"], a["cASA"], a["cZSD"], a["cZSA"]) == (5.0, 11.0, 3.0, 3.0)
    assert np.allclose(e["powers_db"][:3], [-0.03, -22.03, -15.8]) and e["aoa"][0] == -180.0
    assert e["delays"][3] == e["delays"][5] == 0.544
    for m in "ABCDE":
        n = len(d[m]["delays"])
        assert all(d[m][k].shape == (n,) and d[m][k].dtype == np.float64 for k in ("powers_db", "aod", "aoa", "zod", "zoa"))


@pytest.mark.parametrize("model", ["A", "B", "C", "D", "E"])
def test_cdl_los_split_and_properties(model):
    from sionna_b200.phy.channel.cdl import cdl_table
    cdl = _cdl(model)
    t = cdl_table(model)
    p = 10 ** (t["powers_db"] / 10)
    delays = t["delays"]
    p = p / p.sum()
    assert cdl.num_clusters == len(cdl.powers) == len(cdl.delays)
    assert np.isclose(float(cdl.powers.sum()), 1.0, atol=1e-6)
    if not cdl.los:
        assert np.allclose(cdl.powers.numpy(), p, rtol=1e-6)
        assert np.allclose(cdl.delays.numpy(), delays * 100e-9)
        with pytest.raises(AssertionError):
            cdl.k_factor
        return
    nlos = p[1:] / p[1:].sum()                                         # specular row removed, NLoS renormalised
    k = p[0] / p[1:].sum()
    assert cdl.num_clusters == len(delays) - 1
    assert np.isclose(cdl.k_factor, k / nlos[0], rtol=1e-6)
    expect = nlos.copy()
    expect[0] += k
    assert np.allclose(cdl.powers.numpy(), expect / (k + 1), rtol=1e-5)
    # the zero-delay cluster keeps the table's specular / NLoS ratio
    assert np.isclose(cdl.k_factor, p[0] / p[1], rtol=1e-6)
    assert np.allclose(cdl.delays.numpy(), delays[1:] * 100e-9)


def test_cdl_cluster_order_is_a_stable_delay_sort():
    cdl = _cdl("E")
    assert list(cdl._order[:6]) == [0, 1, 2, 4, 3, 5]                  # tie 0.544: lower table index first
    d = cdl.delays.numpy()[cdl._order]
    assert np.all(np.diff(d) >= 0) and d[0] == 0.0
    cdl.delay_spread = 300e-9
    assert cdl.delay_spread == 300e-9 and np.allclose(cdl.delays.numpy()[4], 0.544 * 300e-9)
    with pytest.raises(AssertionError):
        _cdl("F")


def test_cdl_uplink_swaps_arrival_and_departure():
    down, up = _cdl("C", "downlink"), _cdl("C", "uplink")
    assert np.array_equal(up._rays["aoa"], down._rays["aod"]) and np.array_equal(up._rays["zod"], down._rays["zoa"])
    assert np.allclose(down._rays["aoa"][0], np.deg2rad(-101.0 + 15.0 * np.array(
        [0.0447, -0.0447, 0.1413, -0.1413, 0.2492, -0.2492, 0.3715, -0.3715, 0.5129, -0.5129,
         0.6797, -0.6797, 0.8844, -0.8844, 1.1481, -1.1481, 1.5195, -1.5195, 2.1551, -2.1551])))


def test_cdl_coefficients_empty_batch_and_bad_arguments(sb_lib):
    args = [None] * 15 + [0.0, 0.0, None]
    assert sb_lib.sb_cdl_coefficients(*args, 0, 0, 0, 0, 0, 0.0, None) == 0
    assert sb_lib.sb_cdl_coefficients(*args, 1, 23, 4, 8, 14, 14e3, None) != 0
    assert b"sb_cdl_coefficients" in sb_lib.sb_last_error()
