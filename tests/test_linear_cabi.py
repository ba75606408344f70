"""Argument checks of the ZF / MF / pseudo-inverse modes of sb_mimo_linalg, of sb_ofdm_equalize and of
sb_symbol_demap that run before any device access (no GPU needed): malformed arguments are SB_EINVAL, shapes beyond the
limits SB_EUNSUPPORTED with a message, and the largest supported shapes pass the checks with an empty batch."""
import ctypes

import pytest

SB_EINVAL, SB_EUNSUPPORTED = -1, -4


def _buf():
    return ctypes.cast(ctypes.create_string_buffer(256), ctypes.c_void_p)


@pytest.mark.parametrize("mode,k,y,s,out1,text", [
    (7, 2, True, True, True, b"bad arguments"),
    (4, 2, False, True, True, b"needs y, h, s and two outputs"),
    (5, 2, True, False, True, b"needs y, h, s and two outputs"),
    (4, 2, True, True, False, b"needs y, h, s and two outputs"),
    (6, 5, False, False, False, b"need 1 <= K <= M"),
    (5, 0, True, True, True, b"need 1 <= K <= M"),
])
def test_mimo_linalg_new_modes_malformed(sb_lib, mode, k, y, s, out1, text):
    p = _buf()
    rc = sb_lib.sb_mimo_linalg(mode, p if y else None, p, p if s else None, p, p if out1 else None, 1, 4, k, None)
    assert rc == SB_EINVAL
    assert text in sb_lib.sb_last_error()


def _ofdm(lib, eq=2, batch=0, rx=1, ant=4, txs=4, K=4, KU=0, S=14, F=76, ND=64, ptrs=None):
    ptrs = ptrs if ptrs is not None else [None] * 12
    return lib.sb_ofdm_equalize(eq, *ptrs, batch, rx, ant, txs, S, F, K, KU, ND, None)


@pytest.mark.parametrize("args,text", [
    (dict(K=17, ant=32, txs=17), b"17 streams per receiver with 32 receive antennas"),
    (dict(K=4, ant=3), b"4 streams per receiver with 3 receive antennas"),
    (dict(K=0), b"0 streams per receiver"),
])
def test_ofdm_equalize_limits(sb_lib, args, text):
    assert _ofdm(sb_lib, **args) == SB_EUNSUPPORTED
    assert text in sb_lib.sb_last_error()


@pytest.mark.parametrize("args,text", [
    (dict(eq=4), b"equalizer must be"),
    (dict(eq=-1), b"equalizer must be"),
    (dict(batch=-1), b"bad sizes"),
    (dict(S=0), b"bad sizes"),
    (dict(KU=-1), b"bad sizes"),
    (dict(batch=1), b"bad pointers"),
])
def test_ofdm_equalize_malformed(sb_lib, args, text):
    assert _ofdm(sb_lib, **args) == SB_EINVAL
    assert text in sb_lib.sb_last_error()


def test_ofdm_equalize_missing_interferer_table(sb_lib):
    p = _buf()
    ptrs = [p] * 12
    ptrs[7] = None                                                      # d_undesired
    assert _ofdm(sb_lib, batch=1, KU=1, ptrs=ptrs) == SB_EINVAL


@pytest.mark.parametrize("eq", [0, 1, 2, 3])
def test_ofdm_equalize_scratch_limit(sb_lib, eq):
    """With an interfering stream the shared-memory kernel runs; 160 antennas need more than 200 KB per element."""
    p = _buf()
    assert _ofdm(sb_lib, eq=eq, batch=1, ant=160, K=1, KU=1, txs=2, ptrs=[p] * 12) == SB_EUNSUPPORTED
    assert b"sb_ofdm_equalize: 160 receive antennas, 1 streams need" in sb_lib.sb_last_error()
    assert b"the limit is 204800" in sb_lib.sb_last_error()


def test_ofdm_equalize_largest_shapes_pass_the_checks(sb_lib):
    for eq in range(4):
        assert _ofdm(sb_lib, eq=eq, K=16, ant=16, txs=16) == 0
        assert _ofdm(sb_lib, eq=eq, K=1, ant=4096, txs=1) == 0


def _sym(lib, P=16, n=0, no_inner=1, prior=False, prior_inner=1, hard=0, ptrs=False):
    p = _buf() if ptrs else None
    return lib.sb_symbol_demap(p, p, no_inner, p, P, _buf() if prior else None, prior_inner, p, n, hard, None)


@pytest.mark.parametrize("args,text", [
    (dict(P=1), b"num_points = 1, supported are 2 ... 1024"),
    (dict(P=1025), b"num_points = 1025, supported are 2 ... 1024"),
    (dict(no_inner=0), b"bad arguments"),
    (dict(prior=True, prior_inner=0), b"bad arguments"),
    (dict(hard=2), b"bad arguments"),
    (dict(n=-1), b"bad arguments"),
    (dict(n=1), b"missing input or output"),
])
def test_symbol_demap_malformed(sb_lib, args, text):
    assert _sym(sb_lib, **args) == SB_EINVAL
    assert text in sb_lib.sb_last_error()


def test_symbol_demap_range_passes_the_checks(sb_lib):
    for P in (2, 3, 1024):
        assert _sym(sb_lib, P=P) == 0


def test_unsupported_shapes_raise_a_value_error(sb_lib):
    """check() turns SB_EUNSUPPORTED into SbUnsupportedError, which is both the library's SbError and a ValueError;
    other failures stay SbError only."""
    from sionna_b200._lib import SbError, SbUnsupportedError, check
    with pytest.raises(SbUnsupportedError, match="17 streams per receiver") as e:
        check(_ofdm(sb_lib, K=17, ant=32, txs=17), "sb_ofdm_equalize")
    assert isinstance(e.value, ValueError) and isinstance(e.value, SbError)
    with pytest.raises(SbError, match="equalizer must be") as e:
        check(_ofdm(sb_lib, eq=4), "sb_ofdm_equalize")
    assert not isinstance(e.value, ValueError)
