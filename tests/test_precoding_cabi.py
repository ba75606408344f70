"""Argument checks of sb_mimo_precode / sb_ofdm_precode that run before any device access (no GPU needed): malformed
arguments are SB_EINVAL, shapes beyond the limits SB_EUNSUPPORTED with a message, and the largest supported shapes pass
the checks with an empty batch."""
import ctypes

import pytest

SB_EINVAL, SB_EUNSUPPORTED = -1, -4


def _dense(lib, K=4, M=8, kind=0, num=0, alpha_stride=0, x=False, gx=False, alpha=False, h=False, g=False):
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    return lib.sb_mimo_precode(p if h else None, p if alpha else None, alpha_stride, p if x else None,
                               p if g else None, p if gx else None, num, K, M, kind, None)


def _ofdm(lib, batch=0, rx=1, ra=4, tx=1, M=8, K=4, S=14, F=76, NE=64, kind=0, ptrs=None):
    ptrs = ptrs or [None] * 11
    return lib.sb_ofdm_precode(*ptrs, batch, rx, ra, tx, M, K, S, F, NE, kind, None)


@pytest.mark.parametrize("args,text", [
    (dict(K=17, M=32), b"17 streams, the limit is 16"),
    (dict(K=4, M=1025), b"1025 transmit antennas, the limit is 1024"),
])
def test_dense_limits(sb_lib, args, text):
    assert _dense(sb_lib, **args) == SB_EUNSUPPORTED
    assert text in sb_lib.sb_last_error()


@pytest.mark.parametrize("args,text", [
    (dict(K=0), b"bad arguments"),
    (dict(M=0), b"bad arguments"),
    (dict(kind=3), b"kind in {0, 1, 2}"),
    (dict(kind=2, K=8), b"kind in {0, 1}"),
    (dict(alpha_stride=2), b"alpha_stride in {0, 1}"),
    (dict(gx=True), b"Gx needs x"),
    (dict(kind=1, alpha=True), b"alpha needs rzf"),
    (dict(num=-1), b"bad arguments"),
    (dict(num=1), b"need h and an output"),
    (dict(num=1, h=True), b"need h and an output"),
])
def test_dense_malformed_arguments(sb_lib, args, text):
    assert _dense(sb_lib, **args) == SB_EINVAL
    assert text in sb_lib.sb_last_error()


@pytest.mark.parametrize("args,text", [
    (dict(K=18, ra=2, rx=9), b"18 streams, the limit is 16"),
    (dict(M=2048), b"2048 transmit antennas, the limit is 1024"),
])
def test_ofdm_limits(sb_lib, args, text):
    assert _ofdm(sb_lib, **args) == SB_EUNSUPPORTED
    assert text in sb_lib.sb_last_error()


@pytest.mark.parametrize("args,text", [
    (dict(K=4, ra=3), b"does not match the channel dimensions"),
    (dict(K=8, ra=4, rx=1), b"does not match the channel dimensions"),
    (dict(kind=2, K=4, M=8), b"num_streams_per_tx = num_tx_ant"),
    (dict(kind=-1), b"kind in {0, 1, 2}"),
    (dict(NE=77), b"sizes"),
    (dict(S=0), b"sizes"),
    (dict(batch=-1), b"sizes"),
    (dict(batch=1), b"pointers"),
])
def test_ofdm_malformed_arguments(sb_lib, args, text):
    assert _ofdm(sb_lib, **args) == SB_EINVAL
    assert text in sb_lib.sb_last_error()


def test_ofdm_missing_inputs(sb_lib):
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    # h_hat, h, pind, x, alpha, alpha strides, tx_power, tx_power strides, sc_pos, x_precoded, h_eff
    no_x = [p, p, p, None, None, None, None, None, p, p, None]
    assert _ofdm(sb_lib, batch=1, ptrs=no_x) == SB_EINVAL
    no_sc_pos = [p, p, p, None, None, None, None, None, None, None, p]
    assert _ofdm(sb_lib, batch=1, ptrs=no_sc_pos) == SB_EINVAL
    no_strides = [p, p, p, p, p, None, None, None, p, p, None]
    assert _ofdm(sb_lib, batch=1, ptrs=no_strides) == SB_EINVAL


def test_largest_supported_shapes_pass_the_checks(sb_lib):
    assert _dense(sb_lib, K=16, M=1024) == 0
    assert _dense(sb_lib, K=16, M=4, kind=1) == 0                     # K > M is accepted
    assert _ofdm(sb_lib, K=16, ra=2, rx=8, M=1024) == 0
    assert _ofdm(sb_lib, K=16, ra=16, rx=1, M=16, kind=2) == 0
    assert _ofdm(sb_lib, K=16, ra=2, rx=8, M=64, S=14, F=1024, NE=1024) == 0
