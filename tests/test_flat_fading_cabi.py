"""Argument checks of sb_flat_fading / sb_chol_lower that run before any device access (no GPU needed): malformed
arguments are SB_EINVAL, shapes beyond the limits SB_EUNSUPPORTED with a message, and the largest supported shapes pass
the checks with an empty batch."""
import ctypes

import pytest

SB_EINVAL, SB_EUNSUPPORTED = -1, -4


def _ff(lib, num=0, M=16, K=4, h_in=False, h_stride=0, tx=False, tx_stride=0, rx=False, rx_stride=0, per_column=0,
        h_out=True, x=False, x_stride=0, no=False, no_inner=1, y=False):
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    q = lambda flag: p if flag else None                             # noqa: E731
    return lib.sb_flat_fading(q(h_in), h_stride, 1, 2, q(tx), tx_stride, q(rx), rx_stride, per_column, q(h_out), q(x),
                              x_stride, q(no), no_inner, 3, 4, q(y), num, M, K, None)


@pytest.mark.parametrize("args,text", [
    (dict(M=129, rx=True), b"num_rx_ant = 129 with an rx factor, the limit is 128"),
    (dict(M=129, rx=True, per_column=1), b"num_rx_ant = 129 with an rx factor, the limit is 128"),
    (dict(K=129, tx=True), b"num_tx_ant = 129 with a tx factor, the limit is 128"),
    (dict(M=128, K=129, rx=True), b"128 x 129 channel with correlation, the limit is M K <= 16384"),
    (dict(M=200, K=100, tx=True), b"200 x 100 channel with correlation, the limit is M K <= 16384"),
])
def test_flat_fading_limits(sb_lib, args, text):
    assert _ff(sb_lib, **args) == SB_EUNSUPPORTED
    assert text in sb_lib.sb_last_error()


@pytest.mark.parametrize("args,text", [
    (dict(num=-1), b"bad sizes"),
    (dict(M=0), b"bad sizes"),
    (dict(K=0), b"bad sizes"),
    (dict(h_stride=2), b"strides must be 0 or 1"),
    (dict(tx=True, tx_stride=-1), b"strides must be 0 or 1"),
    (dict(rx=True, rx_stride=2), b"strides must be 0 or 1"),
    (dict(x=True, y=True, x_stride=3), b"strides must be 0 or 1"),
    (dict(per_column=1), b"per_column is 0, or 1 with an rx factor set and no tx factor"),
    (dict(per_column=1, rx=True, tx=True), b"per_column is 0, or 1 with an rx factor set and no tx factor"),
    (dict(per_column=2, rx=True), b"per_column is 0, or 1"),
    (dict(h_out=False), b"nothing to compute"),
    (dict(x=True), b"x needs y"),
    (dict(no=True), b"noise needs x"),
    (dict(x=True, y=True, no=True, no_inner=0), b"no_inner >= 1"),
])
def test_flat_fading_malformed_arguments(sb_lib, args, text):
    assert _ff(sb_lib, **args) == SB_EINVAL
    assert text in sb_lib.sb_last_error()


def test_flat_fading_largest_supported_shapes_pass_the_checks(sb_lib):
    assert _ff(sb_lib, M=128, K=128, tx=True, rx=True, x=True, y=True, no=True) == 0
    assert _ff(sb_lib, M=128, K=128, rx=True, rx_stride=1, per_column=1, h_out=False, x=True, y=True) == 0
    assert _ff(sb_lib, M=16384, K=1, rx=False, tx=False) == 0
    assert _ff(sb_lib, M=1, K=128, tx=True, tx_stride=1) == 0
    assert _ff(sb_lib, M=1 << 20, K=1 << 20, h_in=True, x=True, y=True) == 0        # no factors: any M and K


def test_chol_lower_checks(sb_lib):
    assert sb_lib.sb_chol_lower(None, None, 0, 129, None) == SB_EUNSUPPORTED
    assert b"n = 129, the limit is 128" in sb_lib.sb_last_error()
    assert sb_lib.sb_chol_lower(None, None, 0, 0, None) == SB_EINVAL
    assert b"bad sizes" in sb_lib.sb_last_error()
    assert sb_lib.sb_chol_lower(None, None, -1, 4, None) == SB_EINVAL
    assert sb_lib.sb_chol_lower(None, None, 1, 4, None) == SB_EINVAL
    assert b"missing input or output" in sb_lib.sb_last_error()
    assert sb_lib.sb_chol_lower(None, None, 0, 128, None) == 0
