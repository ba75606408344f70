"""Argument checks of sb_mimo_ml / sb_ofdm_ml that run before any device access (no GPU needed): malformed arguments
are SB_EINVAL, configurations beyond the kernels' limits SB_EUNSUPPORTED with a message, a missing or short workspace
SB_ENOMEM."""
import pytest

SB_EINVAL, SB_ENOMEM, SB_EUNSUPPORTED = -1, -3, -4


def _mimo_ml(lib, k, num_points, method=0, output=0, hard_out=0, ws=None, ws_bytes=0, num=1):
    return lib.sb_mimo_ml(None, None, None, None, None, None, ws, ws_bytes, num, 4, k, num_points, method, output,
                          hard_out, None)


@pytest.mark.parametrize("k,num_points,code,text", [
    (9, 2, SB_EUNSUPPORTED, b"streams, the limit is 8"),
    (1, 2048, SB_EUNSUPPORTED, b"2048 points, the limit is 1024"),
    (5, 16, SB_EUNSUPPORTED, b"1048576 candidate vectors"),
    (0, 4, SB_EINVAL, b"bad arguments"),
    (2, 12, SB_EINVAL, b"power-of-two"),
])
def test_limits_and_malformed_arguments(sb_lib, k, num_points, code, text):
    assert _mimo_ml(sb_lib, k, num_points) == code
    assert text in sb_lib.sb_last_error()


def test_malformed_flags(sb_lib):
    assert _mimo_ml(sb_lib, 2, 4, method=2) == SB_EINVAL
    assert _mimo_ml(sb_lib, 2, 4, output=-1) == SB_EINVAL
    assert _mimo_ml(sb_lib, 2, 4, hard_out=3) == SB_EINVAL


def test_ofdm_limits(sb_lib):
    rc = sb_lib.sb_ofdm_ml(*([None] * 14), 0, 1, 1, 4, 3, 3, 12, 3, 0, 24, 256, 0, 0, 0, None)
    assert rc == SB_EUNSUPPORTED and b"candidate vectors" in sb_lib.sb_last_error()


def test_workspace_size(sb_lib):
    for k in (1, 4, 8):
        assert sb_lib.sb_ml_workspace_bytes(1000, k) == 1000 * 8 * (k * k + 2 * k + 1)
    assert sb_lib.sb_ml_workspace_bytes(1000, 9) == 0
    assert sb_lib.sb_ml_workspace_bytes(0, 2) == 0
