"""Argument checks of sb_mimo_kbest / sb_ofdm_kbest that run before any device access (no GPU needed): malformed
arguments are SB_EINVAL, configurations beyond the kernels' limits SB_EUNSUPPORTED with a message, a missing or short
workspace SB_ENOMEM."""
import math

import pytest

SB_EINVAL, SB_ENOMEM, SB_EUNSUPPORTED = -1, -3, -4


def _mimo(lib, K=2, num_points=16, k=16, real_rep=0, output=0, hard_out=0, clip=20.0, M=4, ws=None, ws_bytes=0,
          num=1):
    return lib.sb_mimo_kbest(None, None, None, None, None, ws, ws_bytes, num, M, K, num_points, k, real_rep, output,
                             hard_out, clip, None)


@pytest.mark.parametrize("args,text", [
    (dict(K=17, M=17), b"17 streams are 17 layers, the limit is 16"),
    (dict(K=9, M=9, real_rep=1), b"9 streams are 18 layers, the limit is 16"),
    (dict(k=257), b"k = 257 paths, the limit is 256"),
    (dict(K=1, num_points=512, k=1), b"512 points, the limit is 256"),
    (dict(K=1, num_points=1 << 18, k=1, real_rep=1), b"512 points, the limit is 256"),
    (dict(num_points=256, k=128), b"32768 children per layer, the limit is 16384"),
])
def test_limits(sb_lib, args, text):
    assert _mimo(sb_lib, **args) == SB_EUNSUPPORTED
    assert text in sb_lib.sb_last_error()


def test_largest_supported_shapes_pass_the_checks(sb_lib):
    # k = 64 with 256-QAM (the reference's largest unit-test shape) and 16 layers reach the launch; num = 0: no launch
    assert _mimo(sb_lib, K=3, num_points=256, k=64, M=7, num=0) == 0
    assert _mimo(sb_lib, K=16, num_points=4, k=256, M=16, num=0) == 0
    assert _mimo(sb_lib, K=8, num_points=256, k=256, M=8, real_rep=1, num=0) == 0


@pytest.mark.parametrize("args,text", [
    (dict(K=0), b"bad arguments"),
    (dict(M=1), b"M >= K"),
    (dict(k=0), b"k >= 1"),
    (dict(num_points=12), b"power-of-two"),
    (dict(num_points=1), b"power-of-two"),
    (dict(real_rep=2), b"{0, 1}"),
    (dict(output=-1), b"{0, 1}"),
    (dict(hard_out=3), b"{0, 1}"),
    (dict(clip=-1.0), b"llr_clip >= 0"),
    (dict(clip=math.nan), b"llr_clip >= 0"),
    (dict(num_points=8, real_rep=1), b"even number of bits"),
    (dict(output=1, hard_out=0), b"needs hard_out = 1"),
])
def test_malformed_arguments(sb_lib, args, text):
    assert _mimo(sb_lib, **args) == SB_EINVAL
    assert text in sb_lib.sb_last_error()


def test_infinite_clip_is_accepted(sb_lib):
    assert _mimo(sb_lib, clip=math.inf, num=0) == 0


def test_short_workspace(sb_lib):
    # pointers are checked before the workspace: give non-null dummies (nothing is launched on SB_ENOMEM)
    import ctypes
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    rc = sb_lib.sb_mimo_kbest(p, p, p, p, p, p, 8, 10, 4, 2, 16, 16, 0, 0, 0, 20.0, None)
    assert rc == SB_ENOMEM and b"sb_kbest_workspace_bytes" in sb_lib.sb_last_error()
    rc = sb_lib.sb_mimo_kbest(p, p, p, p, p, None, 0, 10, 4, 2, 16, 16, 0, 0, 0, 20.0, None)
    assert rc == SB_ENOMEM


def test_ofdm_checks(sb_lib):
    base = dict(batch=0, num_rx=1, ant=4, txs=4, syms=3, sc=12, spr=4, ku=0, nd=24, npts=16, k=64, rr=0, out=0, hard=0)

    def call(**kw):
        a = dict(base, **kw)
        return sb_lib.sb_ofdm_kbest(*([None] * 13), 0, a["batch"], a["num_rx"], a["ant"], a["txs"], a["syms"], a["sc"],
                                    a["spr"], a["ku"], a["nd"], a["npts"], a["k"], a["rr"], a["out"], a["hard"], 20.0,
                                    None)
    assert call() == 0
    assert call(ant=3) == SB_EINVAL and b"M >= K" in sb_lib.sb_last_error()
    assert call(k=512) == SB_EUNSUPPORTED and b"the limit is 256" in sb_lib.sb_last_error()
    assert call(spr=9, ant=9, txs=9, rr=1) == SB_EUNSUPPORTED and b"18 layers" in sb_lib.sb_last_error()
    assert call(batch=1) == SB_EINVAL                       # null pointers with a non-empty batch


def test_workspace_size(sb_lib):
    for K, rr in ((1, 0), (4, 0), (16, 0), (2, 1), (8, 1)):
        S = K << rr
        assert sb_lib.sb_kbest_workspace_bytes(1000, K, rr) == 1000 * (8 * (S * S + S + 1) + 8 * K + 4 * S)
    assert sb_lib.sb_kbest_workspace_bytes(1000, 17, 0) == 0
    assert sb_lib.sb_kbest_workspace_bytes(1000, 9, 1) == 0
    assert sb_lib.sb_kbest_workspace_bytes(1000, 2, 2) == 0
    assert sb_lib.sb_kbest_workspace_bytes(0, 2, 0) == 0
