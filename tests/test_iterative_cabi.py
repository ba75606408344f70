"""Argument checks of sb_mimo_ep / sb_ofdm_ep / sb_mimo_mmse_pic / sb_ofdm_mmse_pic that run before any device access
(no GPU needed): malformed arguments are SB_EINVAL, configurations beyond the kernels' limits SB_EUNSUPPORTED with a
message. The detectors need no workspace."""
import math

import pytest

SB_EINVAL, SB_EUNSUPPORTED = -1, -4


def _ep(lib, M=4, K=2, num_points=16, l=10, beta=0.9, output=0, hard_out=0, num=0):
    return lib.sb_mimo_ep(None, None, None, None, None, num, M, K, num_points, l, beta, output, hard_out, None)


def _pic(lib, M=4, K=2, num_points=16, num_iter=1, method=1, hard_out=0, num=0):
    return lib.sb_mimo_mmse_pic(None, None, None, None, None, None, num, M, K, num_points, num_iter, method, hard_out,
                                None)


@pytest.mark.parametrize("args,text", [
    (dict(K=17, M=17), b"17 streams, the limit is 16"),
    (dict(num_points=1024), b"1024 points, the limit is 256"),
])
def test_ep_limits(sb_lib, args, text):
    assert _ep(sb_lib, **args) == SB_EUNSUPPORTED
    assert text in sb_lib.sb_last_error()


@pytest.mark.parametrize("args,text", [
    (dict(K=0), b"bad arguments"),
    (dict(M=0), b"M >= 1"),
    (dict(num_points=12), b"power-of-two"),
    (dict(num_points=8), b"even number of bits"),
    (dict(l=0), b"l >= 1"),
    (dict(beta=1.5), b"0 <= beta <= 1"),
    (dict(beta=math.nan), b"0 <= beta <= 1"),
    (dict(output=2), b"output in {0, 1}"),
    (dict(hard_out=2), b"hard_out in {0, 1}"),
])
def test_ep_malformed_arguments(sb_lib, args, text):
    assert _ep(sb_lib, **args) == SB_EINVAL
    assert text in sb_lib.sb_last_error()


@pytest.mark.parametrize("args,text", [
    (dict(K=17, M=17), b"17 streams, the limit is 16"),
    (dict(num_points=2048), b"2048 points, the limit is 1024"),
])
def test_pic_limits(sb_lib, args, text):
    assert _pic(sb_lib, **args) == SB_EUNSUPPORTED
    assert text in sb_lib.sb_last_error()


@pytest.mark.parametrize("args,text", [
    (dict(K=0), b"bad arguments"),
    (dict(num_points=1), b"power-of-two"),
    (dict(num_iter=0), b"num_iter >= 1"),
    (dict(method=2), b"method in {0, 1}"),
    (dict(hard_out=-1), b"hard_out in {0, 1}"),
])
def test_pic_malformed_arguments(sb_lib, args, text):
    assert _pic(sb_lib, **args) == SB_EINVAL
    assert text in sb_lib.sb_last_error()


def test_largest_supported_shapes_pass_the_checks(sb_lib):
    # num = 0: no launch; M < K is accepted
    assert _ep(sb_lib, K=16, M=16, num_points=256) == 0
    assert _ep(sb_lib, K=4, M=2) == 0
    assert _pic(sb_lib, K=16, M=16, num_points=1024) == 0
    assert _pic(sb_lib, K=4, M=3, num_points=2) == 0


def test_null_pointers_with_a_non_empty_batch(sb_lib):
    assert _ep(sb_lib, num=1) == SB_EINVAL
    assert _pic(sb_lib, num=1) == SB_EINVAL


def test_scratch_beyond_shared_memory(sb_lib):
    # 160 antennas: 8 (M^2 + ...) bytes of whitening scratch per problem exceed 200 KB; rejected before any access
    import ctypes
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert sb_lib.sb_mimo_ep(p, p, p, p, p, 1, 160, 2, 16, 10, 0.9, 0, 0, None) == SB_EUNSUPPORTED
    assert b"shared-memory scratch" in sb_lib.sb_last_error()
    assert sb_lib.sb_mimo_mmse_pic(p, p, p, p, p, p, 1, 160, 2, 16, 1, 1, 0, None) == SB_EUNSUPPORTED
    assert b"shared-memory scratch" in sb_lib.sb_last_error()


def test_ofdm_checks(sb_lib):
    base = dict(batch=0, num_rx=1, ant=4, txs=4, syms=3, sc=12, spr=4, ku=0, nd=24, npts=16)

    def ep(**kw):
        a = dict(base, **kw)
        return sb_lib.sb_ofdm_ep(*([None] * 12), a["batch"], a["num_rx"], a["ant"], a["txs"], a["syms"], a["sc"],
                                 a["spr"], a["ku"], a["nd"], a["npts"], 10, 0.9, 0, 0, None)

    def pic(**kw):
        a = dict(base, **kw)
        return sb_lib.sb_ofdm_mmse_pic(*([None] * 13), a["batch"], a["num_rx"], a["ant"], a["txs"], a["syms"],
                                       a["sc"], a["spr"], a["ku"], a["nd"], a["npts"], 1, 1, 0, None)
    assert ep() == 0 and pic() == 0
    assert ep(spr=17, txs=17) == SB_EUNSUPPORTED and b"17 streams" in sb_lib.sb_last_error()
    assert pic(npts=4096) == SB_EUNSUPPORTED and b"the limit is 1024" in sb_lib.sb_last_error()
    assert ep(batch=1) == SB_EINVAL and pic(batch=1) == SB_EINVAL
