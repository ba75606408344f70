"""Argument checks of sb_turbo_perm_create / sb_turbo_decode / sb_turbo_workspace_bytes that run before any device
access (no GPU needed): malformed arguments and non-permutations are SB_EINVAL, codes beyond the kernel's limits
SB_EUNSUPPORTED with a message, a missing or short workspace SB_ENOMEM."""
import ctypes as C

import numpy as np
import pytest

from oracle import conv as O

SB_EINVAL, SB_ENOMEM, SB_EUNSUPPORTED = -1, -3, -4


def _p(a):
    return None if a is None else a.ctypes.data


def _tables(g):
    t = O.trellis(g, rsc=True)
    return tuple(np.ascontiguousarray(t[n], np.int32) for n in ("from_nodes", "op_by_tonode", "ip_by_tonode"))


def _create(lib, perm, k=None):
    h = C.c_void_p()
    p = None if perm is None else np.ascontiguousarray(perm, np.int32)
    rc = lib.sb_turbo_perm_create(C.byref(h), _p(p), len(p) if k is None else k)
    return rc, h


@pytest.fixture
def perm40(sb_lib):
    rc, h = _create(sb_lib, np.random.default_rng(0).permutation(40))
    assert rc == 0
    yield h
    sb_lib.sb_turbo_perm_destroy(h)


def _decode(lib, perm, batch=0, k=40, num_iter=6, alg=0, terminate=1, hard=1, g=("1011", "1101"), tables=None,
            ns=None, conv_n=2, ws=None, ws_bytes=0, ptrs=(None, None)):
    fr, op, ip = tables or _tables(g)
    ns = ns or 2 ** (len(g[0]) - 1)
    return lib.sb_turbo_decode(ptrs[0], perm, ptrs[1], batch, k, num_iter, alg, terminate, hard, _p(fr), _p(op),
                               _p(ip), ns, conv_n, ws, ws_bytes, None)


def test_perm_create_rejects_non_permutations(sb_lib):
    assert _create(sb_lib, np.arange(10))[0] == 0
    sb_lib.sb_turbo_perm_destroy(_create(sb_lib, np.arange(10))[1])
    for bad, what in (([0, 1, 1, 3], b"appears twice"), ([0, 1, 2, 4], b"outside"), ([0, -1, 2, 3], b"outside"),
                      ([3, 2, 1, 7], b"outside")):
        rc, _ = _create(sb_lib, np.array(bad))
        assert rc == SB_EINVAL and what in sb_lib.sb_last_error(), bad
    h = C.c_void_p()
    assert sb_lib.sb_turbo_perm_create(C.byref(h), None, 4) == SB_EINVAL
    assert sb_lib.sb_turbo_perm_create(None, _p(np.arange(4, dtype=np.int32)), 4) == SB_EINVAL
    assert sb_lib.sb_turbo_perm_create(C.byref(h), _p(np.arange(4, dtype=np.int32)), 0) == SB_EINVAL
    sb_lib.sb_turbo_perm_destroy(None)


def test_decode_errors(sb_lib, perm40):
    assert _decode(sb_lib, perm40) == 0                                     # empty batch
    for kw in (dict(k=0), dict(num_iter=-1), dict(alg=3), dict(terminate=2), dict(hard=-1), dict(batch=-1)):
        assert _decode(sb_lib, perm40, **kw) == SB_EINVAL, kw
    assert _decode(sb_lib, None) == SB_EINVAL and b"interleaver" in sb_lib.sb_last_error()
    assert _decode(sb_lib, perm40, k=41) == SB_EINVAL and b"interleaver" in sb_lib.sb_last_error()
    fr, op, ip = _tables(("1011", "1101"))
    bad = fr.copy()
    bad[0] = bad[1]
    assert _decode(sb_lib, perm40, tables=(bad, op, ip)) == SB_EINVAL
    assert _decode(sb_lib, perm40, ns=6) == SB_EINVAL
    assert _decode(sb_lib, perm40, batch=1) == SB_EINVAL and b"null pointer" in sb_lib.sb_last_error()


def test_decode_limits(sb_lib, perm40):
    rc = _decode(sb_lib, perm40, g=("1" * 10, "1" + "0" * 9), ns=512)
    assert rc == SB_EUNSUPPORTED and b"256 states" in sb_lib.sb_last_error()
    rc = _decode(sb_lib, perm40, g=("1011", "1101", "1111"), conv_n=3)
    assert rc == SB_EUNSUPPORTED and b"rate 1/2" in sb_lib.sb_last_error()


def test_workspace(sb_lib, perm40):
    ws = sb_lib.sb_turbo_workspace_bytes
    assert ws(10000, 40, 1, 8) == 0                                        # alpha and extrinsic on chip
    assert ws(1000, 6144, 1, 8) == 1008 * (6147 * 8 + 6144) * 4          # both in the workspace (16 codewords per CTA)
    assert ws(10, 512, 1, 8) == 16 * 515 * 8 * 4                          # alpha off chip, extrinsic on chip
    assert ws(5, 4096, 0, 256) == 8 * (4096 * 256 + 4096) * 4         # two CTAs of 4 codewords
    assert ws(5, 40, 0, 3) == 0 and ws(5, 0, 0, 8) == 0 and ws(5, 40, 2, 8) == 0
    dummy = C.c_void_p(16)
    y, o = C.c_void_p(8), C.c_void_p(8)
    rc, h = _create(sb_lib, np.arange(512))
    assert rc == 0
    try:
        assert _decode(sb_lib, h, batch=10, k=512, ptrs=(y, o)) == SB_ENOMEM
        assert b"sb_turbo_workspace_bytes" in sb_lib.sb_last_error()
        assert _decode(sb_lib, h, batch=10, k=512, ptrs=(y, o), ws=dummy, ws_bytes=ws(10, 512, 1, 8) - 4) == SB_ENOMEM
    finally:
        sb_lib.sb_turbo_perm_destroy(h)
