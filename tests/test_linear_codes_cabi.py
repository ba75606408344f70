"""Argument checks of sb_gf2_encode / sb_osd_code_create / sb_osd_decode that run before any device access (no GPU
needed): malformed arguments, non-binary and rank-deficient generators are SB_EINVAL, shapes beyond the kernel's limits
SB_EUNSUPPORTED with a message, an empty batch SB_OK."""
import ctypes as C

import numpy as np

SB_EINVAL, SB_EUNSUPPORTED = -1, -4


def _create(lib, gm, k=None, n=None):
    h = C.c_void_p()
    g = np.ascontiguousarray(gm, np.uint8)
    rc = lib.sb_osd_code_create(C.byref(h), g.ctypes.data, g.shape[0] if k is None else k,
                                g.shape[1] if n is None else n)
    return rc, h


HAMMING = np.array([[1, 0, 0, 0, 1, 1, 0], [0, 1, 0, 0, 1, 0, 1], [0, 0, 1, 0, 0, 1, 1], [0, 0, 0, 1, 1, 1, 1]])


def test_gf2_encode_errors(sb_lib):
    enc = sb_lib.sb_gf2_encode
    assert enc(None, None, 0, 0, 4, 7, None, None) == 0                      # empty batch
    assert enc(None, None, 0, 5, 4, 7, None, None) == SB_EINVAL              # missing pointers
    assert b"missing" in sb_lib.sb_last_error()
    assert enc(None, None, 0, 0, 8, 7, None, None) == SB_EINVAL              # k > n
    assert enc(None, None, 0, 0, 0, 7, None, None) == SB_EINVAL
    assert enc(None, None, 0, -1, 4, 7, None, None) == SB_EINVAL
    assert enc(None, None, 4, 0, 4, 7, None, None) == SB_EINVAL              # dtype
    assert b"dtype" in sb_lib.sb_last_error()


def test_osd_code_create_errors(sb_lib):
    rc, h = _create(sb_lib, HAMMING)
    assert rc == 0
    sb_lib.sb_osd_code_destroy(h)
    sb_lib.sb_osd_code_destroy(None)
    bad = HAMMING.copy()
    bad[1, 2] = 2
    assert _create(sb_lib, bad)[0] == SB_EINVAL and b"not binary" in sb_lib.sb_last_error()
    deficient = np.concatenate([HAMMING[:3], (HAMMING[0] ^ HAMMING[1])[None]])
    assert _create(sb_lib, deficient)[0] == SB_EINVAL and b"full rank" in sb_lib.sb_last_error()
    assert _create(sb_lib, HAMMING, k=8, n=7)[0] == SB_EINVAL
    assert _create(sb_lib, HAMMING, k=0)[0] == SB_EINVAL
    h = C.c_void_p()
    assert sb_lib.sb_osd_code_create(C.byref(h), None, 4, 7) == SB_EINVAL
    assert sb_lib.sb_osd_code_create(None, HAMMING.astype(np.uint8).ctypes.data, 4, 7) == SB_EINVAL
    big = np.zeros((2, 1025), np.uint8)
    big[0, 0] = big[1, 1] = 1
    assert _create(sb_lib, big)[0] == SB_EUNSUPPORTED and b"1024" in sb_lib.sb_last_error()
    wide = np.zeros((2, 1024), np.uint8)
    wide[0, 0] = wide[1, 1] = 1
    rc, h = _create(sb_lib, wide)
    assert rc == 0
    sb_lib.sb_osd_code_destroy(h)


def test_osd_decode_errors(sb_lib):
    rc, h = _create(sb_lib, HAMMING)
    assert rc == 0
    dec = sb_lib.sb_osd_decode
    try:
        assert dec(h, None, None, 0, 2, None) == 0                           # empty batch
        assert dec(h, None, None, 0, 100, None) == 0                         # t > k acts as t = k
        assert dec(h, None, None, 3, 2, None) == SB_EINVAL and b"missing" in sb_lib.sb_last_error()
        assert dec(None, None, None, 0, 2, None) == SB_EINVAL
        assert dec(h, None, None, -1, 2, None) == SB_EINVAL
        assert dec(h, None, None, 0, -1, None) == SB_EINVAL
    finally:
        sb_lib.sb_osd_code_destroy(h)
    rng = np.random.default_rng(0)
    g = np.concatenate([np.eye(200, dtype=np.uint8), rng.integers(0, 2, (200, 300), dtype=np.uint8)], axis=1)
    rc, h = _create(sb_lib, g)
    assert rc == 0
    try:
        assert dec(h, None, None, 0, 9, None) == 0                           # C(200, <= 9) < 2^62
        assert dec(h, None, None, 0, 40, None) == SB_EUNSUPPORTED and b"2^62" in sb_lib.sb_last_error()
    finally:
        sb_lib.sb_osd_code_destroy(h)
