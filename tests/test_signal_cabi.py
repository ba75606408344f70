"""Argument checks of sb_convolve / sb_scale_last / sb_power_mean that run before any device access (no GPU needed):
every malformed argument is SB_EINVAL, an empty batch is SB_OK with NULL pointers, and the largest accepted shapes
pass the checks."""
SB_EINVAL, SB_ENOMEM = -1, -3
FAKE = 0x1000                    # never dereferenced: every call below fails its checks or has no rows


def test_convolve_errors(sb_lib):
    conv = sb_lib.sb_convolve

    def c(rows=0, n=10, k=3, offset=0, out_len=12, flags=0, precision=0, xc=0, hc=0, x=None, h=None, w=None, y=None):
        return conv(x, xc, h, hc, w, y, precision, rows, n, k, offset, out_len, flags, None)
    assert c() == 0                                                   # rows = 0: SB_OK with NULL pointers
    assert c(offset=1, out_len=10) == 0 and c(offset=2, out_len=8) == 0   # same, valid
    assert c(rows=4) == SB_EINVAL and b"missing" in sb_lib.sb_last_error()
    assert c(rows=4, x=FAKE, h=FAKE) == SB_EINVAL                     # no output
    assert c(rows=-1) == SB_EINVAL
    assert c(n=0, out_len=2) == SB_EINVAL and b"bad shape" in sb_lib.sb_last_error()
    assert c(k=0, out_len=9) == SB_EINVAL
    assert c(out_len=-1) == SB_EINVAL
    assert c(offset=-1) == SB_EINVAL and b"offset" in sb_lib.sb_last_error()
    assert c(offset=3, out_len=1) == SB_EINVAL                        # offset > k - 1
    assert c(out_len=13) == SB_EINVAL and b"out_len" in sb_lib.sb_last_error()
    assert c(offset=2, out_len=11) == SB_EINVAL                       # > n + k - 1 - offset
    assert c(flags=8) == SB_EINVAL and b"flag" in sb_lib.sb_last_error()
    assert c(flags=-1) == SB_EINVAL
    assert c(precision=2) == SB_EINVAL and b"precision" in sb_lib.sb_last_error()
    assert c(xc=2) == SB_EINVAL and c(hc=-1) == SB_EINVAL
    assert c(flags=1) == SB_EINVAL and b"window" in sb_lib.sb_last_error()
    assert c(flags=1, w=FAKE) == 0 and c(flags=7, w=FAKE, xc=1, hc=1, precision=1) == 0
    big = 2 ** 31 - 1                                                 # the largest shapes the checks accept
    assert c(n=big, k=1, out_len=big) == 0
    assert c(n=1, k=big, offset=big - 1, out_len=1) == 0
    assert c(n=2 ** 30, k=2 ** 30, offset=0, out_len=big) == 0
    assert c(rows=0, n=big, k=big, offset=(big - 1) // 2, out_len=big) == 0


def test_scale_last_errors(sb_lib):
    sc = sb_lib.sb_scale_last
    assert sc(None, 0, None, None, 0, 0, 16, 0, None) == 0
    assert sc(None, 1, None, None, 1, 0, 2 ** 31 - 1, 1, None) == 0
    assert sc(None, 0, None, None, 0, 3, 16, 0, None) == SB_EINVAL and b"missing" in sb_lib.sb_last_error()
    assert sc(FAKE, 0, FAKE, None, 0, 3, 16, 0, None) == SB_EINVAL
    assert sc(None, 0, None, None, 0, -1, 16, 0, None) == SB_EINVAL
    assert sc(None, 0, None, None, 0, 0, 0, 0, None) == SB_EINVAL
    assert sc(None, 0, None, None, 2, 0, 16, 0, None) == SB_EINVAL
    assert sc(None, 2, None, None, 0, 0, 16, 0, None) == SB_EINVAL
    assert sc(None, 0, None, None, 0, 0, 16, 2, None) == SB_EINVAL


def test_power_mean_errors(sb_lib):
    pm = sb_lib.sb_power_mean
    ws = sb_lib.sb_power_mean_workspace_bytes
    assert ws(1024, 64) == 0 and ws(1025, 64) == 2 * 64 * 4 and ws(10 ** 6, 64) == 977 * 64 * 4
    assert ws(0, 64) == 0 and ws(10, 0) == 0
    assert pm(None, None, 0, 64, None, 0, None) == SB_EINVAL          # nothing to average over
    assert pm(None, None, 4, 64, None, 0, None) == SB_EINVAL and b"missing" in sb_lib.sb_last_error()
    assert pm(FAKE, FAKE, 4, 0, None, 0, None) == SB_EINVAL
    assert pm(FAKE, FAKE, 2048, 64, None, 0, None) == SB_ENOMEM and b"workspace" in sb_lib.sb_last_error()
    assert pm(FAKE, FAKE, 2048, 64, FAKE, 100, None) == SB_ENOMEM
