"""Argument checks of sb_conv_encode / sb_viterbi_decode / sb_bcjr_decode that run before any device access (no GPU
needed): malformed arguments are SB_EINVAL, codes beyond the kernels' limits SB_EUNSUPPORTED with a message, a missing
or short workspace SB_ENOMEM."""
import ctypes

import numpy as np
import pytest

from sionna_b200.phy.fec.conv import Trellis

SB_EINVAL, SB_ENOMEM, SB_EUNSUPPORTED = -1, -3, -4


def _tables(gen_poly, rsc=False):
    tr = Trellis(gen_poly, rsc=rsc)
    return [np.ascontiguousarray(t, np.int32) for t in (tr.from_nodes, tr.op_by_tonode, tr.ip_by_tonode)], tr.ns


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _viterbi(lib, gen_poly=("101", "111"), batch=0, num_syms=10, k=10, method=0, terminate=0, info=1, tables=None,
             ns=None, conv_n=None, ws=None, ws_bytes=0, ptrs=None):
    (fr, op, ip), ns0 = _tables(gen_poly) if tables is None else (tables, ns)
    y, o = ptrs or (None, None)
    return lib.sb_viterbi_decode(y, o, batch, num_syms, k, method, terminate, info, _p(fr), _p(op), _p(ip),
                                 ns0 if ns is None else ns, len(gen_poly) if conv_n is None else conv_n, ws, ws_bytes, None)


def _bcjr(lib, gen_poly=("101", "111"), batch=0, num_syms=10, num_out=10, alg=0, terminate=0, hard=0, tables=None,
          ns=None, conv_n=None, ws=None, ws_bytes=0, ptrs=None):
    (fr, op, ip), ns0 = _tables(gen_poly) if tables is None else (tables, ns)
    y, o = ptrs or (None, None)
    return lib.sb_bcjr_decode(y, None, o, batch, num_syms, num_out, alg, terminate, hard, _p(fr), _p(op), _p(ip),
                              ns0 if ns is None else ns, len(gen_poly) if conv_n is None else conv_n, ws, ws_bytes, None)


def _encode(lib, polys=(5, 7), batch=0, k=10, K=3, rsc=0, terminate=0):
    g = np.array(polys, np.int32)
    return lib.sb_conv_encode(None, None, batch, k, _p(g), len(polys), K, rsc, terminate, None)


def test_encoder_checks(sb_lib):
    assert _encode(sb_lib) == 0
    assert _encode(sb_lib, polys=[1] * 8, K=9) == 0
    for kw in (dict(k=0), dict(batch=-1), dict(K=1), dict(rsc=2), dict(terminate=-1)):
        assert _encode(sb_lib, **kw) == SB_EINVAL, kw
        assert b"bad arguments" in sb_lib.sb_last_error()
    assert _encode(sb_lib, polys=(9, 7)) == SB_EINVAL and b"more than 3 bits" in sb_lib.sb_last_error()
    assert _encode(sb_lib, polys=(3, 7), rsc=1) == SB_EINVAL and b"feedback polynomial" in sb_lib.sb_last_error()
    assert _encode(sb_lib, K=10, polys=(513, 700)) == SB_EUNSUPPORTED
    assert b"constraint length 10" in sb_lib.sb_last_error() and b"limits are 9" in sb_lib.sb_last_error()
    assert _encode(sb_lib, polys=[7] * 9) == SB_EUNSUPPORTED and b"9 output bits" in sb_lib.sb_last_error()


@pytest.mark.parametrize("run", [_viterbi, _bcjr])
def test_largest_supported_codes_pass_the_checks(sb_lib, run):
    assert run(sb_lib, gen_poly=("110101001", "101110111")) == 0                  # K = 9, 256 states
    assert run(sb_lib, gen_poly=("11",) * 8) == 0                                  # K = 2, conv_n = 8
    assert run(sb_lib, gen_poly=("101011011",) * 8, num_syms=1 << 20, **(
        dict(k=1 << 20) if run is _viterbi else dict(num_out=1 << 20))) == 0


@pytest.mark.parametrize("run", [_viterbi, _bcjr])
def test_limits(sb_lib, run):
    (fr, op, ip), ns = _tables(("1101011011", "1011101111"))                       # K = 10, 512 states
    assert run(sb_lib, tables=(fr, op, ip), ns=ns, conv_n=2) == SB_EUNSUPPORTED
    assert b"512 states" in sb_lib.sb_last_error() and b"constraint length 9" in sb_lib.sb_last_error()
    assert run(sb_lib, gen_poly=("101",) * 9) == SB_EUNSUPPORTED and b"9 output bits" in sb_lib.sb_last_error()
    assert run(sb_lib, gen_poly=("101",) * 8, num_syms=1 << 28, **(
        dict(k=1) if run is _viterbi else dict(num_out=1))) == SB_EUNSUPPORTED
    assert b"2^31 - 1" in sb_lib.sb_last_error()


@pytest.mark.parametrize("run", [_viterbi, _bcjr])
def test_malformed_trellis(sb_lib, run):
    (fr, op, ip), ns = _tables(("101", "111"))
    assert run(sb_lib, tables=(fr, op, ip), ns=3, conv_n=2) == SB_EINVAL
    assert b"power of two" in sb_lib.sb_last_error()
    assert run(sb_lib, tables=(fr, op, ip), ns=4, conv_n=0) == SB_EINVAL
    bad = fr.copy()
    bad[1, 0] = 0                                                                 # not a predecessor of state 1
    assert run(sb_lib, tables=(bad, op, ip), ns=4, conv_n=2) == SB_EINVAL
    assert b"not those of a rate-1/2 shift register" in sb_lib.sb_last_error()
    bad = op.copy()
    bad[0, 0] = 4
    assert run(sb_lib, tables=(fr, bad, ip), ns=4, conv_n=2) == SB_EINVAL
    bad = ip.copy()
    bad[2, 0] = 0                                                                 # two input-0 edges out of state 0
    assert run(sb_lib, tables=(fr, op, bad), ns=4, conv_n=2) == SB_EINVAL
    assert b"state 0 has two transitions for input 0" in sb_lib.sb_last_error()
    assert sb_lib.sb_viterbi_decode(None, None, 0, 10, 10, 0, 0, 1, None, None, None, 4, 2, None, 0, None) == SB_EINVAL
    assert b"missing trellis tables" in sb_lib.sb_last_error()


def test_malformed_arguments(sb_lib):
    for kw in (dict(method=2), dict(terminate=2), dict(info=-1), dict(k=0), dict(k=11), dict(num_syms=0),
               dict(batch=-1)):
        assert _viterbi(sb_lib, **kw) == SB_EINVAL, kw
        assert b"bad arguments" in sb_lib.sb_last_error()
    for kw in (dict(alg=3), dict(terminate=2), dict(hard=2), dict(num_out=0), dict(num_out=11), dict(num_syms=0)):
        assert _bcjr(sb_lib, **kw) == SB_EINVAL, kw
        assert b"bad arguments" in sb_lib.sb_last_error()
    assert _viterbi(sb_lib, batch=1) == SB_EINVAL and b"null pointer" in sb_lib.sb_last_error()
    assert _bcjr(sb_lib, batch=1) == SB_EINVAL and b"null pointer" in sb_lib.sb_last_error()


def test_workspace(sb_lib):
    # on chip: no workspace; off chip: whole CTAs of decisions (one bit per state and step) or of alpha (ns floats)
    assert sb_lib.sb_viterbi_workspace_bytes(10000, 64, 128) == 0
    assert sb_lib.sb_bcjr_workspace_bytes(100, 69, 16) == 0
    assert sb_lib.sb_viterbi_workspace_bytes(10, 4096, 128) == 12 * 4096 * 16
    assert sb_lib.sb_viterbi_workspace_bytes(10, 4096, 16) == 16 * 4096 * 4
    assert sb_lib.sb_bcjr_workspace_bytes(5, 71, 128) == 8 * 71 * 128 * 4
    assert sb_lib.sb_bcjr_workspace_bytes(5, 71, 3) == 0
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    g = ("11100101", "10011111")
    assert _viterbi(sb_lib, gen_poly=g, batch=10, num_syms=4096, k=4096, ptrs=(p, p)) == SB_ENOMEM
    assert b"sb_viterbi_workspace_bytes" in sb_lib.sb_last_error()
    assert _viterbi(sb_lib, gen_poly=g, batch=10, num_syms=4096, k=4096, ptrs=(p, p), ws=p, ws_bytes=64) == SB_ENOMEM
    assert _bcjr(sb_lib, gen_poly=g, batch=5, num_syms=71, num_out=64, ptrs=(p, p)) == SB_ENOMEM
    assert b"sb_bcjr_workspace_bytes" in sb_lib.sb_last_error()
