"""ctypes binding of libsionna_b200.so (the C-ABI declared in include/sionna_b200.h).

The library is built in-tree by ``sionna_b200.csrc.build`` (called from ``__graft_entry__.build()``).
Loading fails loudly if it is missing: there is no Python / CPU fallback for any kernel.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SIONNA_B200_LIB selects another build of the same sources (A/B experiments of kernel variants)
LIB_PATH = os.environ.get("SIONNA_B200_LIB") or os.path.join(_HERE, "libsionna_b200.so")
_lib = None

i32, i64, u64, f32, vp, sz = C.c_int32, C.c_int64, C.c_uint64, C.c_float, C.c_void_p, C.c_size_t
P_i32 = C.POINTER(C.c_int32)

# name -> (restype, argtypes); every symbol include/sionna_b200.h declares must be listed here
# (tests/test_cabi.py checks header <-> table <-> library agree).
SIGNATURES = {
    "sb_last_error": (C.c_char_p, []),
    "sb_device_info": (i32, [P_i32, P_i32, P_i32, P_i32]),
    "sb_version": (i32, []),
    "sb_launch_count": (i64, []),
    "sb_ldpc_graph_create": (i32, [C.POINTER(vp), i32, i32, i32, vp, vp, vp, i32, vp, i32, vp, i32, i32]),
    "sb_ldpc_graph_create_ordered": (i32, [C.POINTER(vp), i32, i32, i32, vp, vp, vp, i32, vp, i32, vp, i32, i32, vp]),
    "sb_ldpc_graph_destroy": (None, [vp]),
    "sb_ldpc_graph_set_qc": (i32, [vp, i32, i32, vp, vp, vp]),
    "sb_ldpc_graph_is_qc": (i32, [vp]),
    "sb_ldpc_graph_qc_opening": (i32, [vp]),
    "sb_debug_phi": (i32, [vp, vp, vp, i64, vp]),
    "sb_ldpc_graph_on_chip": (i32, [vp]),
    "sb_ldpc_workspace_bytes": (sz, [vp]),
    "sb_ldpc_decode": (i32, [vp, vp, i64, i32, i32, i32, f32, f32, i32, vp, vp, vp, vp, sz, vp]),
    "sb_ldpc_decode_early": (i32, [vp, vp, i64, i32, i32, f32, f32, i32, vp, vp, vp]),
    "sb_ldpc_flat_init": (i32, [vp, vp, vp, vp, vp, i64, i32, i32, vp]),
    "sb_ldpc_flat_cn": (i32, [vp, vp, vp, vp, vp, i32, i64, i32, f32, f32, vp]),
    "sb_ldpc_flat_vn": (i32, [vp, vp, vp, vp, vp, vp, i32, i64, i32, f32, vp]),
    "sb_ldpc_flat_out": (i32, [vp, vp, vp, vp, vp, i64, i32, i32, i32, vp]),
    "sb_ldpc_graph_export": (i32, [vp, vp, vp, vp, vp, vp, vp, vp]),
    "sb_ldpc5g_encoder_create": (i32, [C.POINTER(vp), i32, i32, i32, i32, i32] + [vp] * 9),
    "sb_ldpc5g_encoder_destroy": (None, [vp]),
    "sb_ldpc5g_encode": (i32, [vp, vp, i64, vp, vp]),
    "sb_binary_source": (i32, [vp, i64, u64, u64, vp]),
    "sb_normal": (i32, [vp, i64, f32, f32, u64, u64, vp]),
    "sb_qam_map": (i32, [vp, vp, i32, vp, vp, i64, vp]),
    "sb_demap": (i32, [vp, vp, i64, vp, i32, i32, vp, i64, vp, i64, i32, vp]),
    "sb_demap_qam": (i32, [vp, vp, i64, vp, vp, i32, i32, vp, i64, i32, vp]),
    "sb_symbol_demap": (i32, [vp, vp, i64, vp, i32, vp, i64, vp, i64, i32, vp]),
    "sb_awgn": (i32, [vp, vp, i64, vp, i64, u64, u64, vp]),
    "sb_count_errors": (i32, [vp, vp, i64, i32, vp, vp]),
    "sb_crc_encode": (i32, [vp, vp, i32, i32, vp, i64, vp]),
    "sb_crc_check": (i32, [vp, vp, i32, i32, vp, vp, i64, vp]),
    "sb_scramble": (i32, [vp, vp, i32, vp, i64, i32, i32, vp]),
    "sb_ofdm_modulate": (i32, [vp, vp, i64, i32, i32, vp, vp, i32, i32, vp]),
    "sb_ofdm_demodulate": (i32, [vp, vp, i64, i32, i32, vp, vp, i32, i32, i32, vp]),
    "sb_gather_rows": (i32, [vp, vp, vp, i64, i32, i32, i32, i32, i32, vp]),
    "sb_rg_map": (i32, [vp, vp, vp, vp, i64, i32, i32, i32, i32, vp]),
    "sb_ls_at_pilots": (i32, [vp, vp, vp, vp, i64, vp, vp, i64, i32, i32, i32, vp]),
    "sb_interp_lin": (i32, [vp] * 8 + [i32, vp, i64, i32, i32, i32, i32, i32, vp]),
    "sb_apply_ofdm_channel": (i32, [vp, vp, vp, i64, vp, i64, i32, i32, i32, i32, u64, u64, vp]),
    "sb_apply_time_channel": (i32, [vp, vp, vp, i64, vp, i64, i32, i32, i32, i32, i32, u64, u64, vp]),
    "sb_uniform": (i32, [vp, i64, f32, f32, u64, u64, vp]),
    "sb_tdl_sos": (i32, [vp, vp, vp, vp, vp, f32, f32, vp, i64, i32, i32, i32, i32, f32, vp]),
    "sb_cdl_coefficients": (i32, [vp] * 15 + [f32, f32, vp, i64, i32, i32, i32, i32, f32, vp]),
    "sb_phase_table": (i32, [vp, vp, f32, i32, vp, i64, i32, i32, vp]),
    "sb_cir_gram": (i32, [vp, vp, i64, i32, i32, vp]),
    "sb_cir_link_scale": (i32, [vp, vp, i64, vp, i64, i32, i32, i32, i32, i32, i32, f32, vp]),
    "sb_cir_apply": (i32, [vp, vp, i64, vp, vp, i64, i32, i32, i32, i32, i32, i32, i32, vp]),
    "sb_spatial_corr": (i32, [vp, vp, vp, i64, i32, i64, vp]),
    "sb_flat_fading": (i32, [vp, i64, u64, u64, vp, i64, vp, i64, i32, vp, vp, i64, vp, i64, u64, u64, vp, i64, i32, i32, vp]),
    "sb_chol_lower": (i32, [vp, vp, i64, i32, vp]),
    "sb_pusch_precode": (i32, [vp, vp, vp, i64, i32, i32, i32, i64, vp]),
    "sb_pusch_ls_combine": (i32, [vp, vp, i64, i32, i32, i32, i32, vp]),
    "sb_lmmse_equalize": (i32, [vp, vp, vp, vp, vp, i64, i32, i32, vp]),
    "sb_mimo_linalg": (i32, [i32, vp, vp, vp, vp, vp, i64, i32, i32, vp]),
    "sb_ofdm_frontend": (i32, [vp] * 15 + [i64] + [i32] * 11 + [vp]),
    "sb_ofdm_lmmse": (i32, [vp] * 12 + [i64] + [i32] * 8 + [vp]),
    "sb_ofdm_equalize": (i32, [i32] + [vp] * 12 + [i64] + [i32] * 8 + [vp]),
    "sb_mimo_ml": (i32, [vp] * 7 + [sz, i64] + [i32] * 6 + [vp]),
    "sb_ml_workspace_bytes": (sz, [i64, i32]),
    "sb_ofdm_ml": (i32, [vp] * 14 + [sz, i64] + [i32] * 12 + [vp]),
    "sb_mimo_kbest": (i32, [vp] * 6 + [sz, i64] + [i32] * 7 + [f32, vp]),
    "sb_kbest_workspace_bytes": (sz, [i64, i32, i32]),
    "sb_ofdm_kbest": (i32, [vp] * 13 + [sz, i64] + [i32] * 13 + [f32, vp]),
    "sb_mimo_ep": (i32, [vp] * 5 + [i64] + [i32] * 4 + [f32, i32, i32, vp]),
    "sb_ofdm_ep": (i32, [vp] * 12 + [i64] + [i32] * 10 + [f32, i32, i32, vp]),
    "sb_mimo_mmse_pic": (i32, [vp] * 6 + [i64] + [i32] * 6 + [vp]),
    "sb_ofdm_mmse_pic": (i32, [vp] * 13 + [i64] + [i32] * 12 + [vp]),
    "sb_mimo_precode": (i32, [vp, vp, i64, vp, vp, vp, i64, i32, i32, i32, vp]),
    "sb_ofdm_precode": (i32, [vp] * 11 + [i64] + [i32] * 9 + [vp]),
    "sb_conv_encode": (i32, [vp, vp, i64, i32, vp, i32, i32, i32, i32, vp]),
    "sb_viterbi_decode": (i32, [vp, vp, i64, i32, i32, i32, i32, i32, vp, vp, vp, i32, i32, vp, sz, vp]),
    "sb_viterbi_workspace_bytes": (sz, [i64, i32, i32]),
    "sb_bcjr_decode": (i32, [vp, vp, vp, i64, i32, i32, i32, i32, i32, vp, vp, vp, i32, i32, vp, sz, vp]),
    "sb_bcjr_workspace_bytes": (sz, [i64, i32, i32]),
    "sb_turbo_perm_create": (i32, [C.POINTER(vp), vp, i32]),
    "sb_turbo_perm_destroy": (None, [vp]),
    "sb_turbo_decode": (i32, [vp, vp, vp, i64, i32, i32, i32, i32, i32, vp, vp, vp, i32, i32, vp, sz, vp]),
    "sb_turbo_workspace_bytes": (sz, [i64, i32, i32, i32]),
    "sb_gf2_encode": (i32, [vp, vp, i32, i64, i32, i32, vp, vp]),
    "sb_osd_code_create": (i32, [C.POINTER(vp), vp, i32, i32]),
    "sb_osd_code_destroy": (None, [vp]),
    "sb_osd_decode": (i32, [vp, vp, vp, i64, i32, vp]),
}


# status codes of include/sionna_b200.h that the host layer tells apart
SB_EUNSUPPORTED = -4


class SbError(RuntimeError):
    """Raised when a C-ABI call returns a non-zero status."""


class SbUnsupportedError(SbError, ValueError):
    """SB_EUNSUPPORTED: a shape or configuration beyond a kernel's documented limits (also a ValueError, the type the
    reference raises for arguments it does not accept)."""


def lib():
    """Load (once) and return the ctypes handle. Raises if the library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -m sionna_b200.csrc.build` "
                "(or __graft_entry__.build()). sionna_b200 has no fallback path without its CUDA library.")
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def check(status, what=""):
    if status != 0:
        msg = lib().sb_last_error().decode("utf-8", "replace")
        err = SbUnsupportedError if status == SB_EUNSUPPORTED else SbError
        raise err(f"{what} failed with status {status}: {msg}")


class Handle:
    """Owns one C-ABI handle of type ``sb_<kind>``: created by ``sb_<kind>_create(&h, *args)`` (or by the constructor
    named ``create``) and destroyed once, by ``sb_<kind>_destroy``, when the owner is collected."""

    def __init__(self, kind, *args, create=None):
        name = create or f"sb_{kind}_create"
        h = C.c_void_p()
        check(getattr(lib(), name)(C.byref(h), *args), name)
        self.handle = h
        self._destroy = getattr(lib(), f"sb_{kind}_destroy")

    def __del__(self):
        destroy, self._destroy = getattr(self, "_destroy", None), None
        if destroy is not None:
            try:
                destroy(self.handle)
            except Exception:  # interpreter shutdown
                pass


def ptr(t):
    """Device (or host) pointer of a torch tensor / numpy array as c_void_p; None -> NULL."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return C.c_void_p(t.data_ptr())
    return C.c_void_p(t.ctypes.data)


def current_stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
