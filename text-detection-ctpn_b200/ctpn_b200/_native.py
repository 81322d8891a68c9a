"""ctypes binding of libctpn_b200.so (the C ABI declared in include/ctpn_b200.h).

There is no CPU fallback: if the shared library is missing, importing this module
raises, and every call checks the status code and raises ``CtpnError`` with the
library's own message.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libctpn_b200.so")
# CTPN_B200_LIB=dbg (tests only): the -DCTPN_DEBUG build with the SIMT reference kernels, the hardware probes and the
# ablation / tuning environment switches (tests/_native/libctpn_b200_dbg.so, csrc/testing/ctpn_b200_testing.h)
DEBUG_LIB = os.environ.get("CTPN_B200_LIB", "") == "dbg"
if DEBUG_LIB:
    LIB_PATH = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "tests", "_native", "libctpn_b200_dbg.so")


class CtpnError(RuntimeError):
    pass


ERR_INVALID, ERR_CUDA, ERR_WORKSPACE, ERR_NO_DEVICE = 1, 2, 3, 4     # include/ctpn_b200.h


if not os.path.exists(LIB_PATH):
    raise ImportError(
        "libctpn_b200.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'` "
        "or `make -C text-detection-ctpn_b200/csrc`. There is no CPU fallback." % LIB_PATH)

lib = C.CDLL(LIB_PATH)

_p = C.c_void_p
_i = C.c_int
_f = C.c_float
_z = C.c_size_t

# name -> (restype, argtypes); must list every symbol include/ctpn_b200.h declares
SIGNATURES = {
    "ctpn_version": (_i, []),
    "ctpn_last_error": (C.c_char_p, []),
    "ctpn_device_ok": (_i, [_i]),
    "ctpn_prof_enable": (_i, [_i]),
    "ctpn_prof_report": (_i, [_p, _z, C.POINTER(_z)]),
    "ctpn_crc32c_host": (C.c_uint32, [_p, _z, C.c_uint32]),
    "ctpn_nms_host": (_i, [_p, _p, _p, _i, _i, _f, _i]),
    "ctpn_text_lines_host": (_i, [_p, _p, _i, _i, _i, _i, _p, _p, _i, _p]),
    "ctpn_text_lines_workspace_bytes": (_z, [_i, _i, _i]),
    "ctpn_text_lines": (_i, [_p, _p, _i, _i, _p, _p, _i, _p, _p, _p, _p, _p, _z, _p]),
    "ctpn_text_filter_nms_host": (_i, [_p, _p, _i, _p, _p, _p]),
    "ctpn_text_groups_host": (_i, [_p, _p, _i, _i, _p, _p, _p, _i, _p, _p]),
    "ctpn_bbox_overlaps_host": (_i, [_p, _i, _i, _p, _i, _i, _p]),
    "ctpn_bbox_intersections_host": (_i, [_p, _i, _i, _p, _i, _i, _p]),
    "ctpn_anchor_targets_host": (_i, [_p, _i, _i, _p, _p, _i, _i, _i, _i, C.c_double, C.c_double, _p, _p, _p]),
    "ctpn_resize_out_size": (_i, [_i, _i, C.c_double, C.c_double, _p, _p]),
    "ctpn_resize_linear_u8": (_i, [_p, _i, _i, _i, _i, C.c_double, C.c_double, _p, _i, _i, _p]),
    "ctpn_image_blob_f32": (_i, [_p, _p, _i, _i, _i, C.c_double, C.c_double, _p, _i, _i, _p]),
    "ctpn_resize_linear_u8_ragged": (_i, [_p, _z, _p, _p, _p, _p, _i, _i, _p, _i, _i, _p]),
    "ctpn_image_blob_f32_ragged": (_i, [_p, _z, _p, _p, _p, _p, _p, _i, _p, _i, _i, _p]),
    "ctpn_nms_workspace_bytes": (_z, [_i, _i]),
    "ctpn_nms_sorted": (_i, [_p, _p, _i, _i, _f, _i, _p, _p, _p, _z, _p]),
    "ctpn_proposals_workspace_bytes": (_z, [_i, _i, _i, _i]),
    "ctpn_proposals": (_i, [_p, _i, _p, _p, _i, _i, _i, _i, _i, _i, _f, _f, _i, _p, _p, _p, _p, _z, _p]),
    "ctpn_proposals_ragged": (_i, [_p, _i, _p, _p, _p, _i, _i, _i, _i, _i, _i, _f, _f, _i, _p, _p, _p, _p, _z, _p]),
    "ctpn_pack_weights": (_i, [_p, _i, _i, _i, _i, _i, _p, _p]),
    "ctpn_pack_weights_f16f8": (_i, [_p, _i, _i, _i, _i, _f, _f, _p, _p]),
    "ctpn_conv3x3_f16f8": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _f, _f, _f, _f, _p]),
    "ctpn_conv1_1_tc_f16f8": (_i, [_p, _i, _p, _p, _p, _p, _i, _i, _i, _f, _f, _p]),
    "ctpn_conv1_1_tc": (_i, [_p, _i, _p, _p, _p, _p, _i, _i, _i, _i, _p]),
    "ctpn_conv3x3": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "ctpn_bilstm_recurrent": (_i, [_p, _p, _p, _p, _i, _i, _i, _p]),
    "ctpn_net_create": (_i, [C.POINTER(_p), _i]),
    "ctpn_net_destroy": (_i, [_p]),
    "ctpn_net_set_option": (_i, [_p, C.c_char_p, _i]),
    "ctpn_net_set_weight": (_i, [_p, C.c_char_p, _p, _z]),
    "ctpn_net_workspace_bytes": (_z, [_p, _i, _i, _i]),
    "ctpn_net_forward": (_i, [_p, _p, _i, _i, _i, _i, _p, _p, _p, _z, _p]),
    "ctpn_net_forward_ragged": (_i, [_p, _p, _i, _p, _i, _i, _i, _p, _p, _p, _z, _p]),
    "ctpn_net_feature_hw": (_i, [_i, _i, C.POINTER(_i), C.POINTER(_i)]),
    "ctpn_net_debug_tap": (_i, [_p, C.c_char_p, _p, _z, C.POINTER(_z), _p]),
}

# test library only (csrc/testing/ctpn_b200_testing.h)
TESTING_SIGNATURES = {
    "ctpn_conv1_1": (_i, [_p, _i, _p, _p, _p, _p, _i, _i, _i, _i, _p]),
    "ctpn_conv3x3_simt": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "ctpn_probe_umma_view": (_i, [_p, _p, _i, _i, _i, _i, _p, _p]),
    "ctpn_net_f16f8_scales": (_i, [_p, _p, _p, _p]),
}

for _name, (_res, _args) in list(SIGNATURES.items()) + (list(TESTING_SIGNATURES.items()) if DEBUG_LIB else []):
    _fn = getattr(lib, _name)      # AttributeError here == header/library mismatch
    _fn.restype = _res
    _fn.argtypes = _args


def prof_report():
    """Parsed ctpn_prof_report(): list of {kernel, launches, ms, work}."""
    import json
    need = C.c_size_t()
    check(lib.ctpn_prof_report(None, 0, C.byref(need)), "ctpn_prof_report")
    buf = C.create_string_buffer(need.value)
    check(lib.ctpn_prof_report(buf, need.value, C.byref(need)), "ctpn_prof_report")
    return json.loads(buf.value.decode())


def last_error():
    return lib.ctpn_last_error().decode("utf-8", "replace")


def check(status, what=""):
    if status != 0:
        raise CtpnError("%s failed (status %d): %s" % (what or "ctpn call", status, last_error()))


def ptr(t):
    """Device/host pointer of a torch tensor or numpy array as c_void_p (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return C.c_void_p(t.data_ptr())
    return C.c_void_p(t.ctypes.data)


def stream_ptr(stream=None):
    import torch
    s = stream if stream is not None else torch.cuda.current_stream()
    return C.c_void_p(s.cuda_stream)
