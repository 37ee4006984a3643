"""ctypes binding of libsamroad_b200.so (C ABI declared in include/samroad_b200.h).

This is the whole "FFI": plain pointers and sizes.  torch is used by the callers only to own device
memory (`tensor.data_ptr()`) and streams.  There is no fallback: if the shared library is missing
or a call fails, a RuntimeError carrying `samroad_last_error()` is raised.
"""
from __future__ import annotations

import ctypes as C
import weakref
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libsamroad_b200.so"

F32, I64, I32, U8, F64 = 0, 1, 2, 3, 4
ABI_VERSION = 5
TOPO_NORMAL, TOPO_NO_OFFSET, TOPO_NO_TRANSFORMER = 0, 1, 2
LOSS_BCE, LOSS_FOCAL = 0, 1
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2


class SamRoadCfg(C.Structure):
    _fields_ = [
        ("patch_size", C.c_int32),
        ("embed_dim", C.c_int32),
        ("depth", C.c_int32),
        ("num_heads", C.c_int32),
        ("window_size", C.c_int32),
        ("global_attn_indexes", C.c_int32 * 4),
        ("use_sam_decoder", C.c_int32),
        ("toponet_version", C.c_int32),
        ("lora_rank", C.c_int32),
    ]


class SamroadEncoderTaps(C.Structure):
    _fields_ = [
        ("tokens0", C.c_void_p),
        ("block_mask", C.c_uint64),
        ("blocks", C.c_void_p),
        ("detail_block", C.c_int32),
        ("ln1", C.c_void_p),
        ("qkv", C.c_void_p),
        ("att", C.c_void_p),
        ("x_attn", C.c_void_p),
        ("ln2", C.c_void_p),
        ("h", C.c_void_p),
        ("n1", C.c_void_p),
        ("feat16", C.c_void_p),
        ("d1", C.c_void_p),
        ("d2", C.c_void_p),
    ]


class SamRoadTrainArgs(C.Structure):
    _fields_ = [
        ("B", C.c_int32),
        ("N", C.c_int32),
        ("Ns", C.c_int32),
        ("Np", C.c_int32),
        ("loss_kind", C.c_int32),
        ("dropout_p", C.c_float),
        ("seed", C.c_uint64),
    ]


class SamRoadLabelCfg(C.Structure):
    _fields_ = [
        ("patch_size", C.c_int32),
        ("image_size", C.c_int32),
        ("sample_margin", C.c_int32),
        ("topo_sample_num", C.c_int32),
        ("max_neighbor_queries", C.c_int32),
        ("max_patch_points", C.c_int32),
        ("road_nms_radius", C.c_double),
        ("neighbor_radius", C.c_double),
    ]


class SamRoadTopoCaps(C.Structure):
    _fields_ = [
        ("max_marbles", C.c_int32),
        ("max_queue", C.c_int32),
        ("max_covered", C.c_int32),
        ("max_candidates", C.c_int32),
        ("slots", C.c_int32),
    ]


class SamRoadAplsCaps(C.Structure):
    _fields_ = [
        ("max_nodes", C.c_int32),
        ("max_arcs", C.c_int32),
        ("max_control_points", C.c_int32),
    ]


class SamRoadAplsResult(C.Structure):
    _fields_ = [
        ("pairs", C.c_int64),
        ("cc", C.c_int64),
        ("penalty", C.c_int64),
        ("skipped", C.c_int64),
        ("scored", C.c_int64),
        ("sum_fixed", C.c_uint64 * 3),
        ("sum", C.c_double),
        ("n_sources_gt", C.c_int32),
        ("n_sources_prop", C.c_int32),
        ("terminals_gt", C.c_int32),
        ("terminals_prop", C.c_int32),
    ]


APLS_CANDIDATES = 10

_vp, _i, _f, _d = C.c_void_p, C.c_int, C.c_float, C.c_double
_ip = C.POINTER(C.c_int)
_targs = C.POINTER(SamRoadTrainArgs)

# samroad_argsort_fn: int (*)(const void* keys, int key_dtype, int64_t n, int64_t* order_out, void* user)
ARGSORT_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int64, C.POINTER(C.c_int64), C.c_void_p)

# name -> (restype, argtypes); mirrors include/samroad_b200.h one to one
SIGNATURES = {
    "samroad_create": (_i, [C.POINTER(SamRoadCfg), _i, C.POINTER(_vp)]),
    "samroad_destroy": (_i, [_vp]),
    "samroad_load_tensor": (_i, [_vp, C.c_char_p, _vp, C.POINTER(C.c_int64), _i]),
    "samroad_finalize_weights": (_i, [_vp]),
    "samroad_encode_masks": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "samroad_toponet": (_i, [_vp, _vp, _vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "samroad_fuse_masks": (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "samroad_encode_masks_scene": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    "samroad_graph_create": (_i, [_i, C.POINTER(_vp)]),
    "samroad_graph_destroy": (_i, [_vp]),
    "samroad_extract_graph_points": (_i, [_vp, _vp, _vp, _i, _i, _d, _d, _d, _d, ARGSORT_FN, _vp, _vp, _i,
                                          _ip, _vp, _vp]),
    "samroad_pair_queries_plan": (_i, [_vp, _vp, _i, _vp, _i, _i, _d, _vp, _vp]),
    "samroad_pair_queries_plan_k": (_i, [_vp, _vp, _i, _vp, _i, _i, _d, _i, _vp, _vp]),
    "samroad_pair_queries_fill": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "samroad_aggregate_edges": (_i, [_vp, _vp, _vp, _i, _f, _vp, _i, _ip, _ip, _vp]),
    "samroad_encode_masks_host": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "samroad_infer_batch_host": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "samroad_infer_batch_host_async": (_i, [_vp, _i, _vp, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp, _vp,
                                            _vp]),
    "samroad_infer_batch_host_wait": (_i, [_vp, _i]),
    "samroad_prc_create": (_i, [_i, C.POINTER(_vp)]),
    "samroad_prc_destroy": (_i, [_vp]),
    "samroad_prc_reset": (_i, [_vp, _vp]),
    "samroad_prc_update": (_i, [_vp, _vp, C.c_int64, _vp, _i, _vp, C.c_int64, _vp]),
    "samroad_prc_compute": (_i, [_vp, C.POINTER(C.c_int64), C.POINTER(C.c_float), _vp]),
    "samroad_prc_read_curve": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "samroad_prc_export_keys": (_i, [_vp, _vp, C.c_int64, C.POINTER(C.c_int64), _vp]),
    "samroad_prc_append_keys": (_i, [_vp, _vp, C.c_int64, _vp]),
    "samroad_val_create": (_i, [_i, C.POINTER(_vp)]),
    "samroad_val_destroy": (_i, [_vp]),
    "samroad_val_reset": (_i, [_vp, _vp]),
    "samroad_val_update": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "samroad_val_read": (_i, [_vp, C.POINTER(C.c_int64), C.POINTER(C.c_float), C.POINTER(C.c_int64), _vp]),
    "samroad_train_workspace_bytes": (_i, [_vp, _targs, C.POINTER(C.c_size_t)]),
    "samroad_train_forward": (_i, [_vp, _targs, _vp, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp,
                                   C.c_size_t, _vp, _vp, _vp]),
    "samroad_train_backward": (_i, [_vp, _targs, _vp, _vp, _vp, _i, _vp, C.c_size_t, _vp, _vp]),
    "samroad_update_tensor_device": (_i, [_vp, C.c_char_p, _vp, C.POINTER(C.c_int64), _i, _vp]),
    "samroad_debug_train_dropout_keep": (_i, [_f, C.c_uint64, _i, _i, C.c_int64, _vp, _vp]),
    "samroad_labels_create": (_i, [_i, C.POINTER(SamRoadLabelCfg), C.POINTER(_vp)]),
    "samroad_labels_destroy": (_i, [_vp]),
    "samroad_labels_upload": (_i, [_vp, _vp, _vp, _vp, C.c_int32, _vp, _vp, _vp, _vp, _vp,
                                   C.POINTER(C.c_int32)]),
    "samroad_labels_batch": (_i, [_vp, _i, C.c_uint64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                  C.POINTER(C.c_int32), _vp]),
    "samroad_debug_labels_batch_draws": (_i, [_vp, _i, _i, C.c_uint64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                              _vp, _vp, C.POINTER(C.c_int32), _vp]),
    "samroad_topo_create": (_i, [_i, C.POINTER(SamRoadTopoCaps), C.POINTER(_vp)]),
    "samroad_topo_destroy": (_i, [_vp]),
    "samroad_topo_upload_graph": (_i, [_vp, _i, C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "samroad_topo_run": (_i, [_vp, C.c_int32, _vp, _vp, _d, _d, _d, _d, _vp]),
    "samroad_apls_create": (_i, [_i, C.POINTER(SamRoadAplsCaps), C.POINTER(_vp)]),
    "samroad_apls_destroy": (_i, [_vp]),
    "samroad_apls_upload_graph": (_i, [_vp, _i, C.c_int32, _vp, _vp, _vp, _vp]),
    "samroad_apls_candidates": (_i, [_vp, _i, C.c_int32, _vp, _vp]),
    "samroad_apls_one_way": (_i, [_vp, _i, C.c_int32, _vp, _vp, _d, C.POINTER(SamRoadAplsResult), _vp, _vp]),
    "samroad_label_masks": (_i, [_i, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "samroad_stream_write_value32": (_i, [_vp, C.c_uint32, _vp]),
    "samroad_stream_wait_value32": (_i, [_vp, C.c_uint32, _vp]),
    "samroad_timing_enable": (_i, [_vp, _i]),
    "samroad_timing_read": (_i, [_vp, C.c_char_p, C.c_size_t]),
    "samroad_workspace_bytes": (C.c_size_t, [_vp, _i]),
    "samroad_launch_count": (C.c_uint64, [_i]),
    "samroad_last_error": (C.c_char_p, []),
    "samroad_abi_version": (_i, []),
    "samroad_op_gemm_f16": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp]),
    "samroad_op_gemm_f32": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _i, _vp]),
    "samroad_op_gemm_ln": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _f, _i, _i,
                                _vp, _vp, _vp, _i, _i, _vp]),
    "samroad_op_gemm_ref": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _i, _vp]),
    "samroad_op_layernorm": (_i, [_vp, _vp, _vp, _f, _i, _i, _vp, _vp]),
    "samroad_debug_force_simt_attention": (None, [_i]),
    "samroad_debug_attention_path": (_i, [_i, _i, _i, _vp, _vp]),
    "samroad_debug_disable_2cta_gemm": (None, [_i]),
    "samroad_op_attention": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "samroad_op_sam_decoder": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "samroad_op_encoder_taps": (_i, [_vp, _vp, _i, _i, C.POINTER(SamroadEncoderTaps), _vp, _vp, _vp, _vp]),
}

_lib = None


def load() -> C.CDLL:
    """Load the shared library (once). Fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m sam_road_b200.build` "
            "(nvcc, sm_90a). sam_road_b200 has no CPU or PyTorch fallback path.")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().samroad_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed (code {rc}): {last_error()}")


def refuse_copy(self):
    """__getstate__ of every native handle owner: device state cannot be copied or pickled."""
    raise TypeError(f"{type(self).__name__} owns a native handle and cannot be copied or pickled")


class Handle:
    """Owner of one native handle.  `Handle(create, destroy, *args)` calls the library's `create(*args, &out)`
    (RuntimeError with samroad_last_error() when it fails) and releases the handle with `destroy` on the
    first `close()` or, at the latest, when the object is collected.  It passes straight into ctypes calls;
    once closed it passes as NULL, which every entry point refuses with an error."""

    __getstate__ = refuse_copy

    def __init__(self, create: str, destroy: str, *args):
        lib = load()
        h = C.c_void_p()
        check(getattr(lib, create)(*args, C.byref(h)), create)
        self._as_parameter_ = h.value
        self._finalizer = weakref.finalize(self, getattr(lib, destroy), h.value)

    def close(self) -> None:
        self._as_parameter_ = None
        self._finalizer()     # destroys the handle the first time only


def ptr(t) -> int | None:
    """Device/host pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def current_stream_ptr() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream
