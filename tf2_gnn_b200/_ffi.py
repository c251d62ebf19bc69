"""ctypes binding of libtfgnn_b200.so (include/tfgnn_b200.h).

There is no CPU fallback: if the library is missing, every entry point raises.  Device pointers
are taken zero-copy from any object exposing ``data_ptr()`` (torch) or ``__cuda_array_interface__``
(cupy, numba, ...); TensorFlow tensors go through ``tf.experimental.dlpack`` (see tf_adapter.py).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int32, c_int64, c_uint32, c_void_p
from typing import Optional, Sequence

# TFGNN_B200_LIB: an alternative build of the same in-tree library (kernel A/B experiments)
_LIB_PATH = os.environ.get("TFGNN_B200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc",
                                                             "libtfgnn_b200.so")
_lib: Optional[ctypes.CDLL] = None

# enums of include/tfgnn_b200.h
OK, ERR_INVALID_ARGUMENT, ERR_CUDA, ERR_UNSUPPORTED, ERR_INDEX_OUT_OF_RANGE = 0, 1, 2, 3, 4
AGG = {"sum": 0, "mean": 1, "max": 2, "sqrt_n": 3}
ACT = {None: 0, "relu": 1, "tanh": 2, "leaky_relu": 3, "elu": 4, "selu": 5, "gelu": 6}
ACT_SIGMOID = 7  # library-internal (readout weights); deliberately NOT in the name table: the reference raises on "sigmoid"
FLAG_NORMALIZE, FLAG_ACT_BEFORE_AGG, FLAG_USE_TARGET = 1, 2, 4
READOUT_MODE = {"softmax": 0, "sigmoid": 1, "none": 2, "average": 3}
PATH = {"auto": 0, "atomic": 1, "sorted": 2, "sorted_tc": 3, "fused_tc": 4}
PREPARE_VALIDATE = 1
PREPARE_TRANSPOSE = 2
PREPARE_TRANSPOSE_OWNED = 4
MAX_EDGE_TYPES = 32

EXPORTED_SYMBOLS = (
    "tfgnn_b200_abi_version", "tfgnn_b200_last_error", "tfgnn_b200_prepare", "tfgnn_b200_prepare_sharded", "tfgnn_b200_free_batch",
    "tfgnn_b200_batch_info", "tfgnn_b200_batch_export_csr", "tfgnn_b200_in_degree", "tfgnn_b200_edge_mlp_fwd", "tfgnn_b200_rgcn_fwd", "tfgnn_b200_rgcn_bwd",
    "tfgnn_b200_ggnn_fwd", "tfgnn_b200_ggnn_bwd", "tfgnn_b200_rgin_fwd", "tfgnn_b200_film_fwd", "tfgnn_b200_rgat_fwd",
    "tfgnn_b200_dense_fwd", "tfgnn_b200_gather_rows", "tfgnn_b200_unsorted_segment_reduce",
    "tfgnn_b200_activation", "tfgnn_b200_residual_average", "tfgnn_b200_layer_norm",
    "tfgnn_b200_process_adjacency_sizes", "tfgnn_b200_process_adjacency",
    "tfgnn_b200_assemble_batch_workspace_bytes", "tfgnn_b200_assemble_batch",
    "tfgnn_b200_launch_count", "tfgnn_b200_set_l2_persist_mb", "tfgnn_b200_release_device_state",
    "tfgnn_b200_graph_offsets", "tfgnn_b200_segment_softmax", "tfgnn_b200_weighted_segment_sum",
    "tfgnn_b200_gathered_add", "tfgnn_b200_gru_gate_fwd", "tfgnn_b200_clamp", "tfgnn_b200_dense_bias_fwd",
    "tfgnn_b200_dense_bwd", "tfgnn_b200_layer_norm_bwd", "tfgnn_b200_dropout", "tfgnn_b200_axpby",
    "tfgnn_b200_activation_bwd", "tfgnn_b200_row_scale", "tfgnn_b200_mul_add", "tfgnn_b200_segment_max_bwd",
    "tfgnn_b200_rgcn_fwd_allgather", "tfgnn_b200_softmax_apply", "tfgnn_b200_head_scale", "tfgnn_b200_head_dot",
    "tfgnn_b200_gru_gate_bwd", "tfgnn_b200_rgcn_ln_fwd", "tfgnn_b200_film_bwd",
    "tfgnn_b200_edge_mlp_bwd", "tfgnn_b200_rgat_bwd",
    "tfgnn_b200_segment_sum_rows", "tfgnn_b200_readout_bwd", "tfgnn_b200_gru_gate_bwd_indexed",
)

_PP = POINTER(c_void_p)


def library_path() -> str:
    return _LIB_PATH


def lib() -> ctypes.CDLL:
    """Load (once) and return the CUDA library.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(
            f"{_LIB_PATH} is missing: build it with `python -m tf2_gnn_b200.build` "
            "(there is no CPU fallback for the message-passing path)")
    L = ctypes.CDLL(_LIB_PATH)
    L.tfgnn_b200_abi_version.restype = ctypes.c_int
    L.tfgnn_b200_last_error.restype = c_char_p
    L.tfgnn_b200_launch_count.restype = c_int64
    L.tfgnn_b200_prepare.argtypes = [_PP, POINTER(c_int64), c_int32, c_int64, c_uint32, POINTER(c_void_p), c_void_p]
    L.tfgnn_b200_prepare_sharded.argtypes = [_PP, POINTER(c_int64), c_int32, c_int64, c_int64, c_int64, c_uint32,
                                             POINTER(c_void_p), c_void_p]
    L.tfgnn_b200_free_batch.argtypes = [c_void_p]
    L.tfgnn_b200_batch_info.argtypes = [c_void_p, POINTER(c_int64), POINTER(c_int32), POINTER(c_int64),
                                        POINTER(c_void_p), POINTER(c_void_p)]
    L.tfgnn_b200_batch_export_csr.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p]
    L.tfgnn_b200_in_degree.argtypes = [c_void_p, c_void_p, c_void_p]
    L.tfgnn_b200_edge_mlp_fwd.argtypes = [c_void_p, c_void_p, c_int32, _PP, c_int32, c_int32, c_uint32, c_int32,
                                          c_int32, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_rgcn_fwd.argtypes = [c_void_p, c_void_p, c_int32, _PP, c_int32, c_uint32, c_int32, c_int32,
                                      c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_rgcn_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, _PP, c_int32, c_uint32, c_int32, c_int32,
                                      c_void_p, c_void_p, c_void_p, _PP, c_void_p]
    L.tfgnn_b200_ggnn_fwd.argtypes = [c_void_p, c_void_p, c_int32, _PP, c_int32, c_int32, c_uint32, c_int32,
                                      c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_rgin_fwd.argtypes = [c_void_p, c_void_p, c_int32, _PP, c_int32, c_int32, c_uint32, c_int32,
                                      c_int32, _PP, c_int32, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_film_fwd.argtypes = [c_void_p, c_void_p, c_int32, _PP, c_int32, _PP, c_int32, c_uint32, c_int32,
                                      c_int32, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_film_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, _PP, _PP, c_int32, c_uint32, c_int32,
                                      c_int32, c_void_p, c_void_p, c_void_p, _PP, _PP, c_void_p]
    L.tfgnn_b200_edge_mlp_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, _PP, c_int32, c_int32, c_uint32,
                                          c_int32, c_int32, c_void_p, c_void_p, c_void_p, _PP, c_void_p]
    L.tfgnn_b200_rgat_fwd.argtypes = [c_void_p, c_void_p, c_int32, _PP, _PP, c_int32, c_int32, c_int32, c_int32,
                                      c_void_p, c_void_p]
    L.tfgnn_b200_rgat_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, _PP, _PP, c_int32, c_int32, c_int32, c_int32,
                                      c_void_p, c_void_p, c_void_p, _PP, _PP, c_void_p]
    L.tfgnn_b200_dense_fwd.argtypes = [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_int32, c_int32, c_int32,
                                       c_void_p]
    L.tfgnn_b200_gather_rows.argtypes = [c_void_p, c_int64, c_int32, c_void_p, c_int64, c_int64, c_void_p, c_void_p]
    L.tfgnn_b200_unsorted_segment_reduce.argtypes = [c_void_p, c_void_p, c_int64, c_int64, c_int32, c_int64,
                                                     c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_activation.argtypes = [c_void_p, c_int64, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_residual_average.argtypes = [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]
    L.tfgnn_b200_layer_norm.argtypes = [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_float, c_void_p, c_void_p]
    L.tfgnn_b200_ggnn_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, _PP, c_int32, c_uint32, c_int32,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, _PP, c_void_p, c_void_p,
                                      c_void_p, c_void_p]
    L.tfgnn_b200_process_adjacency_sizes.argtypes = [POINTER(c_int64), c_int32, c_int64, c_int32, POINTER(c_int32),
                                                     c_int32, POINTER(c_int64), POINTER(c_int32)]
    L.tfgnn_b200_process_adjacency.argtypes = [_PP, POINTER(c_int64), c_int32, c_int64, c_int32, POINTER(c_int32),
                                               c_int32, _PP, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_assemble_batch_workspace_bytes.argtypes = [c_int32, c_int32]
    L.tfgnn_b200_assemble_batch_workspace_bytes.restype = ctypes.c_size_t
    L.tfgnn_b200_assemble_batch.argtypes = [c_void_p, _PP, _PP, c_int32, c_int64, c_void_p, c_int32, c_int64,
                                            POINTER(c_int64), c_void_p, c_void_p, _PP, c_void_p, c_void_p]
    L.tfgnn_b200_graph_offsets.argtypes = [c_void_p, c_int64, c_int32, c_void_p, c_int32, c_void_p]
    L.tfgnn_b200_segment_softmax.argtypes = [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_weighted_segment_sum.argtypes = [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                                                  c_void_p, c_void_p]
    L.tfgnn_b200_gathered_add.argtypes = [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_float, c_int32, c_void_p,
                                          c_void_p]
    L.tfgnn_b200_gru_gate_fwd.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_clamp.argtypes = [c_void_p, c_int64, c_float, c_float, c_int32, c_int32, c_void_p]
    L.tfgnn_b200_dense_bias_fwd.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_int32, c_int32,
                                            c_int32, c_void_p]
    L.tfgnn_b200_dense_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_int32, c_int32,
                                       c_void_p, c_void_p, c_void_p, c_void_p]
    L.tfgnn_b200_layer_norm_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_float, c_void_p, c_void_p,
                                            c_void_p, c_void_p]
    L.tfgnn_b200_dropout.argtypes = [c_void_p, c_int64, c_float, ctypes.c_uint64, ctypes.c_uint64, c_void_p, c_void_p]
    L.tfgnn_b200_axpby.argtypes = [c_void_p, c_float, c_void_p, c_float, c_int64, c_void_p, c_void_p]
    L.tfgnn_b200_activation_bwd.argtypes = [c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_row_scale.argtypes = [c_void_p, c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_mul_add.argtypes = [c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_int64, c_int32, c_void_p,
                                     c_int32, c_void_p]
    L.tfgnn_b200_segment_max_bwd.argtypes = [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int32, c_int64,
                                             c_void_p, c_void_p]
    L.tfgnn_b200_rgcn_fwd_allgather.argtypes = [c_void_p, c_void_p, c_int32, _PP, c_int32, c_uint32, c_int32, c_int32, _PP,
                                                c_int32, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_softmax_apply.argtypes = [c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p]
    L.tfgnn_b200_head_scale.argtypes = [c_void_p, c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_head_dot.argtypes = [c_void_p, c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_gru_gate_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p,
                                          c_void_p, c_void_p]
    L.tfgnn_b200_rgcn_ln_fwd.argtypes = [c_void_p, c_void_p, c_int32, _PP, c_int32, c_uint32, c_int32, c_int32, c_int32,
                                         c_void_p, c_void_p, c_float, c_void_p, c_void_p]
    L.tfgnn_b200_segment_sum_rows.argtypes = [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p]
    L.tfgnn_b200_readout_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32,
                                         c_int32, c_int32, c_int32, c_float, c_float, c_int32, c_int32, c_void_p, c_void_p,
                                         c_void_p]
    L.tfgnn_b200_gru_gate_bwd_indexed.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
                                                  c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]
    L.tfgnn_b200_set_l2_persist_mb.argtypes = [c_int32]
    L.tfgnn_b200_release_device_state.argtypes = []
    for name in EXPORTED_SYMBOLS:
        fn = getattr(L, name)
        if fn.restype is ctypes.c_int and name not in ("tfgnn_b200_abi_version",):
            fn.restype = ctypes.c_int
    if L.tfgnn_b200_abi_version() != 1:
        raise RuntimeError("libtfgnn_b200.so ABI version mismatch; rebuild with python -m tf2_gnn_b200.build")
    _lib = L
    import atexit
    atexit.register(_release_device_state)
    return L


def _release_device_state() -> None:
    """Restore the persisting-L2 limit the fused kernel raised and trim the library's memory pool
    (include/tfgnn_b200.h, "Device-global state")."""
    try:
        if _lib is not None:
            _lib.tfgnn_b200_release_device_state()
    except Exception:
        pass


def check(rc: int) -> None:
    """Map a non-zero return code to the Python exception the reference would raise."""
    if rc == OK:
        return
    msg = lib().tfgnn_b200_last_error().decode("utf-8", "replace")
    if rc == ERR_INVALID_ARGUMENT:
        raise ValueError(msg)
    if rc == ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    if rc == ERR_INDEX_OUT_OF_RANGE:
        raise IndexError(msg)
    raise RuntimeError(msg)


def device_ptr(x) -> int:
    """Raw device address of a CUDA tensor/array (zero-copy)."""
    if x is None:
        return 0
    if hasattr(x, "data_ptr"):
        return int(x.data_ptr())
    cai = getattr(x, "__cuda_array_interface__", None)
    if cai is not None:
        return int(cai["data"][0])
    raise TypeError(f"cannot take a device pointer from {type(x)!r}")


def ptr_array(tensors: Sequence) -> "ctypes.Array":
    arr = (c_void_p * max(len(tensors), 1))()
    for i, t in enumerate(tensors):
        arr[i] = device_ptr(t)
    return arr


def launch_count() -> int:
    return int(lib().tfgnn_b200_launch_count())
