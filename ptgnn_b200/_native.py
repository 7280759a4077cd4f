"""ctypes binding of the C ABI declared in ``include/ptgnn_b200.h`` (libptgnn_b200.so, built in-tree).

There is deliberately NO fallback: if the shared library is missing or a call fails, an exception is raised.
PyTorch is used only for device memory (``Tensor.data_ptr()``), streams and ``torch.distributed``.
"""
import ctypes
import os
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libptgnn_b200.so")

REDUCE = {"sum": 0, "add": 0, "mean": 1, "max": 2, "min": 3}
READOUT_SUM, READOUT_MEAN, READOUT_WEIGHTED_SUM = 0, 1, 2
POOL = {"sum": 0, "mean": 1, "max": 2}
ACT_NONE, ACT_GELU, ACT_TANH, ACT_RELU = 0, 1, 2, 3

c_i32, c_i64, c_f32, c_void_p, c_size_t = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t

# symbol -> (restype, argtypes); must list every function include/ptgnn_b200.h declares (tests check this).
SIGNATURES = {
    "ptgnn_b200_abi_version": (ctypes.c_int, []),
    "ptgnn_b200_last_error": (ctypes.c_char_p, []),
    "ptgnn_b200_launch_count": (c_i64, []),
    "ptgnn_b200_kernel_timing_enable": (ctypes.c_int, [c_i32]),
    "ptgnn_b200_kernel_timing_read": (ctypes.c_int, [c_void_p, c_void_p, c_i32]),
    "ptgnn_b200_plan_workspace_bytes": (c_size_t, [c_i64, c_i64]),
    "ptgnn_b200_plan_build": (ctypes.c_int, [c_i64, c_i64, c_i32, c_void_p, c_void_p, c_void_p] + [c_void_p] * 8 + [c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_plan_convert": (ctypes.c_int, [c_i64, c_i64, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_plan_sort": (ctypes.c_int, [c_i64, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_segment_reduce_f32": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_void_p]),
    "ptgnn_b200_scatter_workspace_bytes": (c_size_t, [c_i64, c_i64]),
    "ptgnn_b200_scatter_f32": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_i64, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_gated_workspace_bytes": (c_size_t, [c_i32, c_i64, c_i64, c_i32, c_i32, c_i32]),
    "ptgnn_b200_gated_weight_cache_bytes": (c_size_t, [c_i32, c_i32, c_i32, c_i32]),
    "ptgnn_b200_gated_forward": (ctypes.c_int, [c_i32, c_void_p, c_void_p, c_i64, c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i32, c_void_p, c_void_p, c_size_t,
                                                c_void_p, c_size_t, c_i32, c_void_p]),
    "ptgnn_b200_mlp_workspace_bytes": (c_size_t, [c_i32, c_i64, c_i64, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "ptgnn_b200_mlp_forward": (ctypes.c_int, [c_i32, c_void_p, c_void_p, c_i64, c_i32, c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p,
                                              c_void_p, c_void_p, c_i32, c_i32, c_i32, c_void_p, c_void_p, c_f32, c_void_p, c_void_p, c_i32,
                                              c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_block_plan_block_targets": (c_i32, [c_i64]),
    "ptgnn_b200_block_plan_workspace_bytes": (c_size_t, [c_i64, c_i64, c_i32, c_i32]),
    "ptgnn_b200_block_plan_build": (ctypes.c_int, [c_i64, c_i32, c_void_p, c_void_p, c_void_p, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_fused_supported": (c_i32, [c_i32, c_i32, c_i32]),
    "ptgnn_b200_gated_fused_workspace_bytes": (c_size_t, [c_i32, c_i64, c_i64, c_i32, c_i32, c_i32]),
    "ptgnn_b200_gated_fused_weight_cache_bytes": (c_size_t, [c_i32, c_i32, c_i32, c_i32]),
    "ptgnn_b200_packed_state_bytes": (c_size_t, [c_i64, c_i32]),
    "ptgnn_b200_gated_forward_fused": (ctypes.c_int, [c_i32, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i32, c_i32, c_i32, c_void_p, c_void_p,
                                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i32, c_void_p, c_void_p, c_void_p,
                                                      c_size_t, c_void_p, c_size_t, c_i32, c_void_p]),
    "ptgnn_b200_mlp_fused_workspace_bytes": (c_size_t, [c_i32, c_i64, c_i64, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "ptgnn_b200_mlp_fused_weight_cache_bytes": (c_size_t, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "ptgnn_b200_mlp_forward_fused": (ctypes.c_int, [c_i32, c_void_p, c_void_p, c_i64, c_i64, c_i32, c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p,
                                                    c_i32, c_i32, c_i32, c_void_p, c_void_p, c_f32, c_void_p, c_void_p, c_i32, c_void_p, c_void_p,
                                                    c_size_t, c_void_p, c_size_t, c_i32, c_void_p]),
    "ptgnn_b200_gather_split_f16": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ptgnn_b200_gru_gate_grads_f32": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ptgnn_b200_offset_ids": (ctypes.c_int, [c_void_p, c_i64, c_void_p, c_void_p, c_i32, c_void_p, c_void_p]),
    "ptgnn_b200_segment_ids": (ctypes.c_int, [c_void_p, c_i32, c_i64, c_void_p, c_void_p]),
    "ptgnn_b200_linear_workspace_bytes": (c_size_t, [c_i32, c_i32]),
    "ptgnn_b200_linear_f32": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_i32, c_i32, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_grucell_workspace_bytes": (c_size_t, [c_i32, c_i32]),
    "ptgnn_b200_grucell_f32": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_edge_messages_workspace_bytes": (c_size_t, [c_i32, c_i32, c_i32, c_i32]),
    "ptgnn_b200_edge_messages_f32": (ctypes.c_int, [c_void_p, c_void_p, c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                    c_i32, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_graph_readout_workspace_bytes": (c_size_t, [c_i64, c_i64, c_i32]),
    "ptgnn_b200_graph_readout": (ctypes.c_int, [c_i32, c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_i64, c_void_p, c_i32, c_void_p, c_void_p,
                                                c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_global_gru_supported": (c_i32, [c_i32, c_i32]),
    "ptgnn_b200_global_gru_workspace_bytes": (c_size_t, [c_i32, c_i64, c_i64, c_i32, c_i32]),
    "ptgnn_b200_global_gru_weight_cache_bytes": (c_size_t, [c_i32, c_i32]),
    "ptgnn_b200_global_gru_update": (ctypes.c_int, [c_i32, c_void_p, c_void_p, c_i64, c_i32, c_void_p, c_i64, c_void_p, c_i32, c_void_p, c_void_p,
                                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_size_t,
                                                    c_i32, c_void_p]),
    "ptgnn_b200_attention_readout_supported": (c_i32, [c_i32, c_i32, c_i32]),
    "ptgnn_b200_attention_readout_workspace_bytes": (c_size_t, [c_i64, c_i64, c_i32, c_i32]),
    "ptgnn_b200_attention_readout": (ctypes.c_int, [c_i32, c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_i64, c_void_p, c_void_p,
                                                    c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_attention_readout_backward_f32": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_i64, c_void_p, c_void_p,
                                                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_selfatt_supported": (c_i32, [c_i32, c_i32, c_i32]),
    "ptgnn_b200_selfatt_workspace_bytes": (c_size_t, [c_i64, c_i64, c_i32]),
    "ptgnn_b200_selfatt_forward": (ctypes.c_int, [c_i32, c_void_p, c_i64, c_i32, c_i32, c_i32, c_void_p, c_i64, c_i64, c_void_p, c_void_p,
                                                  c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_selfatt_backward_f32": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_i32, c_i32, c_void_p, c_i64, c_i64, c_void_p, c_void_p,
                                                       c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_graph_norm_supported": (c_i32, [c_i32]),
    "ptgnn_b200_graph_norm_workspace_bytes": (c_size_t, [c_i64, c_i64, c_i32]),
    "ptgnn_b200_graph_norm_forward": (ctypes.c_int, [c_i32, c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_void_p,
                                                     c_void_p, c_f32, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_graph_norm_backward_f32": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_void_p, c_i64, c_void_p,
                                                          c_void_p, c_f32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                          c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_pna_supported": (c_i32, [c_i32]),
    "ptgnn_b200_pna_forward": (ctypes.c_int, [c_i32, c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_i64, c_f32, c_void_p, c_void_p, c_void_p,
                                              c_void_p]),
    "ptgnn_b200_pna_backward_f32": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_i64, c_f32, c_void_p, c_void_p, c_void_p,
                                                   c_void_p, c_void_p, c_void_p]),
    "ptgnn_b200_copy_attention_supported": (c_i32, [c_i32, c_i32, c_i32]),
    "ptgnn_b200_copy_attention_workspace_bytes": (c_size_t, [c_i64, c_i64, c_i32, c_i32]),
    "ptgnn_b200_copy_attention": (ctypes.c_int, [c_i32, c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_i64, c_void_p, c_void_p, c_void_p,
                                                 c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_copy_attention_backward_f32": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_i64, c_void_p, c_void_p,
                                                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_embedding_bag_supported": (c_i32, [c_i32, c_i32]),
    "ptgnn_b200_embedding_bag": (ctypes.c_int, [c_i32, c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p,
                                                c_void_p, c_void_p]),
    "ptgnn_b200_embedding_bag_pairs": (ctypes.c_int, [c_void_p, c_void_p, c_i64, c_i32, c_i64, c_void_p, c_void_p, c_void_p]),
    "ptgnn_b200_embedding_bag_backward_workspace_bytes": (c_size_t, [c_i64, c_i32, c_i64, c_i32]),
    "ptgnn_b200_embedding_bag_backward_f32": (ctypes.c_int, [c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_i32, c_void_p, c_void_p,
                                                             c_i64, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptgnn_b200_gated_gnn_forward_host_f32":(ctypes.c_int, [c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_i32,
                                                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i32, c_void_p]),
}



class BlockPlanStruct(ctypes.Structure):
    """`ptgnn_b200_block_plan` of include/ptgnn_b200.h."""
    _fields_ = [("block_targets", c_i32), ("group_off", c_void_p), ("src_f", c_void_p), ("tl_f", c_void_p), ("status", c_void_p)]


ABI_VERSION = 4        # moves only on incompatible changes of an existing entry point (include/ptgnn_b200.h)
_lib: Optional[ctypes.CDLL] = None


class NativeLibraryError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Loads libptgnn_b200.so (once).  Raises NativeLibraryError if it has not been built -- never falls back."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryError(
                f"{LIB_PATH} not found: build it with `python -m ptgnn_b200.build` (or __graft_entry__.build()). "
                "ptgnn_b200 has no CPU / PyTorch fallback for its CUDA kernels."
            )
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(handle, name)
            except AttributeError:      # a library built before this entry point was added (the ABI version only moves on incompatible changes)
                raise NativeLibraryError(f"{LIB_PATH} does not export {name}: it is older than this package; rebuild it with "
                                         "`python -m ptgnn_b200.build`") from None
            fn.restype = res
            fn.argtypes = args
        if handle.ptgnn_b200_abi_version() != ABI_VERSION:
            raise NativeLibraryError("libptgnn_b200.so ABI version mismatch; rebuild")
        _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().ptgnn_b200_last_error().decode("utf-8", "replace")
        codes = {-1: ValueError, -2: NotImplementedError, -3: RuntimeError, -4: RuntimeError, -5: IndexError}
        raise codes.get(rc, RuntimeError)(f"{what} failed (code {rc}): {msg}")


def launch_count() -> int:
    return int(lib().ptgnn_b200_launch_count())


KERNEL_CATEGORIES = ("plan", "message", "reduce", "gru", "dense", "pack")


def kernel_timing(enable: bool) -> None:
    check(lib().ptgnn_b200_kernel_timing_enable(int(enable)), "kernel_timing_enable")


def read_kernel_timing() -> dict:
    """{category: (total_ms, launches)} accumulated since the last read (synchronises the device)."""
    n = len(KERNEL_CATEGORIES)
    ms = (ctypes.c_double * n)()
    cnt = (c_i64 * n)()
    check(lib().ptgnn_b200_kernel_timing_read(ms, cnt, n), "kernel_timing_read")
    return {name: (float(ms[i]), int(cnt[i])) for i, name in enumerate(KERNEL_CATEGORIES)}


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def ptr_table(tensors: Sequence[torch.Tensor]):
    """[host] array of device (or host) pointers, as the C ABI expects for per-type lists."""
    tab = (c_void_p * max(len(tensors), 1))()
    for i, t in enumerate(tensors):
        tab[i] = t.data_ptr()
    return tab


def i64_array(values: Sequence[int]):
    arr = (c_i64 * max(len(values), 1))()
    for i, v in enumerate(values):
        arr[i] = int(v)
    return arr


def current_stream(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(t: torch.Tensor, name: str, dtype: torch.dtype) -> torch.Tensor:
    if not t.is_cuda:
        raise NativeLibraryError(
            f"{name} is on {t.device}; ptgnn_b200 only runs on CUDA (sm_90a) and has no CPU fallback"
        )
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()
