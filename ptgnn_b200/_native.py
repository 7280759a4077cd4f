"""ctypes binding of the C ABI declared in ``include/ptgnn_b200.h`` (libptgnn_b200.so, built in-tree).

There is deliberately NO fallback: if the shared library is missing or a call fails, an exception is raised.
PyTorch is used only for device memory (``Tensor.data_ptr()``), streams and ``torch.distributed``.
"""
import ctypes
import os
import re
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libptgnn_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ptgnn_b200.h")

REDUCE = {"sum": 0, "add": 0, "mean": 1, "max": 2, "min": 3}
READOUT_SUM, READOUT_MEAN, READOUT_WEIGHTED_SUM = 0, 1, 2
POOL = {"sum": 0, "mean": 1, "max": 2}
ACT_NONE, ACT_GELU, ACT_TANH, ACT_RELU = 0, 1, 2, 3

c_i32, c_i64, c_f32, c_void_p, c_size_t = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t


class NativeLibraryError(RuntimeError):
    pass


_SCALAR_TYPES = {"int": c_i32, "int32_t": c_i32, "int64_t": c_i64, "size_t": c_size_t, "float": c_f32}


def _ctype(decl: str, proto: str, result: bool = False):
    words = re.sub(r"\bconst\b", " ", decl).replace("*", " * ").split()
    if "*" in words:
        if not result:
            return c_void_p          # callers pass Tensor.data_ptr(), None, host arrays or ctypes.byref(...)
        if words == ["char", "*"]:
            return ctypes.c_char_p
    else:
        base = " ".join(words if result or len(words) == 1 else words[:-1])      # a parameter drops its name
        if base in _SCALAR_TYPES:
            return _SCALAR_TYPES[base]
    raise NativeLibraryError(f"no ctypes type for `{decl.strip()}` in the C ABI prototype `{proto}`")


def parse_signatures(header: str) -> dict:
    """{name: (restype, argtypes)} of every ``ptgnn_b200_*`` prototype in the C header text ``header``.  A type without a
    mapping raises NativeLibraryError: a wrong guess would pass every call through ctypes and corrupt it."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*|^[ \t]*#[^\n]*", " ", header, flags=re.S | re.M)
    signatures = {}
    for statement in text.split(";"):
        m = re.search(r"([\w\s*]*?)\b(ptgnn_b200_\w+)\s*\(([^()]*)\)\s*$", statement)
        if m is not None:
            result, name, params = m.group(1), m.group(2), m.group(3).strip()
            proto = " ".join(m.group(0).split())
            signatures[name] = (_ctype(result, proto, result=True),
                                [] if params == "void" else [_ctype(p, proto) for p in params.split(",")])
    return signatures


# symbol -> (restype, argtypes) of every function include/ptgnn_b200.h declares: the header is the only place they are written
with open(HEADER_PATH, encoding="utf-8") as _f:
    SIGNATURES = parse_signatures(_f.read())


class BlockPlanStruct(ctypes.Structure):
    """`ptgnn_b200_block_plan` of include/ptgnn_b200.h."""
    _fields_ = [("block_targets", c_i32), ("group_off", c_void_p), ("src_f", c_void_p), ("tl_f", c_void_p), ("status", c_void_p)]


ABI_VERSION = 4        # moves only on incompatible changes of an existing entry point (include/ptgnn_b200.h)
_lib: Optional[ctypes.CDLL] = None


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


def call(name: str, device, *args) -> None:
    """Enqueues the entry point ``name`` on ``device``'s current stream: ``args`` are its parameters except the trailing ``stream``.
    The argument count is checked first (ctypes rejects too few arguments but passes surplus ones through); a nonzero return code
    raises as in ``check``."""
    if len(args) + 1 != len(SIGNATURES[name][1]):
        raise TypeError(f"{name} takes {len(SIGNATURES[name][1]) - 1} arguments before its stream, got {len(args)}")
    with torch.cuda.device(device):
        rc = getattr(lib(), name)(*args, current_stream(device))
    check(rc, name)


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
