"""``torch_scatter``-compatible front end of the native segmented reduce.

Mirrors the slice of the third-party API the reference's hot path uses
(`/root/reference/ptgnn/neuralmodels/gnn/messagepassing/abstractmessagepassing.py:4,44-50`):
``scatter(src, index, dim=0, dim_size=N, reduce=...)`` with a 2-D fp32 ``src`` and a 1-D int64 ``index``, plus
``scatter_sum/mean/max/min`` (max/min return ``(out, arg)`` with torch_scatter's conventions: empty rows are 0 with
``arg == src.size(0)``, ties go to the first occurrence).  CUDA only; no fallback.
"""
from typing import Optional, Tuple

import torch

from . import _native as N


_LONG_SEGMENT_ROWS = 1024      # average rows per output row from which the two-level reduction is used (readout-style calls)


def _run_two_level(src: torch.Tensor, index: torch.Tensor, dim_size: int, reduce: str):
    """Few, very long segments (graph-level readouts: node_to_graph_idx has ~10^2 targets for ~10^5 rows).  The segmented-reduce
    kernel parallelises over TARGET rows, so such a call would run on a handful of warps (measured: 28 ms for 204,800 x 128 -> 80).
    Two levels of the same kernel instead: every segment is cut, in its stable sorted order, into sub-segments of `chunk` ~
    sqrt(average segment length) rows, numbered compactly (exclusive scan of the per-target chunk counts, all on the device, no
    synchronisation); level 1 reduces the sub-segments, level 2 the partial results of each target.  sum / mean re-associate the
    fp32 sum by chunks (max / min are exact); arg outputs are not offered on this path."""
    from .edgeplan import EdgePlan

    E, D = src.shape
    chunk = max(64, min(1024, int((E / max(dim_size, 1)) ** 0.5)))
    plan = EdgePlan([(index, index)], dim_size)                   # row_ptr + stable sorted positions; reports out-of-range indices
    tgt = plan.tgt32.long()
    row_ptr = plan.row_ptr.long()
    count = row_ptr[1:] - row_ptr[:-1]
    chunks = (count + (chunk - 1)) // chunk                       # sub-segments of every target
    first = torch.cumsum(chunks, 0) - chunks                      # ... and the id of its first one
    rank = plan.pos.long() - row_ptr[:-1].index_select(0, tgt)    # position of a row inside its target's segment
    sub = first.index_select(0, tgt) + torch.div(rank, chunk, rounding_mode="floor")
    num_sub = E // chunk + dim_size                               # upper bound of sum(chunks), known without a device read
    level = "sum" if reduce in ("sum", "mean") else reduce
    part, _ = _run(src, sub, 0, num_sub, level, False, two_level=False)
    owner = torch.zeros(num_sub, dtype=torch.int64, device=src.device)
    owner.index_put_((sub,), tgt)                                 # duplicates write the same value; unused ids stay with target 0 ...
    if level != "sum":         # ... where, like every empty sub-segment (torch_scatter's 0), they must lose against every real value
        filled = torch.zeros(num_sub, dtype=torch.bool, device=src.device)
        filled.index_fill_(0, sub, True)
        lowest = torch.finfo(torch.float32).min if level == "max" else torch.finfo(torch.float32).max
        part = torch.where(filled[:, None], part, torch.full_like(part, lowest))
    out, _ = _run(part, owner, 0, dim_size, level, False, two_level=False)
    if reduce == "mean":
        out = out / count.clamp(min=1).to(torch.float32)[:, None]
    plan.poll()
    return out, None


def _run(src: torch.Tensor, index: torch.Tensor, dim: int, dim_size: Optional[int], reduce: str, want_arg: bool, two_level: bool = True):
    if src.dim() != 2 or dim not in (0, -2) or index.dim() != 1:
        raise NotImplementedError("native scatter supports src [E, D] reduced along dim=0 with a 1-D index")
    src = N.require_cuda(src, "src", torch.float32)
    index = N.require_cuda(index, "index", torch.int64)
    E, D = src.shape
    if index.shape[0] != E:
        raise ValueError("index and src disagree on the number of rows")
    if dim_size is None:
        dim_size = int(index.max().item()) + 1 if E else 0
    if two_level and not want_arg and dim_size > 0 and E >= 32768 and E // dim_size >= _LONG_SEGMENT_ROWS:
        return _run_two_level(src, index, dim_size, reduce)
    lib = N.lib()
    out = torch.empty(dim_size, D, dtype=torch.float32, device=src.device)
    arg = torch.empty(dim_size, D, dtype=torch.int64, device=src.device) if want_arg else None
    ws_bytes = lib.ptgnn_b200_scatter_workspace_bytes(dim_size, E)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=src.device)
    _poll_status()
    status = torch.zeros(1, dtype=torch.int32).pin_memory()     # written by the kernels, polled without synchronising
    N.call("ptgnn_b200_scatter_f32", src.device, N.ptr(src), N.ptr(index), E, D, dim_size, N.REDUCE[reduce], N.ptr(out), N.ptr(arg),
           status.data_ptr(), N.ptr(ws), ws_bytes)
    _PENDING.append((status, dim_size))
    return out, arg


# Out-of-range indices are reported by the kernels through a pinned status word; the reference (torch_scatter) raises an
# IndexError / device assert in that case.  Checked without synchronising: at the next scatter call, or by check_scatter_status().
_PENDING: list = []


def _poll_status() -> None:
    keep = []
    try:
        for status, n in _PENDING:
            bad = int(status[0])
            if bad:
                raise IndexError(f"scatter: {bad} indices outside [0, {n}); such rows were routed to row 0, the result is not valid")
        keep = _PENDING[-8:]
    finally:
        _PENDING[:] = keep


def check_scatter_status(device=None) -> None:
    """Synchronises and raises IndexError if any scatter call issued so far saw an out-of-range index."""
    torch.cuda.synchronize(device)
    _poll_status()


def scatter(src, index, dim: int = -1, out=None, dim_size: Optional[int] = None, reduce: str = "sum") -> torch.Tensor:
    if out is not None:
        raise NotImplementedError("scatter(out=...) is not used by the reference hot path")
    if reduce not in N.REDUCE:
        raise ValueError(f"unknown reduce {reduce!r}")
    return _run(src, index, dim, dim_size, reduce, False)[0]


def scatter_sum(src, index, dim: int = -1, out=None, dim_size: Optional[int] = None) -> torch.Tensor:
    return scatter(src, index, dim, out, dim_size, "sum")


scatter_add = scatter_sum


def scatter_mean(src, index, dim: int = -1, out=None, dim_size: Optional[int] = None) -> torch.Tensor:
    return scatter(src, index, dim, out, dim_size, "mean")


def scatter_max(src, index, dim: int = -1, out=None, dim_size: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    assert out is None
    return _run(src, index, dim, dim_size, "max", True)


def scatter_min(src, index, dim: int = -1, out=None, dim_size: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    assert out is None
    return _run(src, index, dim, dim_size, "min", True)
