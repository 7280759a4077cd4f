"""Importable stand-in for the third-party ``torch_scatter`` package, backed by the native segmented-reduce kernels.

The reference imports ``torch_scatter`` by name (`/root/reference/ptgnn/neuralmodels/gnn/messagepassing/abstractmessagepassing.py:4`,
``pna_aggregation.py:3``, ``graphnorm.py:3``, ``reduceops/varsizedsummary.py:7``, ``implementations/varmisuse/varmisuse.py:8``,
``sequence/grucopydecoder.py:9-10``).  ``ptgnn_b200.overlay.install()`` registers this package as ``sys.modules['torch_scatter']``
when the real wheel is absent (or when asked to), so those modules import unchanged.

Semantics follow torch_scatter 2.0.x (SURVEY.md Appendix A): ``dim_size`` defaults to ``index.max() + 1``; ``max``/``min`` return
``(out, arg)``, untouched rows are 0 with ``arg == src.size(dim)``, ties go to the first occurrence.  CUDA tensors only (no CPU
fallback); fp32 arithmetic (other floating dtypes are computed in fp32 and cast back, as the reference's hot path does).
Shapes the kernels do not take directly -- reduction along a dimension other than 0, 1-D inputs, row widths that are not a
multiple of 4 -- are brought to ``[E, D]`` form by a transpose / zero-padding around the same kernels.
"""
import importlib
from typing import Optional, Tuple

import torch

# the submodule itself: the package attribute `ptgnn_b200.scatter` is re-bound to the function of that name by ptgnn_b200/__init__
_native = importlib.import_module("..scatter", __package__)

__version__ = "2.0.9+ptgnn_b200"


def _to_rows(src: torch.Tensor, index: torch.Tensor, dim: int):
    """-> (rows [E, D4] fp32 contiguous, index [E], restore(out_rows [N, D4]) -> tensor shaped like src with size N along dim)."""
    if dim < 0:
        dim += src.dim()
    if index.dim() != 1:
        # torch_scatter broadcasts `index` to src's shape; the reference only ever passes 1-D indices along `dim`
        if index.shape == src.shape:
            moved_i = index.movedim(dim, 0).reshape(src.shape[dim], -1)
            if not bool((moved_i == moved_i[:, :1]).all()):
                raise NotImplementedError("torch_scatter shim: index must be constant across the non-reduced dimensions")
            index = moved_i[:, 0]
        else:
            raise NotImplementedError("torch_scatter shim: index must be 1-D (or already broadcast to src's shape)")
    moved = src.movedim(dim, 0)
    tail_shape = moved.shape[1:]
    rows = moved.reshape(moved.shape[0], -1).to(torch.float32)
    D = rows.shape[1]
    pad = (-D) % 4
    if pad:
        rows = torch.cat([rows, rows.new_zeros(rows.shape[0], pad)], dim=1)
    rows = rows.contiguous()

    def restore(out_rows: torch.Tensor, dtype=src.dtype) -> torch.Tensor:
        out = out_rows[:, :D].reshape((out_rows.shape[0],) + tuple(tail_shape)).movedim(0, dim)
        return out.to(dtype)

    return rows, index.contiguous(), restore


_MAX_ROW = 512   # widest row the segmented-reduce kernels take in one launch


def _chunked(fn, rows: torch.Tensor):
    """Applies fn to column chunks of at most _MAX_ROW floats and concatenates the results (tuples element-wise)."""
    if rows.shape[1] <= _MAX_ROW:
        return fn(rows)
    parts = [fn(rows[:, c:c + _MAX_ROW].contiguous()) for c in range(0, rows.shape[1], _MAX_ROW)]
    if isinstance(parts[0], tuple):
        return tuple(torch.cat([p[i] for p in parts], dim=1) for i in range(len(parts[0])))
    return torch.cat(parts, dim=1)


def _dim_size(index: torch.Tensor, dim_size: Optional[int]) -> int:
    if dim_size is not None:
        return int(dim_size)
    return int(index.max().item()) + 1 if index.numel() else 0


def scatter(src: torch.Tensor, index: torch.Tensor, dim: int = -1, out: Optional[torch.Tensor] = None,
            dim_size: Optional[int] = None, reduce: str = "sum") -> torch.Tensor:
    if out is not None:
        raise NotImplementedError("torch_scatter shim: scatter(out=...) is not supported")
    if reduce in ("mul",):
        raise NotImplementedError("torch_scatter shim: reduce='mul' has no native kernel")
    if reduce == "add":
        reduce = "sum"
    rows, idx, restore = _to_rows(src, index, dim)
    n = _dim_size(idx, dim_size)
    return restore(_chunked(lambda r: _native.scatter(r, idx, dim=0, dim_size=n, reduce=reduce), rows))


def scatter_sum(src, index, dim: int = -1, out=None, dim_size: Optional[int] = None) -> torch.Tensor:
    return scatter(src, index, dim, out, dim_size, "sum")


scatter_add = scatter_sum


def scatter_mean(src, index, dim: int = -1, out=None, dim_size: Optional[int] = None) -> torch.Tensor:
    return scatter(src, index, dim, out, dim_size, "mean")


def _with_arg(src, index, dim, dim_size, which) -> Tuple[torch.Tensor, torch.Tensor]:
    rows, idx, restore = _to_rows(src, index, dim)
    fn = _native.scatter_max if which == "max" else _native.scatter_min
    n = _dim_size(idx, dim_size)
    out, arg = _chunked(lambda r: fn(r, idx, dim=0, dim_size=n), rows)
    return restore(out), restore(arg, torch.int64)


def scatter_max(src, index, dim: int = -1, out=None, dim_size: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    assert out is None, "torch_scatter shim: scatter_max(out=...) is not supported"
    return _with_arg(src, index, dim, dim_size, "max")


def scatter_min(src, index, dim: int = -1, out=None, dim_size: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    assert out is None, "torch_scatter shim: scatter_min(out=...) is not supported"
    return _with_arg(src, index, dim, dim_size, "min")


from .composite import scatter_log_softmax, scatter_logsumexp, scatter_softmax, scatter_std  # noqa: E402,F401

__all__ = ["scatter", "scatter_sum", "scatter_add", "scatter_mean", "scatter_max", "scatter_min", "scatter_softmax",
           "scatter_log_softmax", "scatter_logsumexp", "scatter_std"]
