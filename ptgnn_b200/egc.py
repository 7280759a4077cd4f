"""``EGCMessagePassingLayer`` (EGC-S with per-edge-type bases) on the native operators -- SURVEY.md §8 row f-4.

Same constructor, attribute names (hence ``state_dict`` keys) and forward contract as
`/root/reference/ptgnn/neuralmodels/gnn/messagepassing/egcmessagepassing.py:8-99`.  The layer is the hot path's
gather -> per-type Linear -> scatter with a wider message (``num_bases * output_state_dimension`` columns, :75-83), followed by a
per-node combination of the aggregated bases with weights from one more Linear (:64-66, :90).

* Fused path (DESIGN.md §3.14), wherever ``ptgnn_b200_egc_supported`` takes the dimensions: the message features are cut into slabs
  of 128, each one launch of the fused aggregation kernel whose write-out sums the bases of its output columns -- no
  ``[E, bases * out]`` message tensor.  fp32 states (3xFP16, fp32-exact) and bf16 states (bf16 output, rounded where autocast
  rounds); fp32 states train through ``autograd._EgcLayerFunction``.
* Composed path, every other shape, and fp32 states under ``PTGNN_B200_FP32_MODE=tf32``: the stand-alone native kernels
  (``edge_messages``, ``segment_reduce``, ``linear``) and a node-sized pointwise combination.  Forward only; fp32 states.

Training-mode dropout with ``p > 0`` (a mask on the gathered ``[E_t, H]`` rows, :76) has no native path and raises.
"""
import ctypes
from typing import Dict, List, Tuple

import torch
from torch import nn

from . import _native as N
from . import composed as C
from .messagepassing import AbstractMessagePassingLayer, _check_shape, _check_states, _reduce_code, _refuse_autograd, fused_allowed


def use_fused(lib, bf16: bool, in_dim: int, out: int, heads: int, bases: int) -> bool:
    """The fused slabs wherever the library takes the dimensions; PTGNN_B200_FP32_MODE=tf32 selects the composed path for fp32
    states, as it selects the round-1 path for the other layers."""
    return fused_allowed(bf16) and bool(lib.ptgnn_b200_egc_supported(int(bf16), in_dim, out, heads, bases))


class EGCMessagePassingLayer(AbstractMessagePassingLayer):
    def __init__(self, input_state_dimension: int, output_state_dimension: int, num_edge_types: int, message_aggregation_function: str,
                 num_bases: int = 4, num_heads: int = 8, dropout_rate: float = 0.0):
        super().__init__()
        if output_state_dimension % num_heads != 0:
            raise AssertionError("output_state_dimension must be a multiple of num_heads")
        self._dims = (int(input_state_dimension), int(output_state_dimension), int(num_heads), int(num_bases))
        self._reduce_name = message_aggregation_function
        self._drop_p = float(dropout_rate)
        # the two parameter holders keep the reference's (name-mangled) attribute names and construction order: identical
        # state_dict keys, identical parameters for the same seed
        self.__bases = nn.ModuleList(nn.Linear(input_state_dimension, num_bases * output_state_dimension, bias=False) for _ in range(num_edge_types))
        self.__weight_coeffs = nn.Linear(input_state_dimension, num_heads * num_bases)

    def forward(self, node_states: torch.Tensor, adjacency_lists: List[Tuple[torch.Tensor, torch.Tensor]],
                node_to_graph_idx: torch.Tensor = None, reference_node_ids: Dict[str, torch.Tensor] = None,
                reference_node_graph_idx: Dict[str, torch.Tensor] = None, edge_features: List[torch.Tensor] = None) -> torch.Tensor:
        from . import autograd as _ag

        in_dim, out, heads, bases = self._dims
        assert len(adjacency_lists) == len(self.__bases)
        if self.training and self._drop_p > 0:
            raise NotImplementedError("EGCMessagePassingLayer: training-mode dropout has no native path")
        reduce = _reduce_code(self._reduce_name)
        bf16 = node_states.dtype == torch.bfloat16
        fused = use_fused(N.lib(), bf16, in_dim, out, heads, bases)
        coeff = self.__weight_coeffs
        if _ag.needs_grad(self, node_states):
            if bf16 or not fused:
                _refuse_autograd(self, node_states)
            _check_states(node_states, in_dim, "EGCMessagePassingLayer")
            return _ag.egc_forward_with_grad(self, node_states, adjacency_lists, self._reduce_name, coeff.weight, coeff.bias,
                                             [b.weight for b in self.__bases])
        if node_states.dtype != torch.float32 and not (bf16 and fused):
            raise NotImplementedError("EGCMessagePassingLayer: bf16 states need a shape the fused kernel takes; otherwise fp32 states only")
        _check_states(node_states, in_dim, "EGCMessagePassingLayer")
        h = N.require_cuda(node_states, "node_states", node_states.dtype)
        n = h.shape[0]
        plan = self._plan(adjacency_lists, n, None)
        if fused:
            return self._forward_fused(h, plan, reduce, bf16)
        node_weights = C.linear(h, coeff.weight, coeff.bias).reshape(n, heads, bases, 1)                                   # :64-66
        messages = C.edge_messages(plan, h, None, [b.weight for b in self.__bases], False)        # [E, bases * out]           :75-83
        aggregated = C.segment_reduce(messages, plan, reduce).reshape(n, heads, bases, out // heads)                        # :85-89
        return (aggregated * node_weights).sum(dim=-2).reshape(n, out)                                                      # :90

    def _forward_fused(self, h: torch.Tensor, plan, reduce: int, bf16: bool) -> torch.Tensor:
        in_dim, out, heads, bases = self._dims
        n, T = h.shape[0], plan.num_types
        weights = [N.require_cuda(b.weight, "bases weight", torch.float32) for b in self.__bases]
        cw = N.require_cuda(self.__weight_coeffs.weight, "weight_coeffs.weight", torch.float32)
        cb = N.require_cuda(self.__weight_coeffs.bias, "weight_coeffs.bias", torch.float32)
        for i, w in enumerate(weights):      # raw pointers cross the C ABI next: the shapes must be what the kernels assume
            _check_shape(w, (bases * out, in_dim), f"bases[{i}].weight")
        _check_shape(cw, (heads * bases, in_dim), "weight_coeffs.weight"); _check_shape(cb, (heads * bases,), "weight_coeffs.bias")
        lib = N.lib()
        # the packed slabs (fp16 hi | lo' or bf16, in the kernel's order): once per parameter version in eval mode
        kind = "egc_bf16_fused" if bf16 else "egc_f32_fused"
        cache, valid = self._weight_cache(kind, lib.ptgnn_b200_egc_fused_weight_cache_bytes(int(bf16), T, in_dim, out, heads, bases), weights,
                                          h.device)
        ws_bytes = lib.ptgnn_b200_egc_fused_workspace_bytes(int(bf16), n, T, in_dim, out, heads, bases)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=h.device)
        result = torch.empty(n, out, dtype=h.dtype, device=h.device)
        bp = plan.block_plan()
        N.call("ptgnn_b200_egc_forward_fused", h.device, int(bf16), N.ptr(h), n, in_dim, out, heads, bases, T, ctypes.byref(bp),
               N.ptr(plan.row_ptr), N.ptr_table(weights), N.ptr(cw), N.ptr(cb), reduce, N.ptr(result), N.ptr(ws), ws_bytes, N.ptr(cache),
               0 if cache is None else cache.numel(), int(valid))
        self._weight_cache_filled(kind, h.device)
        return result

    @property
    def input_state_dimension(self) -> int:
        return self._dims[0]

    @property
    def output_state_dimension(self) -> int:
        return self._dims[1]
