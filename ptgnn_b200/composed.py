"""The *composed* path: reference configurations the fused layer entry points do not cover, assembled from the stand-alone native
pieces of the C ABI (``ptgnn_b200_edge_messages_f32``, ``ptgnn_b200_linear_f32``, ``ptgnn_b200_segment_reduce_f32``,
``ptgnn_b200_grucell_f32``):

* edge features, ``F > 0`` (`/root/reference/ptgnn/neuralmodels/gnn/messagepassing/gatedmessagepassing.py:16,22,59`,
  ``mlpmessagepassing.py:27,41,97``): ``W_t [h_src ; h_tgt ; f_e] = W_t[:, :K] [h_src ; h_tgt] + W_t[:, K:] f_e`` -- the state part is
  the gathered-row GEMM of the message kernel, the feature part one dense GEMM per edge type over the contiguous ``[E_t, F]`` rows;
* message MLPs with hidden layers and / or biases (``mlp.py:50-77``): first layer as above, later layers as per-type dense GEMMs;
* module aggregators -- any ``AbstractMessageAggregation`` such as the reference's ``PnaMessageAggregation``
  (``pna_aggregation.py:27-56``): it receives the ``[E, D]`` messages in the reference's order (``cat`` over types) and the
  concatenated targets, exactly what ``mlpmessagepassing.py:100-112`` passes; its own ``torch_scatter`` calls resolve to the native
  segmented reduce through ``ptgnn_b200.torch_scatter_shim``.

fp32 only (``edge_messages`` and ``aggregate`` also take bf16 rows, for the bf16 Mlp backward); the ``[E, D]`` message tensor IS materialised here (these are the slow, general configurations -- none of the reference's
implementations uses them by default); the tail of an Mlp layer (activation, LayerNorm, dense, of whatever width the aggregator
produced) runs as the module's own device-side torch ops.
"""
from typing import List, Optional, Sequence

import torch
import torch.nn.functional as F_
from torch import nn

from . import _native as N
from .edgeplan import EdgePlan

_ACT = {type(None): N.ACT_NONE, nn.GELU: N.ACT_GELU, nn.Tanh: N.ACT_TANH, nn.ReLU: N.ACT_RELU, nn.Identity: N.ACT_NONE}


def _pad4(t: torch.Tensor) -> torch.Tensor:
    """Zero-pads the last dimension to a multiple of 4 (the kernels move 16-byte pieces)."""
    pad = (-t.shape[-1]) % 4
    return F_.pad(t, (0, pad)) if pad else t


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, activation: Optional[nn.Module] = None) -> torch.Tensor:
    """``activation(x @ weight.T + bias)`` on the native dense kernel; activations without a native code run as torch ops."""
    x = N.require_cuda(x, "x", torch.float32)
    rows, k = x.shape
    n_out = weight.shape[0]
    act_code = _ACT.get(type(activation))
    post = None if act_code is not None else activation
    xw, ww = _pad4(x), _pad4(N.require_cuda(weight, "weight", torch.float32))
    n_pad = (-n_out) % 4
    if n_pad:
        ww = F_.pad(ww, (0, 0, 0, n_pad))
        bias = None if bias is None else F_.pad(bias, (0, n_pad))
    xw, ww = xw.contiguous(), ww.contiguous()
    b = None if bias is None else N.require_cuda(bias, "bias", torch.float32)
    out = torch.empty(rows, n_out + n_pad, dtype=torch.float32, device=x.device)
    lib = N.lib()
    ws_bytes = lib.ptgnn_b200_linear_workspace_bytes(xw.shape[1], n_out + n_pad)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=x.device)
    N.call("ptgnn_b200_linear_f32", x.device, N.ptr(xw), rows, xw.shape[1], N.ptr(ww), N.ptr(b), n_out + n_pad, act_code or N.ACT_NONE,
           N.ptr(out), N.ptr(ws), ws_bytes)
    out = out[:, :n_out] if n_pad else out
    return post(out) if post is not None else out


def edge_messages(plan: EdgePlan, source_rows: torch.Tensor, target_rows: Optional[torch.Tensor], weights: Sequence[torch.Tensor],
                  use_target: bool) -> torch.Tensor:
    """``[E, D]`` fp32 messages in the reference's row order (cat over edge types): row e = W_t(e) [source_rows[src(e)] ; target_rows[tgt(e)]].
    bf16 rows: the bf16 messages of the three-kernel path (bf16 products, fp32 accumulation, rounded to bf16), up-cast."""
    D = weights[0].shape[0]
    E = plan.num_edges
    bf16 = source_rows.dtype == torch.bfloat16
    out = torch.empty(E, D, dtype=torch.bfloat16 if bf16 else torch.float32, device=source_rows.device)
    if E == 0:
        return out.float()
    ident = torch.arange(E, dtype=torch.int32, device=source_rows.device)
    ws_list = [N.require_cuda(w, "edge weight", torch.float32) for w in weights]
    lib = N.lib()
    H = source_rows.shape[1]
    if bf16:
        ws_bytes = lib.ptgnn_b200_edge_messages_bf16_workspace_bytes(plan.num_types, H, D, int(use_target))
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=source_rows.device)
        N.call("ptgnn_b200_edge_messages_bf16", source_rows.device, N.ptr(source_rows), N.ptr(target_rows), H, D, plan.num_types,
               plan.type_off_c, N.ptr(plan.src32), N.ptr(plan.tgt32), N.ptr(ident), N.ptr_table(ws_list), int(use_target), N.ptr(out),
               N.ptr(ws), ws_bytes)
        return out.float()
    ws_bytes = lib.ptgnn_b200_edge_messages_workspace_bytes(plan.num_types, H, D, int(use_target))
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=source_rows.device)
    N.call("ptgnn_b200_edge_messages_f32", source_rows.device, N.ptr(source_rows), N.ptr(target_rows), H, D, plan.num_types, plan.type_off_c,
           N.ptr(plan.src32), N.ptr(plan.tgt32), N.ptr(ident), N.ptr_table(ws_list), int(use_target), N.ptr(out), N.ptr(ws), ws_bytes)
    return out


def segment_reduce(messages: torch.Tensor, plan: EdgePlan, reduce_code: int, return_arg: bool = False):
    """torch_scatter.scatter(messages, targets, dim=0, dim_size=N, reduce) over the plan's target-sorted CSR (messages in edge order).
    return_arg (max / min): also the [N, D] int64 edge id of each winning message (E for empty targets, torch_scatter's sentinel)."""
    E, D = messages.shape
    out = torch.empty(plan.num_nodes, D, dtype=torch.float32, device=messages.device)
    arg = torch.empty(plan.num_nodes, D, dtype=torch.int64, device=messages.device) if return_arg else None
    N.call("ptgnn_b200_segment_reduce_f32", messages.device, N.ptr(messages), N.ptr(plan.row_ptr), N.ptr(plan.perm) if E else None,
           plan.num_nodes, E, D, reduce_code, N.ptr(out), N.ptr(arg))
    return (out, arg) if return_arg else out


def aggregate(plan: EdgePlan, source_rows: torch.Tensor, weights: Sequence[torch.Tensor], reduce_code: int, use_target: bool = False) -> torch.Tensor:
    """``reduce_{e -> v} W_type(e) source_rows[src(e)]`` as [num_nodes, D] fp32: the fused gather -> Linear -> segmented-reduce kernel
    where it takes the dimensions (D == 128, K in {64, 128}: no [E, D] message tensor), else ``edge_messages`` + ``segment_reduce``.
    Used by the backward passes (aggregate re-computation; d h_src on the transposed graph).  bf16 rows: the aggregate the bf16 layer
    forward computes (messages rounded to bf16, fp32 reduction) on the same kernels as that forward, before any rounding of its own;
    use_target (bf16 only): the messages read [source_rows[src(e)] ; source_rows[tgt(e)]]."""
    import ctypes

    from .messagepassing import _use_fused

    D = weights[0].shape[0]
    K = source_rows.shape[1]
    lib = N.lib()
    if source_rows.dtype == torch.bfloat16:
        if plan.num_edges == 0 or not _use_fused(lib, True, K, D):
            return segment_reduce(edge_messages(plan, source_rows, source_rows if use_target else None, weights, use_target), plan, reduce_code)
        ws_list = [N.require_cuda(w, "edge weight", torch.float32) for w in weights]
        ws_bytes = lib.ptgnn_b200_fused_aggregate_bf16_workspace_bytes(plan.num_types, K, int(use_target))
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=source_rows.device)
        out = torch.empty(plan.num_nodes, D, dtype=torch.float32, device=source_rows.device)
        N.call("ptgnn_b200_fused_aggregate_bf16", source_rows.device, N.ptr(source_rows), plan.num_nodes, K, plan.num_types,
               ctypes.byref(plan.block_plan()), N.ptr(plan.row_ptr), N.ptr_table(ws_list), int(use_target), reduce_code, N.ptr(out),
               N.ptr(ws), ws_bytes)
        return out
    if plan.num_edges == 0 or not _use_fused(lib, False, K, D):
        return segment_reduce(edge_messages(plan, source_rows, None, weights, False), plan, reduce_code)
    rows = N.require_cuda(source_rows, "source_rows", torch.float32)
    ws_list = [N.require_cuda(w, "edge weight", torch.float32) for w in weights]
    n = plan.num_nodes
    ws_bytes = lib.ptgnn_b200_mlp_fused_workspace_bytes(0, n, n, plan.num_types, K, D, D, 0)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=rows.device)
    out = torch.empty(n, D, dtype=torch.float32, device=rows.device)
    bp = plan.block_plan()
    # the Mlp entry point without activation / LayerNorm / dense layer = the bare aggregation
    N.call("ptgnn_b200_mlp_forward_fused", rows.device, 0, N.ptr(rows), None, n, n, K, D, D, plan.num_types, ctypes.byref(bp),
           N.ptr(plan.row_ptr), N.ptr_table(ws_list), 0, reduce_code, N.ACT_NONE, None, None, 0.0, None, None, N.ACT_NONE, N.ptr(out),
           N.ptr(ws), ws_bytes, None, 0, 0)
    return out


def grucell(inp: torch.Tensor, hidden: torch.Tensor, gru: nn.GRUCell) -> torch.Tensor:
    rows, H = hidden.shape
    D = inp.shape[1]
    out = torch.empty_like(hidden)
    lib = N.lib()
    ws_bytes = lib.ptgnn_b200_grucell_workspace_bytes(H, D)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=hidden.device)
    p = [N.require_cuda(t, "gru parameter", torch.float32) for t in (gru.weight_ih, gru.weight_hh, gru.bias_ih, gru.bias_hh)]
    N.call("ptgnn_b200_grucell_f32", hidden.device, N.ptr(inp.contiguous()), N.ptr(hidden), rows, H, D, N.ptr(p[0]), N.ptr(p[1]), N.ptr(p[2]),
           N.ptr(p[3]), N.ptr(out), N.ptr(ws), ws_bytes)
    return out


def _edge_feature_list(edge_features: Optional[List[torch.Tensor]], plan: EdgePlan, feature_dim: int, device) -> List[Optional[torch.Tensor]]:
    if feature_dim == 0:
        return [None] * plan.num_types
    if edge_features is None or len(edge_features) != plan.num_types:
        raise ValueError("one [E_t, F] edge-feature tensor per edge type is required")
    out = []
    for t, f in enumerate(edge_features):
        e_t = plan.type_off[t + 1] - plan.type_off[t]
        if f.dim() != 2 or f.shape[0] != e_t or f.shape[1] != feature_dim:
            raise ValueError(f"edge_features[{t}] must be [{e_t}, {feature_dim}], got {tuple(f.shape)}")
        out.append(N.require_cuda(f, f"edge_features[{t}]", torch.float32))
    return out


def first_layer_messages(plan: EdgePlan, h_src: torch.Tensor, h_tgt: Optional[torch.Tensor], weights: Sequence[torch.Tensor],
                         biases: Sequence[Optional[torch.Tensor]], feats: Sequence[Optional[torch.Tensor]], state_cols: int) -> torch.Tensor:
    """Row e of the result = W_t [h_src[src(e)] ; h_tgt[tgt(e)] ; f_e] + b_t, cat(types) order."""
    msg = edge_messages(plan, h_src, h_tgt, [w[:, :state_cols].contiguous() for w in weights], h_tgt is not None)
    for t in range(plan.num_types):
        lo, hi = plan.type_off[t], plan.type_off[t + 1]
        if hi == lo:
            continue
        if feats[t] is not None:
            msg[lo:hi] += linear(feats[t], weights[t][:, state_cols:])
        if biases[t] is not None:
            msg[lo:hi] += biases[t]
    return msg
