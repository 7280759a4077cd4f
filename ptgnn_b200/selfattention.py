"""``MultiHeadSelfAttentionMessagePassing`` with the reference's ``nn.Module`` API, on the native chunked attention kernel.

Counterpart of `ptgnn/neuralmodels/gnn/messagepassing/selfattmessagepassing.py:9-136` of the reference: a transformer layer among
the nodes of each graph.  With ``t = x W_qkv^T`` viewed as ``[R, heads, 2 dk + dv]`` (head block ``[a | b | v]``), row ``i`` attends
with ``a_i`` over the ``b_j`` of the rows of its chunk, ``o_i = sum_j softmax_j(a_i . b_j / sqrt(dk)) v_j``; graph ``g`` owns the row
range ``[off_g, off_g + c_g)`` (``c_g`` = the number of nodes with id ``g``, ``off`` their prefix sum: the ranges come from the
counts, as in the reference, also for an unsorted ``node_to_graph_idx``), cut into chunks of ``max_num_nodes`` rows.  Then
``y1 = LN1(o W_sum^T + x)``, ``y2 = LN2(W_out relu(W_int y1 + b_int) + b_out + y1)``.

* The node-sized products run on the native dense ``linear`` (the intermediate one with its bias and ReLU fused), the attention on
  ``ptgnn_b200_selfatt_forward`` (DESIGN.md §3.8: the ``[L, L]`` scores never reach memory), LayerNorms and residuals as library ops.
* bf16 states: the products run on up-cast rows and ``t`` is rounded to bf16 for the kernel; the layer returns the input dtype.
* Gradients (fp32): ``_SelfAttentionFn`` around the kernel (saves ``t``, ``o`` and ``lse``) with ``_LinearFn`` and differentiable
  torch ops for the rest.
* The graph count is the container's ``num_graphs`` when it handed one over (then a call makes no host synchronisation), else
  ``max + 1`` read once per ``node_to_graph_idx`` tensor.

Not supported (``NotImplementedError``): training-mode dropout with ``p > 0``, gradients with bf16 states, node-range shards
(``gather_states``), ``target_reference != "all"``, and dimensions outside ``dk, dv in {16, 32, 64, 128}``.
"""
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F_
from torch import nn

from . import _native as N
from .edgeplan import EdgePlan
from .messagepassing import AbstractMessagePassingLayer, _check_shape
from .reduceops import graph_states

_RELU = nn.ReLU()
_DIMS = "dk and dv in {16, 32, 64, 128}"


def _qkv(t: torch.Tensor, plan: EdgePlan, heads: int, dk: int, dv: int) -> Tuple[torch.Tensor, bool, int]:
    t, bf16, rows, _ = graph_states(t, plan, "qkv")
    _check_shape(t, (rows, heads * (2 * dk + dv)), "qkv")
    return t, bf16, rows


def native_selfatt(t: torch.Tensor, plan: EdgePlan, heads: int, dk: int, dv: int, max_chunk: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``ptgnn_b200_selfatt_forward``: (o [R, heads * dv] in t's dtype, lse [R, heads] fp32) for t [R, heads * (2 dk + dv)] fp32 or bf16
    and the plan of the node -> graph map."""
    t, bf16, rows = _qkv(t, plan, heads, dk, dv)
    lib = N.lib()
    if not lib.ptgnn_b200_selfatt_supported(int(bf16), dk, dv):
        raise NotImplementedError(f"the self-attention kernel takes {_DIMS}, got dk={dk}, dv={dv}")
    G = plan.num_nodes
    ws_bytes = lib.ptgnn_b200_selfatt_workspace_bytes(rows, G, heads)
    o = torch.empty(rows, heads * dv, dtype=t.dtype, device=t.device)
    lse = torch.empty(rows, heads, dtype=torch.float32, device=t.device)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=t.device)
    N.call("ptgnn_b200_selfatt_forward", t.device, int(bf16), N.ptr(t), rows, heads, dk, dv, N.ptr(plan.row_ptr), G, int(max_chunk), N.ptr(o),
           N.ptr(lse), plan.status.data_ptr() + 4, N.ptr(ws), ws_bytes)
    return o, lse


def native_selfatt_backward(t: torch.Tensor, plan: EdgePlan, heads: int, dk: int, dv: int, max_chunk: int, o: torch.Tensor,
                            lse: torch.Tensor, d_o: torch.Tensor) -> torch.Tensor:
    """``ptgnn_b200_selfatt_backward_f32``: d t [R, heads * (2 dk + dv)] from d o [R, heads * dv].  fp32."""
    t, _, rows = _qkv(N.require_cuda(t, "qkv", torch.float32), plan, heads, dk, dv)
    o, d_o = N.require_cuda(o, "o", torch.float32), N.require_cuda(d_o, "d_o", torch.float32)
    lse = N.require_cuda(lse, "lse", torch.float32)
    for x, n, shape in ((o, "o", (rows, heads * dv)), (d_o, "d_o", (rows, heads * dv)), (lse, "lse", (rows, heads))):
        _check_shape(x, shape, n)
    lib = N.lib()
    if not lib.ptgnn_b200_selfatt_supported(0, dk, dv):
        raise NotImplementedError(f"the self-attention kernel takes {_DIMS}, got dk={dk}, dv={dv}")
    G = plan.num_nodes
    ws_bytes = lib.ptgnn_b200_selfatt_workspace_bytes(rows, G, heads)
    d_t = torch.empty_like(t)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=t.device)
    N.call("ptgnn_b200_selfatt_backward_f32", t.device, N.ptr(t), rows, heads, dk, dv, N.ptr(plan.row_ptr), G, int(max_chunk), N.ptr(o),
           N.ptr(lse), N.ptr(d_o), N.ptr(d_t), N.ptr(ws), ws_bytes)
    return d_t


class MultiHeadSelfAttentionMessagePassing(AbstractMessagePassingLayer):
    """
    A transformer layer among all nodes in a graph.
    """

    def __init__(
        self,
        input_state_dimension: int,
        key_query_dimension: int,
        value_dimension: int,
        output_dimension: int,
        intermediate_dimension: int,
        num_heads: int,
        dropout_rate: float = 0.0,
        target_reference: str = "all",
        max_num_nodes: int = 250,
    ):
        super().__init__()
        self.__num_heads = num_heads
        self.__key_query_dim = key_query_dimension
        self.__value_dim = value_dimension
        self.__selfatt_head_transforms = nn.Linear(
            in_features=input_state_dimension, out_features=num_heads * (2 * key_query_dimension + value_dimension), bias=False
        )
        self.__summarization_layer = nn.Linear(in_features=num_heads * value_dimension, out_features=output_dimension, bias=False)
        self.__intermediate_layer = nn.Linear(in_features=output_dimension, out_features=intermediate_dimension)
        self.__output_layer = nn.Linear(in_features=intermediate_dimension, out_features=output_dimension)
        self.__layer_norm1 = nn.LayerNorm(output_dimension)
        self.__layer_norm2 = nn.LayerNorm(output_dimension)
        self.__dropout_layer = nn.Dropout(p=dropout_rate)
        self.__target_reference = target_reference
        self.__max_num_nodes = max_num_nodes

    def forward(
        self,
        node_states: torch.Tensor,
        adjacency_lists: List[Tuple[torch.Tensor, torch.Tensor]],
        node_to_graph_idx: torch.Tensor,
        reference_node_ids: Dict[str, torch.Tensor] = None,
        reference_node_graph_idx: Dict[str, torch.Tensor] = None,
        edge_features: List[torch.Tensor] = None,
        gather_states: Optional[torch.Tensor] = None,
    ) -> torch.Tensor:
        from . import autograd as _ag
        from . import composed as C
        from .globalexchange import per_graph_layer_plan

        name = type(self).__name__
        if self.__target_reference != "all":
            raise NotImplementedError(f"{name}: target_reference other than 'all' (the reference's branch adds all node states to the "
                                      "referenced rows and only works when every node is referenced)")
        if self.training and self.__dropout_layer.p > 0:
            raise NotImplementedError(f"{name}: training-mode dropout with p > 0 (the mask on the attention probabilities)")
        heads, dk, dv = self.__num_heads, self.__key_query_dim, self.__value_dim
        if not N.lib().ptgnn_b200_selfatt_supported(int(node_states.dtype == torch.bfloat16), dk, dv):
            raise NotImplementedError(f"{name}: the self-attention kernel takes {_DIMS}, got dk={dk}, dv={dv}")
        if self.__max_num_nodes < 1:
            raise ValueError(f"{name}: max_num_nodes must be >= 1, got {self.__max_num_nodes}")
        plan, grad, bf16 = per_graph_layer_plan(self, node_states, node_to_graph_idx, gather_states, self.input_state_dimension)
        x = node_states.to(torch.float32)
        linear = _ag._LinearFn.apply if grad else C.linear
        t = linear(x, self.__selfatt_head_transforms.weight, None)
        if grad:
            o = _ag.selfatt_with_grad(plan, heads, dk, dv, self.__max_num_nodes, t)
        else:
            o = native_selfatt(t.to(torch.bfloat16) if bf16 else t, plan, heads, dk, dv, self.__max_num_nodes)[0].to(torch.float32)
        plan.poll()
        ln1, ln2 = self.__layer_norm1, self.__layer_norm2
        y1 = F_.layer_norm(self.__dropout_layer(linear(o, self.__summarization_layer.weight, None)) + x, ln1.normalized_shape, ln1.weight,
                           ln1.bias, ln1.eps)
        inter = self.__intermediate_layer
        if grad:
            hidden = F_.relu(linear(y1, inter.weight, inter.bias))
        else:
            hidden = C.linear(y1, inter.weight, inter.bias, _RELU)
        out = self.__dropout_layer(linear(hidden, self.__output_layer.weight, self.__output_layer.bias))
        y2 = F_.layer_norm(out + y1, ln2.normalized_shape, ln2.weight, ln2.bias, ln2.eps)
        return y2.to(node_states.dtype)

    @property
    def input_state_dimension(self) -> int:
        return self.__selfatt_head_transforms.in_features

    @property
    def output_state_dimension(self) -> int:
        return self.__output_layer.out_features
