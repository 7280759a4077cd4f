"""Per-graph summaries of node states, with the reference's ``nn.Module`` API, on the native readout kernel.

Counterparts of `ptgnn/neuralmodels/reduceops/varsizedsummary.py:11-81` of the reference:

* ``ElementsToSummaryRepresentationInput`` -- the input record (embeddings, element -> sample map, number of samples);
* ``SimpleVarSizedElementReduce``          -- sum / mean on ``ptgnn_b200_graph_readout``; max / min on the native ``scatter``;
* ``WeightedSumVarSizedElementReduce``     -- ``sum_n sigmoid(x_n . w) x_n`` on ``ptgnn_b200_graph_readout``;
* ``SelfAttentionVarSizedElementReduce`` / ``MultiheadSelfAttentionVarSizedElementReduce`` (``:84-178``) -- a per-graph softmax
  readout on ``ptgnn_b200_attention_readout`` (DESIGN §3.7): the key and value layers are folded into G-row products, so the
  ``[N, hidden]`` keys and the ``[N, heads, D]`` products are never formed.  Forward in fp32 or bf16, gradients in fp32.

Constructor signatures and (name-mangled) ``state_dict`` keys are the reference's.  ``GruGlobalStateUpdate`` reads these modules
and the reference's own instances of the same two classes directly (``readout_of``), so the reference's factories need no change.
"""
import math
from abc import abstractmethod
from typing import NamedTuple, Optional, Tuple, Union

import torch
from torch import nn

from . import _native as N
from .edgeplan import EdgePlan, plan_for
from .messagepassing import _check_shape


class ElementsToSummaryRepresentationInput(NamedTuple):
    """Input to AbstractVarSizedElementReduce layers."""

    element_embeddings: torch.Tensor  # [num_elements, D] float
    element_to_sample_map: torch.Tensor  # [num_elements] int64, values in [0, num_samples)
    num_samples: Union[torch.Tensor, int]


class AbstractVarSizedElementReduce(nn.Module):
    """Interface for computing summary representations from multiple variable-sized sets of representations."""

    @abstractmethod
    def forward(self, inputs: ElementsToSummaryRepresentationInput) -> torch.Tensor:
        """Returns: float tensor of shape [num_samples, D']"""


def graph_plan(node_to_graph_idx: torch.Tensor, num_graphs: int) -> EdgePlan:
    """The nodes grouped by graph, in node order within each graph: the plan of the single edge list (n2g, n2g) with
    ``num_graphs`` targets.  Cached by tensor identity and version like the edge plans; graph ids outside [0, num_graphs)
    are reported through the plan's status words (IndexError at the next poll)."""
    n2g = N.require_cuda(node_to_graph_idx, "node_to_graph_idx", torch.int64)
    if n2g.dim() != 1:
        raise ValueError("node_to_graph_idx must be a 1-D tensor")
    return plan_for([(n2g, n2g)], int(num_graphs))


def graph_states(node_states: torch.Tensor, plan: EdgePlan, name: str = "node_states") -> Tuple[torch.Tensor, bool, int, int]:
    """The rows of a per-graph kernel's input, one per node of ``plan`` (``graph_plan``): (the contiguous CUDA tensor, bf16, N, D).
    bf16 stays bf16, anything else must be fp32."""
    bf16 = node_states.dtype == torch.bfloat16
    x = N.require_cuda(node_states, name, torch.bfloat16 if bf16 else torch.float32)
    if x.dim() != 2:
        raise ValueError(f"{name} must be [num_nodes, D], got {tuple(x.shape)}")
    num_nodes, D = x.shape
    if plan.num_edges != num_nodes:
        raise ValueError(f"node_to_graph_idx and {name} disagree on the number of nodes")
    return x, bf16, num_nodes, D


def native_readout(node_states: torch.Tensor, plan: EdgePlan, mode: int, gate_weight: Optional[torch.Tensor] = None,
                   want_gates: bool = False):
    """``ptgnn_b200_graph_readout``: (g [G, H] fp32, s [N] fp32 or None).  fp32 or bf16 states; H a multiple of 32 in [32, 256]."""
    x, bf16, num_nodes, H = graph_states(node_states, plan)
    G = plan.num_nodes
    lib = N.lib()
    ws_bytes = lib.ptgnn_b200_graph_readout_workspace_bytes(num_nodes, G, H)
    if ws_bytes == 0:
        raise NotImplementedError(f"the graph readout kernel takes H a multiple of 32 in [32, 256], got H={H}")
    w = None
    if mode == N.READOUT_WEIGHTED_SUM:
        w = N.require_cuda(gate_weight, "weights_layer.weight", torch.float32)
        _check_shape(w, (1, H), "weights_layer.weight")      # raw pointers cross the C ABI next
    g = torch.empty(G, H, dtype=torch.float32, device=x.device)
    s = torch.empty(num_nodes, dtype=torch.float32, device=x.device) if want_gates and w is not None else None
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=x.device)
    N.call("ptgnn_b200_graph_readout", x.device, int(bf16), N.ptr(x), num_nodes, H, N.ptr(plan.row_ptr), N.ptr(plan.perm) if num_nodes else None,
           G, N.ptr(w), mode, N.ptr(g), N.ptr(s), N.ptr(ws), ws_bytes)
    return g, s


def readout_of(module: nn.Module):
    """(kind, gate weight) for the reducers the native layer computes itself -- this module's classes and the reference's
    classes of the same names, recognised by class name and parameter layout -- else None (the module is called as is).
    kind: "weighted", "sum", "mean", "max" or "min"."""
    name = type(module).__name__
    if name == "WeightedSumVarSizedElementReduce":
        lin = getattr(module, "_WeightedSumVarSizedElementReduce__weights_layer", None)
        params = list(module.parameters())
        if isinstance(lin, nn.Linear) and lin.bias is None and lin.out_features == 1 and len(params) == 1:
            return "weighted", lin.weight
        return None
    if name == "SimpleVarSizedElementReduce":
        kind = getattr(module, "_SimpleVarSizedElementReduce__summarization_type", None)
        if kind in ("sum", "mean", "max", "min") and not list(module.parameters()):
            return kind, None
    return None


def reduce_states(kind: str, gate_weight: Optional[torch.Tensor], node_states: torch.Tensor, node_to_graph_idx: torch.Tensor,
                  plan: EdgePlan, want_gates: bool = False):
    """g [G, H] fp32 (and the gates s [N] of the weighted sum when asked for)."""
    if kind in ("max", "min"):     # the native two-level scatter (long segments) -- no separate kernel for these
        from .scatter import scatter

        return scatter(node_states.to(torch.float32), node_to_graph_idx, dim=0, dim_size=plan.num_nodes, reduce=kind), None
    mode = {"weighted": N.READOUT_WEIGHTED_SUM, "sum": N.READOUT_SUM, "mean": N.READOUT_MEAN}[kind]
    return native_readout(node_states, plan, mode, gate_weight, want_gates)


def _num_samples(inputs: ElementsToSummaryRepresentationInput) -> int:
    n = inputs.num_samples
    return int(n.item()) if isinstance(n, torch.Tensor) else int(n)


class SimpleVarSizedElementReduce(AbstractVarSizedElementReduce):
    def __init__(self, summarization_type: str):
        super().__init__()
        assert summarization_type in {"sum", "mean", "max", "min"}
        self.__summarization_type = summarization_type

    def forward(self, inputs: ElementsToSummaryRepresentationInput) -> torch.Tensor:
        if torch.is_grad_enabled() and inputs.element_embeddings.requires_grad:
            raise NotImplementedError("the stand-alone readout is forward-only: call it under torch.no_grad()")
        plan = graph_plan(inputs.element_to_sample_map, _num_samples(inputs))
        g, _ = reduce_states(self.__summarization_type, None, inputs.element_embeddings, inputs.element_to_sample_map, plan)
        plan.poll()
        return g.to(inputs.element_embeddings.dtype)


class WeightedSumVarSizedElementReduce(AbstractVarSizedElementReduce):
    def __init__(self, representation_size: int):
        super().__init__()
        self.__weights_layer = nn.Linear(representation_size, 1, bias=False)

    def forward(self, inputs: ElementsToSummaryRepresentationInput) -> torch.Tensor:
        if torch.is_grad_enabled() and (inputs.element_embeddings.requires_grad or self.__weights_layer.weight.requires_grad):
            raise NotImplementedError("the stand-alone readout is forward-only: call it under torch.no_grad()")
        plan = graph_plan(inputs.element_to_sample_map, _num_samples(inputs))
        g, _ = reduce_states("weighted", self.__weights_layer.weight, inputs.element_embeddings, inputs.element_to_sample_map, plan)
        plan.poll()
        return g.to(inputs.element_embeddings.dtype)


def native_attention_readout(node_states: torch.Tensor, plan: EdgePlan, qt: torch.Tensor, heads: int):
    """``ptgnn_b200_attention_readout``: (o [G, heads, D] fp32, lse [G, heads] fp32) with o[b, h] = sum_n softmax_n(x_n . qt[b, h]) x_n
    over the nodes of graph b.  fp32 or bf16 states; D in {32, 64, 128, 256}, heads in {1, 2, 4, 8}."""
    x, bf16, num_nodes, D = graph_states(node_states, plan)
    G = plan.num_nodes
    lib = N.lib()
    if not lib.ptgnn_b200_attention_readout_supported(int(bf16), D, heads):
        raise NotImplementedError(f"the attention readout kernel takes D in {{32, 64, 128, 256}} and heads in {{1, 2, 4, 8}}, got D={D}, heads={heads}")
    q = N.require_cuda(qt, "qt", torch.float32)
    _check_shape(q, (G, heads, D), "qt")        # raw pointers cross the C ABI next
    ws_bytes = lib.ptgnn_b200_attention_readout_workspace_bytes(num_nodes, G, D, heads)
    o = torch.empty(G, heads, D, dtype=torch.float32, device=x.device)
    lse = torch.empty(G, heads, dtype=torch.float32, device=x.device)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=x.device)
    N.call("ptgnn_b200_attention_readout", x.device, int(bf16), N.ptr(x), num_nodes, D, heads, N.ptr(plan.row_ptr),
           N.ptr(plan.perm) if num_nodes else None, G, N.ptr(q), N.ptr(o), N.ptr(lse), N.ptr(ws), ws_bytes)
    return o, lse


def native_attention_readout_backward(node_states: torch.Tensor, plan: EdgePlan, qt: torch.Tensor, o: torch.Tensor, lse: torch.Tensor,
                                      d_o: torch.Tensor):
    """``ptgnn_b200_attention_readout_backward_f32``: (d_x [N, D], d_qt [G, heads, D]) from d_o [G, heads, D].  fp32 states."""
    x, _, num_nodes, D = graph_states(N.require_cuda(node_states, "node_states", torch.float32), plan)
    G, heads = plan.num_nodes, qt.shape[1]
    tabs = [N.require_cuda(t, n, torch.float32) for t, n in ((qt, "qt"), (o, "o"), (d_o, "d_o"))]
    for t, n in zip(tabs, ("qt", "o", "d_o")):
        _check_shape(t, (G, heads, D), n)
    lse = N.require_cuda(lse, "lse", torch.float32)
    _check_shape(lse, (G, heads), "lse")
    lib = N.lib()
    ws_bytes = lib.ptgnn_b200_attention_readout_workspace_bytes(num_nodes, G, D, heads)
    if ws_bytes == 0:
        raise NotImplementedError(f"the attention readout kernel takes D in {{32, 64, 128, 256}} and heads in {{1, 2, 4, 8}}, got D={D}, heads={heads}")
    d_x = torch.empty_like(x)
    d_qt = torch.empty(G, heads, D, dtype=torch.float32, device=x.device)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
    N.call("ptgnn_b200_attention_readout_backward_f32", x.device, N.ptr(x), num_nodes, D, heads, N.ptr(plan.row_ptr),
           N.ptr(plan.perm) if num_nodes else None, G, N.ptr(tabs[0]), N.ptr(tabs[1]), N.ptr(lse), N.ptr(tabs[2]), N.ptr(d_x), N.ptr(d_qt),
           N.ptr(ws), ws_bytes)
    return d_x, d_qt


def attention_readout(module: nn.Module, inputs: ElementsToSummaryRepresentationInput, query_layer: nn.Module, key_weight: torch.Tensor,
                      heads: int, scale: float, value_weight: Optional[torch.Tensor], output_weight: torch.Tensor) -> torch.Tensor:
    """The attention reducers' forward (varsizedsummary.py:100-113 and :145-178) with the per-node algebra moved to G rows:
        z_{n,h} = q_{b,h} . (W_{k,h} x_n) * scale = x_n . qt[b, h],   qt[b, h] = scale W_{k,h}^T q_{b,h}
        sum_n p_{n,h} W_{v,h} x_n = W_{v,h} o[b, h],   o[b, h] = sum_n p_{n,h} x_n   (the kernel)
    then the output layer on [G, heads * D] (or [G, hidden] with the value layer)."""
    from . import autograd as _ag
    from . import composed as C

    x = inputs.element_embeddings
    if x.dim() != 2:
        raise ValueError(f"element_embeddings must be [num_elements, D], got {tuple(x.shape)}")
    D = x.shape[1]
    hidden = key_weight.shape[0]
    grad = _ag.needs_grad(module, x)
    bf16 = x.dtype == torch.bfloat16
    if grad and bf16:
        raise NotImplementedError("attention readout with gradients: fp32 states only (call it under torch.no_grad() for bf16)")
    if not N.lib().ptgnn_b200_attention_readout_supported(int(bf16), D, heads):
        raise NotImplementedError(f"the attention readout kernel takes D in {{32, 64, 128, 256}} and heads in {{1, 2, 4, 8}}, got D={D}, heads={heads}")
    n2g = inputs.element_to_sample_map
    plan = graph_plan(n2g, _num_samples(inputs))
    G = plan.num_nodes
    # 1. the per-graph queries [G, hidden]
    native = readout_of(query_layer)
    if native is None:
        q = query_layer(inputs)
    elif grad:
        q = _ag.graph_readout_with_grad(native[0], native[1], x, n2g, plan)
    else:
        q = reduce_states(native[0], native[1], x, n2g, plan)[0]
    if q.dim() != 2 or q.shape[1] != hidden:
        raise ValueError(f"the query summarizer returned shape {tuple(q.shape)}: its width must be hidden_size={hidden}")
    if q.shape[0] != G:
        raise ValueError(f"the query summarizer returned {q.shape[0]} rows for {G} samples")
    q = q.to(torch.float32)
    linear = _ag._LinearFn.apply if grad else C.linear
    dh = hidden // heads
    # 2. qt [G, heads, D]: one G * heads-row product on the key weight, with the row of (b, h) holding q_{b,h} * scale in head h's
    #    columns and zeros elsewhere (exact zeros: the products of the other heads add nothing)
    if heads == 1:
        q_rows = q * scale
    else:
        eye = torch.eye(heads, dtype=torch.float32, device=q.device)
        q_rows = (eye[None, :, :, None] * (q * scale).view(G, 1, heads, dh)).reshape(G * heads, hidden)
    qt = linear(q_rows, key_weight.t(), None).view(G, heads, D)
    # 3. the kernel
    if grad:
        o = _ag.attention_readout_with_grad(plan, heads, x, qt)
    else:
        o = native_attention_readout(x, plan, qt, heads)[0]
    plan.poll()
    # 4. value layer (head h's block of W_v on o[b, h]: the diagonal blocks of one G * heads-row product) and output layer
    if value_weight is not None:
        y = linear(o.reshape(G * heads, D), value_weight, None).view(G, heads, heads, dh)
        o = torch.diagonal(y, dim1=1, dim2=2).transpose(1, 2)                 # [G, heads, dh]
    out = linear(o.reshape(G, -1), output_weight, None)
    return out.to(x.dtype)


class SelfAttentionVarSizedElementReduce(AbstractVarSizedElementReduce):
    def __init__(
        self,
        input_representation_size: int,
        hidden_size: int,
        output_representation_size: int,
        query_representation_summarizer: AbstractVarSizedElementReduce,
    ):
        super().__init__()
        self.__query_layer = query_representation_summarizer
        self.__key_layer = nn.Linear(input_representation_size, hidden_size, bias=False)
        self.__output_layer = nn.Linear(input_representation_size, output_representation_size, bias=False)

    def forward(self, inputs: ElementsToSummaryRepresentationInput) -> torch.Tensor:
        return attention_readout(self, inputs, self.__query_layer, self.__key_layer.weight, 1, 1.0, None, self.__output_layer.weight)


class MultiheadSelfAttentionVarSizedElementReduce(AbstractVarSizedElementReduce):
    def __init__(
        self,
        input_representation_size: int,
        hidden_size: int,
        output_representation_size: int,
        num_heads: int,
        query_representation_summarizer: AbstractVarSizedElementReduce,
        use_value_layer: bool = False,
    ):
        super().__init__()
        self.__query_layer = query_representation_summarizer
        self.__key_layer = nn.Linear(input_representation_size, hidden_size, bias=False)
        assert hidden_size % num_heads == 0, "Hidden size must be divisible by the number of heads."
        self.__use_value_layer = use_value_layer
        if use_value_layer:
            self.__value_layer = nn.Linear(input_representation_size, hidden_size, bias=False)
            self.__output_layer = nn.Linear(hidden_size, output_representation_size, bias=False)
        else:
            self.__output_layer = nn.Linear(input_representation_size * num_heads, output_representation_size, bias=False)
        self.__num_heads = num_heads

    def forward(self, inputs: ElementsToSummaryRepresentationInput) -> torch.Tensor:
        heads = self.__num_heads
        value = self.__value_layer.weight if self.__use_value_layer else None
        scale = 1.0 / math.sqrt(self.__key_layer.weight.shape[0] // heads)
        return attention_readout(self, inputs, self.__query_layer, self.__key_layer.weight, heads, scale, value, self.__output_layer.weight)
