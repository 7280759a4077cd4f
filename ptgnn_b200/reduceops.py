"""Per-graph summaries of node states, with the reference's ``nn.Module`` API, on the native readout kernel.

Counterparts of `ptgnn/neuralmodels/reduceops/varsizedsummary.py:11-81` of the reference:

* ``ElementsToSummaryRepresentationInput`` -- the input record (embeddings, element -> sample map, number of samples);
* ``SimpleVarSizedElementReduce``          -- sum / mean on ``ptgnn_b200_graph_readout``; max / min on the native ``scatter``;
* ``WeightedSumVarSizedElementReduce``     -- ``sum_n sigmoid(x_n . w) x_n`` on ``ptgnn_b200_graph_readout``.

Constructor signatures and (name-mangled) ``state_dict`` keys are the reference's.  ``GruGlobalStateUpdate`` reads these modules
and the reference's own instances of the same two classes directly (``readout_of``), so the reference's factories need no change.
"""
from abc import abstractmethod
from typing import NamedTuple, Optional, Union

import torch
from torch import nn

from . import _native as N
from .edgeplan import EdgePlan, plan_for


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


def native_readout(node_states: torch.Tensor, plan: EdgePlan, mode: int, gate_weight: Optional[torch.Tensor] = None,
                   want_gates: bool = False):
    """``ptgnn_b200_graph_readout``: (g [G, H] fp32, s [N] fp32 or None).  fp32 or bf16 states; H a multiple of 32 in [32, 256]."""
    dtype = torch.bfloat16 if node_states.dtype == torch.bfloat16 else torch.float32
    x = N.require_cuda(node_states, "node_states", dtype)
    if x.dim() != 2:
        raise ValueError(f"node_states must be [num_nodes, H], got {tuple(x.shape)}")
    num_nodes, H = x.shape
    if plan.num_edges != num_nodes:
        raise ValueError("node_to_graph_idx and node_states disagree on the number of nodes")
    G = plan.num_nodes
    lib = N.lib()
    ws_bytes = lib.ptgnn_b200_graph_readout_workspace_bytes(num_nodes, G, H)
    if ws_bytes == 0:
        raise NotImplementedError(f"the graph readout kernel takes H a multiple of 32 in [32, 256], got H={H}")
    w = None
    if mode == N.READOUT_WEIGHTED_SUM:
        w = N.require_cuda(gate_weight, "weights_layer.weight", torch.float32)
        if tuple(w.shape) != (1, H):        # raw pointers cross the C ABI next
            raise ValueError(f"weights_layer.weight must have shape (1, {H}), got {tuple(w.shape)}")
    g = torch.empty(G, H, dtype=torch.float32, device=x.device)
    s = torch.empty(num_nodes, dtype=torch.float32, device=x.device) if want_gates and w is not None else None
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        rc = lib.ptgnn_b200_graph_readout(int(dtype == torch.bfloat16), N.ptr(x), num_nodes, H, N.ptr(plan.row_ptr),
                                          N.ptr(plan.perm) if num_nodes else None, G, N.ptr(w), mode, N.ptr(g), N.ptr(s), N.ptr(ws),
                                          ws_bytes, N.current_stream(x.device))
    N.check(rc, "ptgnn_b200_graph_readout")
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
