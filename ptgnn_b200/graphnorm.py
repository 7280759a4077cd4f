"""``GraphNorm`` with the reference's ``nn.Module`` API, on the native per-graph normalisation kernels.

Counterpart of `ptgnn/neuralmodels/gnn/messagepassing/graphnorm.py:9-54` of the reference (arXiv:2009.03294): per graph ``g`` and
column ``d``, ``mu = mean_{i in g} x_i``, ``s_i = x_i - alpha mu``, ``sigma^2 = mean_{i in g} s_i^2 + eps`` and
``y_i = gamma s_i / sqrt(sigma^2) + bias``.  The reference runs two ``scatter_mean`` calls and seven full passes over ``[N, D]``; here
one statistics pass and one output pass (``ptgnn_b200_graph_norm_forward``, DESIGN.md §3.9) read the states twice in all.

* bf16 states: read and written in bf16, statistics in fp32.
* Gradients (fp32): ``_GraphNormFn`` around the kernels (saves ``x`` and the ``[G, D]`` mean and rstd; the backward recomputes the
  normalised states).
* The graph count is the container's ``num_graphs`` when it handed one over (then a call makes no host synchronisation), else
  ``max + 1`` read once per ``node_to_graph_idx`` tensor.  A larger count only adds empty graphs.

Not supported (``NotImplementedError``): gradients with bf16 states, node-range shards (``gather_states``), and state dimensions other
than a multiple of 32 in [32, 256].
"""
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _native as N
from .edgeplan import EdgePlan
from .messagepassing import AbstractMessagePassingLayer, _check_states

_DIMS = "a state dimension that is a multiple of 32 in [32, 256]"


def _aligned(t: torch.Tensor, what: str, dtype: torch.dtype) -> torch.Tensor:
    """A contiguous CUDA tensor of ``dtype`` whose data starts on a 16-byte boundary (the kernels load four columns at once)."""
    t = N.require_cuda(t, what, dtype)
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _params(gamma: torch.Tensor, alpha: torch.Tensor, bias: torch.Tensor, D: int, device):
    out = []
    for p, n in ((gamma, "gamma"), (alpha, "alpha"), (bias, "bias")):
        if p.numel() != D:
            raise ValueError(f"{n} must have {D} elements, got {tuple(p.shape)}")
        out.append(_aligned(p.detach().reshape(D).to(device), n, torch.float32))
    return out


def _check(x: torch.Tensor, plan: EdgePlan) -> Tuple[int, int]:
    if x.dim() != 2:
        raise ValueError(f"node_states must be [num_nodes, D], got {tuple(x.shape)}")
    num_nodes, D = x.shape
    if plan.num_edges != num_nodes:
        raise ValueError("node_to_graph_idx and node_states disagree on the number of nodes")
    if not N.lib().ptgnn_b200_graph_norm_supported(D):
        raise NotImplementedError(f"the GraphNorm kernels take {_DIMS}, got D={D}")
    return num_nodes, D


def native_graph_norm(x: torch.Tensor, plan: EdgePlan, gamma: torch.Tensor, alpha: torch.Tensor, bias: torch.Tensor, eps: float,
                      out: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``ptgnn_b200_graph_norm_forward``: (y [N, D] in x's dtype, mean [G, D] fp32, rstd [G, D] fp32) for x [N, D] fp32 or bf16 and the
    plan of the node -> graph map (``reduceops.graph_plan``).  ``out``: an aligned contiguous [N, D] tensor of x's dtype for y."""
    dtype = torch.bfloat16 if x.dtype == torch.bfloat16 else torch.float32
    x = _aligned(x, "node_states", dtype)
    num_nodes, D = _check(x, plan)
    g, a, b = _params(gamma, alpha, bias, D, x.device)
    G = plan.num_nodes
    lib = N.lib()
    ws_bytes = lib.ptgnn_b200_graph_norm_workspace_bytes(num_nodes, G, D)
    y = torch.empty_like(x) if out is None else out
    if y.dtype != x.dtype or tuple(y.shape) != tuple(x.shape) or not y.is_contiguous() or y.data_ptr() % 16 != 0:
        raise ValueError(f"out must be an aligned contiguous {tuple(x.shape)} {x.dtype} tensor")
    mean = torch.empty(G, D, dtype=torch.float32, device=x.device)
    rstd = torch.empty(G, D, dtype=torch.float32, device=x.device)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        rc = lib.ptgnn_b200_graph_norm_forward(int(dtype == torch.bfloat16), N.ptr(x), num_nodes, D, N.ptr(plan.row_ptr), N.ptr(plan.perm),
                                               N.ptr(plan.tgt32), G, N.ptr(g), N.ptr(a), N.ptr(b), float(eps), N.ptr(y), N.ptr(mean),
                                               N.ptr(rstd), N.ptr(ws), ws_bytes, N.current_stream(x.device))
    N.check(rc, "ptgnn_b200_graph_norm_forward")
    return y, mean, rstd


def native_graph_norm_backward(x: torch.Tensor, plan: EdgePlan, gamma: torch.Tensor, alpha: torch.Tensor, eps: float, mean: torch.Tensor,
                               rstd: torch.Tensor, d_y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """``ptgnn_b200_graph_norm_backward_f32``: (d x [N, D], d gamma [D], d alpha [D], d bias [D]) from d y [N, D].  fp32."""
    x = _aligned(x, "node_states", torch.float32)
    num_nodes, D = _check(x, plan)
    d_y = _aligned(d_y, "d_out", torch.float32)
    G = plan.num_nodes
    mean, rstd = _aligned(mean, "mean", torch.float32), _aligned(rstd, "rstd", torch.float32)
    for t, n, shape in ((d_y, "d_out", (num_nodes, D)), (mean, "mean", (G, D)), (rstd, "rstd", (G, D))):
        if tuple(t.shape) != shape:
            raise ValueError(f"{n} must have shape {shape}, got {tuple(t.shape)}")
    g, a, _ = _params(gamma, alpha, alpha, D, x.device)
    lib = N.lib()
    ws_bytes = lib.ptgnn_b200_graph_norm_workspace_bytes(num_nodes, G, D)
    d_x = torch.empty_like(x)
    d_params = torch.empty(3, D, dtype=torch.float32, device=x.device)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        rc = lib.ptgnn_b200_graph_norm_backward_f32(N.ptr(x), N.ptr(d_y), num_nodes, D, N.ptr(plan.row_ptr), N.ptr(plan.perm), N.ptr(plan.tgt32),
                                                    G, N.ptr(g), N.ptr(a), float(eps), N.ptr(mean), N.ptr(rstd), N.ptr(d_x), N.ptr(d_params[0]),
                                                    N.ptr(d_params[1]), N.ptr(d_params[2]), N.ptr(ws), ws_bytes, N.current_stream(x.device))
    N.check(rc, "ptgnn_b200_graph_norm_backward_f32")
    return d_x, d_params[0], d_params[1], d_params[2]


class GraphNorm(AbstractMessagePassingLayer):
    """
    A GraphNorm layer implemented as in

    GraphNorm: A Principled Approach to Accelerating Graph Neural Network Training (arXiv:2009.03294v1)
      Tianle Cai, Shengjie Luo, Keyulu Xu, Di He, Tie-yan Liu, Liwei Wang

    """

    def __init__(self, input_state_dimension: int, eps: float = 1e-10):
        super().__init__()
        self.__input_state_dim = input_state_dimension
        self.__eps = eps

        self.gamma = nn.Parameter(torch.ones(1, input_state_dimension))
        self.alpha = nn.Parameter(torch.ones(1, input_state_dimension))
        self.bias = nn.Parameter(torch.zeros(1, input_state_dimension))

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
        from .globalexchange import num_graphs_of
        from .reduceops import graph_plan

        name = type(self).__name__
        if gather_states is not None:
            raise NotImplementedError(f"{name} on node-range shards: a graph can straddle ranks (shard by graph instead)")
        _check_states(node_states, self.__input_state_dim, name)
        if not N.lib().ptgnn_b200_graph_norm_supported(self.__input_state_dim):
            raise NotImplementedError(f"{name}: the GraphNorm kernels take {_DIMS}, got D={self.__input_state_dim}")
        bf16 = node_states.dtype == torch.bfloat16
        grad = _ag.needs_grad(self, node_states)
        if grad and bf16:
            raise NotImplementedError(f"{name} with gradients: fp32 states only (call it under torch.no_grad() for bf16)")
        plan = graph_plan(node_to_graph_idx, num_graphs_of(node_to_graph_idx))
        if grad:
            out = _ag.graph_norm_with_grad(plan, self.__eps, node_states.to(torch.float32), self.gamma, self.alpha, self.bias)
        else:
            out = native_graph_norm(node_states if bf16 else node_states.to(torch.float32), plan, self.gamma, self.alpha, self.bias,
                                    self.__eps)[0]
        plan.poll()
        return out if bf16 else out.to(node_states.dtype)

    @property
    def input_state_dimension(self) -> int:
        return self.__input_state_dim

    @property
    def output_state_dimension(self) -> int:
        return self.__input_state_dim
