"""Global graph exchange layers with the reference's ``nn.Module`` API, computed by the CUDA library.

Counterparts of `ptgnn/neuralmodels/gnn/messagepassing/globalgraphexchange.py:13-72` of the reference:

* ``AbstractGlobalGraphExchange`` -- reduce every graph's node states to one summary g[b], dropout on it, update every node;
* ``GruGlobalStateUpdate``        -- the update ``h'_n = GRUCell(g[graph(n)], h_n)``.

Constructors, properties and (name-mangled) ``state_dict`` keys are the reference's.  The forward:

1. the summary ``g [G, S]``: the native readout kernel (``ptgnn_b200_graph_readout``) for this package's and the reference's
   ``WeightedSumVarSizedElementReduce`` / ``SimpleVarSizedElementReduce`` instances (max / min: the native ``scatter``); any other
   reducer module is called as is;
2. training-mode dropout on ``g`` -- a G-row torch op, where the reference applies it;
3. ``GRUCell(g[graph(n)], h_n)``: the input side ``g W_ih^T + b_ih`` has G distinct rows, so it is computed once as a [G, 3H] table
   and the weights-stationary GRU kernel runs over the node rows with state chunks only (``ptgnn_b200_global_gru_update``).  State
   sizes that kernel does not take (H not a multiple of 64) run the native ``grucell`` on the gathered per-node summaries.

The number of graphs comes from the container (``GraphNeuralNetwork.forward`` hands its ``num_graphs`` over), or is read from the device
once per ``node_to_graph_idx`` tensor.  A count larger than ``max + 1`` only adds empty graphs.
"""
from abc import abstractmethod
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _native as N
from .edgeplan import EdgePlan, _version, current_num_graphs, current_state_chain
from .messagepassing import AbstractMessagePassingLayer, _check_shape, _check_states
from .reduceops import AbstractVarSizedElementReduce, ElementsToSummaryRepresentationInput, graph_plan, readout_of, reduce_states

_COUNT_CACHE: "OrderedDict[tuple, Tuple[torch.Tensor, int]]" = OrderedDict()
_COUNT_CACHE_SIZE = 4


def num_graphs_of(node_to_graph_idx: torch.Tensor) -> int:
    """The container's graph count if it handed one over (no device read), else ``max + 1``, read from the device at most once per
    tensor (identity + version, like the plan cache; entries keep their tensor alive so that the key cannot alias)."""
    handed = current_num_graphs()
    if handed is not None:
        return int(handed)
    key = (node_to_graph_idx.data_ptr(), node_to_graph_idx.shape[0], _version(node_to_graph_idx), node_to_graph_idx.device)
    hit = _COUNT_CACHE.get(key)
    if hit is not None:
        _COUNT_CACHE.move_to_end(key)
        return hit[1]
    count = int(node_to_graph_idx.max().item()) + 1 if node_to_graph_idx.numel() else 0
    _COUNT_CACHE[key] = (node_to_graph_idx, count)
    while len(_COUNT_CACHE) > _COUNT_CACHE_SIZE:
        _COUNT_CACHE.popitem(last=False)
    return count


class AbstractGlobalGraphExchange(AbstractMessagePassingLayer):
    def __init__(self, global_graph_representation_module: AbstractVarSizedElementReduce, dropout_rate: float = 0.0):
        super().__init__()
        self.__global_graph_representation_module = global_graph_representation_module
        self.__dropout = nn.Dropout(p=dropout_rate)

    @abstractmethod
    def _update_node_states(self, node_states: torch.Tensor, global_info_per_node: torch.Tensor) -> torch.Tensor:
        raise NotImplementedError()

    def _update_from_summaries(self, node_states: torch.Tensor, summaries: torch.Tensor, plan: EdgePlan) -> torch.Tensor:
        """The update from the per-graph summaries [G, S]; by default the reference's per-node form (the plan's ``tgt32`` is the
        node -> graph map, with out-of-range ids clamped, so the gather stays in bounds)."""
        return self._update_node_states(node_states, summaries.index_select(0, plan.tgt32.long()))

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
        if gather_states is not None:
            raise NotImplementedError("global graph exchange on node-range shards: a graph can straddle ranks (shard by graph instead)")
        from . import autograd as _ag

        _check_states(node_states, self.input_state_dimension, type(self).__name__)
        grad = _ag.needs_grad(self, node_states)
        if grad and node_states.dtype != torch.float32:
            raise NotImplementedError("global graph exchange with gradients: fp32 states only")
        plan = graph_plan(node_to_graph_idx, num_graphs_of(node_to_graph_idx))
        reducer = self.__global_graph_representation_module
        native = readout_of(reducer)
        if native is None:
            summaries = reducer(ElementsToSummaryRepresentationInput(node_states, node_to_graph_idx, plan.num_nodes))
        elif grad:
            summaries = _ag.graph_readout_with_grad(native[0], native[1], node_states, node_to_graph_idx, plan)
        else:
            summaries = reduce_states(native[0], native[1], node_states, node_to_graph_idx, plan)[0]
        summaries = self.__dropout(summaries.to(torch.float32))
        return self._update_from_summaries(node_states, summaries, plan)


class GruGlobalStateUpdate(AbstractGlobalGraphExchange):
    def __init__(
        self,
        global_graph_representation_module: AbstractVarSizedElementReduce,
        input_state_size: int,
        summarized_state_size: int,
        dropout_rate: float = 0.0,
    ):
        super().__init__(global_graph_representation_module, dropout_rate)
        self.__input_dim = input_state_size
        self.__summarized_state_size = summarized_state_size
        self.__gru_cell = nn.GRUCell(input_size=summarized_state_size, hidden_size=input_state_size)

    def _update_node_states(self, node_states: torch.Tensor, global_info_per_node: torch.Tensor) -> torch.Tensor:
        """The reference's per-node form (globalgraphexchange.py:59-62), on the native GRUCell kernel (fp32)."""
        from . import composed as C

        return C.grucell(N.require_cuda(global_info_per_node, "global_info_per_node", torch.float32),
                         N.require_cuda(node_states, "node_states", torch.float32), self.__gru_cell)

    def _update_from_summaries(self, node_states: torch.Tensor, summaries: torch.Tensor, plan: EdgePlan) -> torch.Tensor:
        from . import autograd as _ag

        gru = self.__gru_cell
        H, S = self.__input_dim, self.__summarized_state_size
        _check_shape(summaries, (plan.num_nodes, S), "graph summaries")
        _check_shape(gru.weight_ih, (3 * H, S), "GRUCell.weight_ih"); _check_shape(gru.weight_hh, (3 * H, H), "GRUCell.weight_hh")
        _check_shape(gru.bias_ih, (3 * H,), "GRUCell.bias_ih"); _check_shape(gru.bias_hh, (3 * H,), "GRUCell.bias_hh")
        if _ag.needs_grad(self, node_states) or summaries.requires_grad:
            return _ag.global_gru_with_grad(self, node_states, summaries, plan, gru.weight_ih, gru.weight_hh, gru.bias_ih, gru.bias_hh)
        return self.table_update(node_states, summaries, plan)

    def table_update(self, node_states: torch.Tensor, summaries: torch.Tensor, plan: EdgePlan) -> torch.Tensor:
        """``GRUCell(summaries[graph(n)], h_n)`` through the input-side table and the state-only GRU kernel (no autograd).  Inside a
        container's layer loop it takes the packed form of its input from the previous layer and hands on the packed form of its
        output (edgeplan.state_chain)."""
        gru = self.__gru_cell
        bf16 = node_states.dtype == torch.bfloat16
        h = N.require_cuda(node_states, "node_states", torch.bfloat16 if bf16 else torch.float32)
        num_nodes, H = h.shape
        S = self.__summarized_state_size
        g = N.require_cuda(summaries.detach(), "summaries", torch.float32)
        p = [N.require_cuda(t.detach(), n, torch.float32) for t, n in ((gru.weight_ih, "weight_ih"), (gru.weight_hh, "weight_hh"),
                                                                         (gru.bias_ih, "bias_ih"), (gru.bias_hh, "bias_hh"))]
        lib = N.lib()
        chain = None if bf16 else current_state_chain()
        if not lib.ptgnn_b200_global_gru_supported(int(bf16), H) or S % 4 != 0:
            if bf16:
                raise NotImplementedError(f"GruGlobalStateUpdate with bf16 states needs H a multiple of 64 and S a multiple of 4 (H={H}, S={S})")
            out = self._update_node_states(h, g.index_select(0, plan.tgt32.long()))      # the per-node form (tgt32: ids clamped in range)
            if chain is not None:
                chain.store(out, None)
            return out
        kind = "global_gru_bf16" if bf16 else "global_gru_f32"
        cache, valid = self._weight_cache(kind, lib.ptgnn_b200_global_gru_weight_cache_bytes(int(bf16), H), [p[1], p[3]], h.device)
        ws_bytes = lib.ptgnn_b200_global_gru_workspace_bytes(int(bf16), num_nodes, plan.num_nodes, H, S)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=h.device)
        out = torch.empty_like(h)
        packed_in = chain.lookup(node_states) if (chain is not None and h is node_states) else None
        packed_out = None
        if chain is not None and chain.want_output:
            packed_out = torch.empty(max(lib.ptgnn_b200_packed_state_bytes(num_nodes, H), 1), dtype=torch.uint8, device=h.device)
        with torch.cuda.device(h.device):
            rc = lib.ptgnn_b200_global_gru_update(
                int(bf16), N.ptr(h), N.ptr(packed_in), num_nodes, H, N.ptr(plan.tgt32), plan.num_nodes, N.ptr(g), S, N.ptr(p[0]),
                N.ptr(p[1]), N.ptr(p[2]), N.ptr(p[3]), N.ptr(out), N.ptr(packed_out), plan.status.data_ptr() + 4, N.ptr(ws), ws_bytes,
                N.ptr(cache), 0 if cache is None else cache.numel(), int(valid), N.current_stream(h.device),
            )
        N.check(rc, "ptgnn_b200_global_gru_update")
        self._weight_cache_filled(kind, h.device)
        if chain is not None:
            chain.store(out, packed_out)
        return out

    @property
    def input_state_dimension(self) -> int:
        return self.__input_dim

    @property
    def output_state_dimension(self) -> int:
        return self.__input_dim
