"""``GraphNeuralNetwork`` container with the reference's API, owning the layer loop.

Counterpart of `/root/reference/ptgnn/neuralmodels/gnn/graphneuralnetwork.py:28-209` (class ``GraphNeuralNetwork``)
and the carrier types of `ptgnn/neuralmodels/gnn/structs.py:52-76` of the reference.  Differences that matter on the GPU:
the container builds the edge plan once per minibatch and shares it with all of its layers (the reference rebuilds the
equivalent grouping inside every ``scatter`` call), and it never mutates the caller's ``adjacency_lists`` list in place.
Metric bookkeeping (``num_graphs/num_nodes/num_edges``, post-expansion edge count) is bit-identical.
"""
from typing import Any, Dict, List, NamedTuple, Optional, Tuple

import torch
from torch import nn

from .edgeplan import EdgePlan, clear_plan_cache, plan_for, shared_num_graphs, shared_plan, state_chain
from .messagepassing import AbstractMessagePassingLayer


class GnnOutput(NamedTuple):
    input_node_representations: torch.Tensor
    output_node_representations: torch.Tensor
    node_to_graph_idx: torch.Tensor
    node_idx_references: Dict[str, torch.Tensor]
    node_graph_idx_reference: Dict[str, torch.Tensor]
    num_graphs: int

    @property
    def reference_nodes_idx(self) -> Dict[str, torch.Tensor]:
        return self.node_idx_references

    @property
    def reference_nodes_graph_idx(self) -> Dict[str, torch.Tensor]:
        return self.node_graph_idx_reference


def register_with_reference_metrics() -> bool:
    """Makes ``GraphNeuralNetwork`` a (virtual) subclass of the reference's ``ModuleWithMetrics`` if that class has been
    imported: reference parents collect and reset child metrics with ``isinstance(child, ModuleWithMetrics)``
    (`/root/reference/ptgnn/baseneuralmodel/modulewithmetrics.py:44-46,56-57`).  ``ModuleWithMetrics`` is an ``ABC``, so
    registration is all it takes; idempotent, never imports the reference itself.  Called when a container is constructed (by
    then any reference parent has imported the class) and by ``ptgnn_b200.overlay.install()``."""
    import sys

    mod = sys.modules.get("ptgnn.baseneuralmodel.modulewithmetrics")
    base = getattr(mod, "ModuleWithMetrics", None)
    if base is None or not hasattr(base, "register"):
        return False
    if not issubclass(GraphNeuralNetwork, base):
        base.register(GraphNeuralNetwork)
    return True


class GraphNeuralNetwork(nn.Module):
    """Generic message-passing GNN over discrete edge types.  Implements the reference's ``ModuleWithMetrics`` protocol
    (``report_metrics`` / ``reset_metrics`` / ``_module_metrics`` / ``_reset_module_metrics``) and registers itself as a virtual
    subclass of the reference's class when that is loaded, so that it also works as a CHILD of reference modules."""

    def __init__(
        self,
        message_passing_layers: List[AbstractMessagePassingLayer],
        node_embedder: nn.Module,
        introduce_backwards_edges: bool,
        add_self_edges: bool,
        edge_dropout_rate: float = 0.0,
        edge_feature_embedder: Optional[nn.Module] = None,
    ):
        super().__init__()
        assert 0 <= edge_dropout_rate < 1
        self.__message_passing_layers = nn.ModuleList(message_passing_layers)
        self.__node_embedder = node_embedder
        self.__introduce_backwards_edges = introduce_backwards_edges
        self.__add_self_edges = add_self_edges
        self.__edge_dropout_rate = edge_dropout_rate
        self.__edge_feature_embedder = edge_feature_embedder
        self._reset_module_metrics()
        register_with_reference_metrics()

    # ---- metrics protocol (modulewithmetrics.py:8-77) ---------------------------------------------
    def _reset_module_metrics(self) -> None:
        self.__num_graphs, self.__num_edges, self.__num_nodes = 0, 0, 0

    def _module_metrics(self) -> Dict[str, Any]:
        return {"num_graphs": int(self.__num_graphs), "num_nodes": int(self.__num_nodes), "num_edges": int(self.__num_edges)}

    def report_metrics(self) -> Dict[str, Any]:
        metrics = self._module_metrics()
        for child in self.modules():
            if child is not self and hasattr(child, "_module_metrics"):
                metrics.update(child._module_metrics())
        return metrics

    def reset_metrics(self) -> None:
        for child in self.modules():
            if hasattr(child, "_reset_module_metrics"):
                child._reset_module_metrics()

    def train(self, mode: bool = True):
        self.reset_metrics()
        return super().train(mode=mode)

    def eval(self):
        self.reset_metrics()
        return super().eval()

    # ---- properties ---------------------------------------------------------------------------------
    @property
    def input_node_state_dim(self) -> int:
        return self.__message_passing_layers[0].input_state_dimension

    @property
    def output_node_state_dim(self) -> int:
        return self.__message_passing_layers[-1].output_state_dimension

    @property
    def message_passing_layers(self) -> List[AbstractMessagePassingLayer]:
        return self.__message_passing_layers

    # ---- layer loop -----------------------------------------------------------------------------------
    def gnn(
        self,
        node_representations: torch.Tensor,
        adjacency_lists: List[Tuple[torch.Tensor, torch.Tensor]],
        edge_feature_embeddings: List[torch.Tensor],
        node_to_graph_idx: torch.Tensor,
        reference_node_ids: Dict[str, torch.Tensor],
        reference_node_graph_idx: Dict[str, torch.Tensor],
        return_all_states: bool = False,
        plan: Optional[EdgePlan] = None,
        num_graphs: Optional[int] = None,
    ) -> torch.Tensor:
        """``num_graphs`` (optional): the number of graphs in the minibatch, handed to the global-exchange layers so that they do not
        read ``node_to_graph_idx.max() + 1`` from the device."""
        if self.__edge_dropout_rate > 0 and self.training:
            # graphneuralnetwork.py:105-119: Bernoulli keep-mask per edge (device-side index bookkeeping; a new plan is built
            # for the surviving edges, so this also invalidates any plan handed in)
            kept_adj, kept_feats = [], []
            feats_in = edge_feature_embeddings if edge_feature_embeddings is not None else [None] * len(adjacency_lists)
            for (src, tgt), feats in zip(adjacency_lists, feats_in):
                mask = torch.rand_like(src, dtype=torch.float32) > self.__edge_dropout_rate
                kept_adj.append((src.masked_select(mask), tgt.masked_select(mask)))
                kept_feats.append(None if feats is None else feats[mask])
            adjacency_lists = kept_adj
            edge_feature_embeddings = kept_feats if edge_feature_embeddings is not None else None
            plan = None
        if node_representations.is_cuda:
            plan = plan_for(adjacency_lists, node_representations.shape[0], plan)
        all_states = [node_representations]
        layers = list(self.__message_passing_layers)
        # per-thread hand-offs: the layers of this call (and only they) reuse the plan and the graph count, and pass their packed
        # states on
        with shared_plan(plan), shared_num_graphs(num_graphs), state_chain() as chain:
            for i, layer in enumerate(layers):
                chain.want_output = i + 1 < len(layers)
                node_representations = layer(
                    node_states=node_representations,
                    adjacency_lists=adjacency_lists,
                    node_to_graph_idx=node_to_graph_idx,
                    reference_node_ids=reference_node_ids,
                    reference_node_graph_idx=reference_node_graph_idx,
                    edge_features=edge_feature_embeddings,
                )
                all_states.append(node_representations)
        if return_all_states:
            node_representations = torch.cat(all_states, dim=-1)
        return node_representations

    def capture(self, node_states: torch.Tensor, adjacency_lists: List[Tuple[torch.Tensor, torch.Tensor]],
                node_to_graph_idx: Optional[torch.Tensor] = None, return_all_states: bool = False,
                num_graphs: Optional[int] = None) -> "GraphedLayerLoop":
        """CUDA-graph the layer loop (edge plan + all layers) for FIXED shapes: the returned object replays it with one launch.
        ``node_states`` / ``adjacency_lists`` (already expanded, see ``expand_adjacency``) are the static input buffers -- refill
        them in place (e.g. with ``copy_`` from pinned host memory) and call ``replay()``.  The per-type edge COUNTS are frozen at
        capture; the edge contents, the node states and -- because the plan is rebuilt inside the graph -- the graph structure
        are whatever the buffers hold at replay time.  Parameters must not change between capture and replay (eval mode).
        With global-exchange, self-attention or GraphNorm layers the number of graphs is frozen at capture too: ``num_graphs``, or -- when it is not given --
        ``node_to_graph_idx.max() + 1``, read once before the warm-up; ``node_to_graph_idx`` is then a static input buffer as well."""
        from .globalexchange import AbstractGlobalGraphExchange
        from .graphnorm import GraphNorm
        from .selfattention import MultiHeadSelfAttentionMessagePassing

        per_graph = (AbstractGlobalGraphExchange, MultiHeadSelfAttentionMessagePassing, GraphNorm)
        if num_graphs is None and any(isinstance(layer, per_graph) for layer in self.__message_passing_layers):
            if node_to_graph_idx is None:
                raise ValueError("capture(): global-exchange, self-attention and GraphNorm layers need node_to_graph_idx")
            num_graphs = int(node_to_graph_idx.max().item()) + 1 if node_to_graph_idx.numel() else 0
        return GraphedLayerLoop(self, node_states, adjacency_lists, node_to_graph_idx, return_all_states, num_graphs)

    def expand_adjacency(self, adjacency_lists, num_nodes: int, device) -> List[Tuple[torch.Tensor, torch.Tensor]]:
        """Backward + self edge lists (graphneuralnetwork.py:172-186) as a NEW list."""
        expanded = list(adjacency_lists)
        if self.__introduce_backwards_edges:
            expanded += [(tgt, src) for src, tgt in adjacency_lists]
        if self.__add_self_edges:
            ident = torch.arange(num_nodes, dtype=torch.int64, device=device)
            expanded.append((ident, ident))
        return expanded

    def forward(
        self,
        *,
        node_data,
        adjacency_lists: List[Tuple[torch.Tensor, torch.Tensor]],
        edge_feature_data: List,
        node_to_graph_idx: torch.Tensor,
        reference_node_ids: Dict[str, torch.Tensor],
        reference_node_graph_idx: Dict[str, torch.Tensor],
        num_graphs,
        **kwargs,
    ) -> GnnOutput:
        initial = self.__node_embedder(**node_data)
        device = node_to_graph_idx.device
        num_nodes = node_to_graph_idx.shape[0]
        expanded = self.expand_adjacency(adjacency_lists, num_nodes, device)
        if self.__edge_feature_embedder is None:
            edge_features = [torch.empty(src.shape[0], 0, device=device) for src, _ in expanded]
        else:   # graphneuralnetwork.py:167-186: embed per raw type, reuse for the backward types, zeros for the self edges
            edge_features = [self.__edge_feature_embedder(**edge_data) for edge_data in edge_feature_data]
            if self.__introduce_backwards_edges:
                edge_features = edge_features + list(edge_features)
            if self.__add_self_edges:
                edge_features.append(torch.zeros(num_nodes, edge_features[-1].shape[-1], device=device))
        if "num_graphs" not in kwargs and isinstance(num_graphs, int):
            kwargs["num_graphs"] = num_graphs
        output = self.gnn(initial, expanded, edge_features, node_to_graph_idx, reference_node_ids,
                          reference_node_graph_idx, **kwargs)
        self.__num_edges += sum(src.shape[0] for src, _ in expanded)
        self.__num_graphs += num_graphs
        self.__num_nodes += num_nodes
        return GnnOutput(
            input_node_representations=initial,
            output_node_representations=output,
            node_to_graph_idx=node_to_graph_idx,
            node_idx_references=reference_node_ids,
            node_graph_idx_reference=reference_node_graph_idx,
            num_graphs=num_graphs,
        )


class GraphedLayerLoop:
    """``GraphNeuralNetwork.gnn`` captured into one CUDA graph (see ``GraphNeuralNetwork.capture``).  Replaces ~50 kernel
    launches and ~10 ctypes calls per minibatch by one ``cudaGraphLaunch``: what the reference would get from
    ``torch.cuda.graphs`` around its own loop, here including the plan build."""

    def __init__(self, gnn: GraphNeuralNetwork, node_states, adjacency_lists, node_to_graph_idx, return_all_states: bool,
                 num_graphs: Optional[int] = None):
        if gnn.training:
            raise RuntimeError("capture() needs eval mode (the derived-weight caches are only trusted there)")
        self.node_states, self.adjacency_lists = node_states, list(adjacency_lists)
        self._gnn = gnn
        dev = node_states.device
        run = lambda: gnn.gnn(node_states, self.adjacency_lists, None, node_to_graph_idx, {}, {}, return_all_states=return_all_states,  # noqa: E731
                              num_graphs=num_graphs)
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():     # warm-up outside the graph: fills weight caches and allocator pools
            for _ in range(2):
                clear_plan_cache()
                run()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        clear_plan_cache()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.output = run()
        self._plan = plan_for(self.adjacency_lists, node_states.shape[0])    # built during capture; keeps its buffers and status words
        self._graph_plan = None
        if num_graphs is not None and node_to_graph_idx is not None:         # the global-exchange layers' node -> graph plan, likewise
            self._graph_plan = plan_for([(node_to_graph_idx, node_to_graph_idx)], num_graphs)
        clear_plan_cache()

    def replay(self) -> torch.Tensor:
        self._plan.poll()          # errors the previous replay's kernels reported (bad indices, fp16-range overflow)
        if self._graph_plan is not None:
            self._graph_plan.poll()
        self.graph.replay()
        return self.output
