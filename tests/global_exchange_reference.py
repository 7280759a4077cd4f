"""CPU restatement of the reference's GruGlobalStateUpdate for the tests (like ``fused_reference.py``), on the oracle's ``scatter``
(torch_scatter semantics) and ``gru_cell``:

* ``graph_readout``             -> ``ptgnn/neuralmodels/reduceops/varsizedsummary.py:26-81`` (Simple / WeightedSum reducers)
* ``global_gru_update_forward`` -> ``ptgnn/neuralmodels/gnn/messagepassing/globalgraphexchange.py:29-62`` in eval mode

Pinned to the reference's own outputs by ``test_oracle_global_exchange.py`` (fixtures written by
``golden/generate_global_exchange_golden.py``).  Works in any dtype, float64 included, and under autograd.
"""
from typing import Optional

import torch
import torch.nn.functional as F

from oracle.ptgnn_oracle import gru_cell, scatter


def graph_readout(x: torch.Tensor, node_to_graph_idx: torch.Tensor, num_graphs: int, kind: str,
                  gate_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``kind`` "weighted" -- WeightedSumVarSizedElementReduce, sum_n sigmoid(x_n w^T) x_n; "sum" / "mean" / "max" / "min" --
    SimpleVarSizedElementReduce."""
    if kind == "weighted":
        weights = torch.sigmoid(F.linear(x, gate_weight).squeeze(-1))
        return scatter(x * weights.unsqueeze(-1), node_to_graph_idx, num_graphs, "sum")
    return scatter(x, node_to_graph_idx, num_graphs, kind)


def global_gru_update_forward(node_states: torch.Tensor, node_to_graph_idx: torch.Tensor, kind: str, gate_weight: Optional[torch.Tensor],
                              gru_w_ih: torch.Tensor, gru_w_hh: torch.Tensor, gru_b_ih: torch.Tensor, gru_b_hh: torch.Tensor,
                              num_graphs: Optional[int] = None) -> torch.Tensor:
    """The readout over ``max + 1`` graphs (or ``num_graphs``), then GRUCell(g[graph(n)], h_n)."""
    G = int(node_to_graph_idx.max()) + 1 if num_graphs is None else num_graphs
    g = graph_readout(node_states, node_to_graph_idx, G, kind, gate_weight)
    return gru_cell(g[node_to_graph_idx], node_states, gru_w_ih, gru_w_hh, gru_b_ih, gru_b_hh)
