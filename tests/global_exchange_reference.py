"""CPU restatement of the reference's GruGlobalStateUpdate for the tests (like ``fused_reference.py``), on the oracle's ``scatter``
(torch_scatter semantics) and ``gru_cell``:

* ``graph_readout``             -> ``ptgnn/neuralmodels/reduceops/varsizedsummary.py:26-81`` (Simple / WeightedSum reducers)
* ``global_gru_update_forward`` -> ``ptgnn/neuralmodels/gnn/messagepassing/globalgraphexchange.py:29-62`` in eval mode

Pinned to the reference's own outputs by ``test_oracle_global_exchange.py`` (fixtures written by
``golden/generate_global_exchange_golden.py``).  Works in any dtype, float64 included, and under autograd.

``readout_bound`` is the float64 readout of the native per-graph readout kernel with a bound for every element (DESIGN.md §3.5
gives the summation order).  With u = 2^-24 and gamma_k = k u / (1 - k u): a chunk's gate dot product is a per-lane fmaf chain
over H / 32 features, then a five-level butterfly: |dz| <= gamma_{H/32+5} sum_f |x_f w_f|.  s = 1 / (1 + expf(-z)): expf <= 2
ulp, the add and the division 1/2 ulp each, so |ds| <= s (1 - s) |dz| + 4 u s.  A chunk of at most CHUNK = 32 rows accumulates
fmaf(s, x, acc) in node order, then the graph's k chunks are added in chunk order from 0: |d g| <= gamma_{32 + k} sum_n s_n |x_n|
+ sum_n |x_n| |ds_n|; mean adds u |g|.  The float64 s is used in place of the computed one: the 1 % slack on the bound covers that.
"""
from typing import Optional

import torch
import torch.nn.functional as F

from oracle.ptgnn_oracle import gru_cell, scatter

CHUNK = 32
U = 2.0 ** -24


def _gamma(k):
    return k * U / (1 - k * U)


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


def readout_bound(x64: torch.Tensor, n2g: torch.Tensor, G: int, kind: str, w64: Optional[torch.Tensor]):
    """float64 readout ("weighted" / "sum" / "mean") of the rows x64 -> (g [G, H], bound [G, H], gate s [N])."""
    H = x64.shape[1]
    ax = x64.abs()
    if kind == "weighted":
        z = x64 @ w64.reshape(-1)
        s = torch.sigmoid(z)
        dz = _gamma(H // 32 + 5) * (ax @ w64.abs().reshape(-1))
        ds = s * (1 - s) * dz + 4 * U * s
    else:
        s = torch.ones(x64.shape[0], dtype=torch.float64)
        ds = torch.zeros_like(s)
    idx = n2g.reshape(-1, 1).expand(-1, H)
    g = torch.zeros(G, H, dtype=torch.float64).scatter_add_(0, idx, x64 * s[:, None])
    mass = torch.zeros(G, H, dtype=torch.float64).scatter_add_(0, idx, ax * s[:, None])
    prop = torch.zeros(G, H, dtype=torch.float64).scatter_add_(0, idx, ax * ds[:, None])
    count = torch.bincount(n2g, minlength=G).to(torch.float64)
    chunks = torch.ceil(count / CHUNK)
    bound = _gamma(CHUNK + chunks)[:, None] * mass + prop
    if kind == "mean":
        c = count.clamp(min=1)[:, None]
        g, bound = g / c, bound / c + U * (g / c).abs()
    return g, bound * 1.01, s
