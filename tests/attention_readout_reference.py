"""CPU restatement of the reference's attention reducers for the tests (like ``global_exchange_reference.py``), with the reference's own
ops and the oracle's ``scatter`` (torch_scatter semantics):

* ``self_attention_forward``           -> ``ptgnn/neuralmodels/reduceops/varsizedsummary.py:100-113``
* ``multihead_self_attention_forward`` -> ``ptgnn/neuralmodels/reduceops/varsizedsummary.py:145-178``

``queries`` is the query summarizer's output [G, hidden] (``global_exchange_reference.graph_readout`` restates the Simple and WeightedSum
summarizers).  The segmented log-softmax is ``torch_scatter.scatter_log_softmax(..., eps=0)``; its per-graph maximum is taken without
gradient (the log-softmax does not depend on it).  Pinned to the reference's outputs by ``test_oracle_attention_readout.py`` (fixtures
written by ``golden/generate_attention_readout_golden.py``).  Works in any dtype, float64 included, and under autograd.
"""
from math import sqrt
from typing import Optional

import torch
import torch.nn.functional as F

from oracle.ptgnn_oracle import scatter


def segment_log_softmax(scores: torch.Tensor, index: torch.Tensor) -> torch.Tensor:
    """scores [N] or [N, heads], per segment of ``index`` along dim 0."""
    n = int(index.max()) + 1 if index.numel() else 0
    idx = index.reshape((-1,) + (1,) * (scores.dim() - 1)).expand(scores.size())
    with torch.no_grad():
        mx = torch.full((n,) + tuple(scores.shape[1:]), float("-inf"), dtype=scores.dtype)
        mx.scatter_reduce_(0, idx, scores.detach(), "amax", include_self=True)
    centred = scores - mx.gather(0, idx)
    s = torch.zeros_like(mx).scatter_add_(0, idx, centred.exp())
    return centred - s.log().gather(0, idx)


def self_attention_forward(x: torch.Tensor, node_to_graph_idx: torch.Tensor, num_graphs: int, queries: torch.Tensor, key_weight: torch.Tensor,
                           output_weight: torch.Tensor) -> torch.Tensor:
    queries_all = queries[node_to_graph_idx]
    keys = F.linear(x, key_weight)
    scores = torch.einsum("vh,vh->v", queries_all, keys)
    probs = torch.exp(segment_log_softmax(scores, node_to_graph_idx))
    return scatter(F.linear(x, output_weight) * probs.unsqueeze(-1), node_to_graph_idx, num_graphs, "sum")


def multihead_self_attention_forward(x: torch.Tensor, node_to_graph_idx: torch.Tensor, num_graphs: int, queries: torch.Tensor,
                                     key_weight: torch.Tensor, num_heads: int, output_weight: torch.Tensor,
                                     value_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    n = x.shape[0]
    q = queries[node_to_graph_idx]
    q = q.reshape((n, num_heads, q.shape[1] // num_heads))
    keys = F.linear(x, key_weight)
    keys = keys.reshape((n, num_heads, keys.shape[1] // num_heads))
    scores = torch.einsum("bhk,bhk->bh", q, keys) / sqrt(keys.shape[-1])
    probs = torch.exp(segment_log_softmax(scores, node_to_graph_idx))
    if value_weight is not None:
        values = F.linear(x, value_weight)
        outputs = probs.unsqueeze(-1) * values.reshape((n, num_heads, values.shape[1] // num_heads))
    else:
        outputs = probs.unsqueeze(-1) * x.unsqueeze(1)
    per_sample = scatter(outputs.reshape((n, -1)), node_to_graph_idx, num_graphs, "sum")
    return F.linear(per_sample, output_weight)
