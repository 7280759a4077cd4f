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


# ---- the attention readout kernel's backward (attn_readout.cu) ----------------------------------------------------------------
CHUNK = 32              # pergraph::CHUNK
U = 2.0 ** -24          # unit roundoff of fp32


def _gamma(n):
    return n * U / (1 - n * U)


def _kernel_backward(x, qt, o, lse, d_o, n2g, G, with_bound):
    """float64 (dx [N, D], d qt [G, heads, D]) and, if asked, their bounds, on x's device (one head at a time)."""
    x, qt, o, lse, d_o = (t.double() for t in (x, qt, o, lse, d_o))
    N, D = x.shape
    heads = qt.shape[1]
    dev = x.device
    n2g = n2g.to(dev)
    chunks = torch.ceil(torch.bincount(n2g, minlength=G).double() / CHUNK)[:, None]
    g_in = _gamma(D // 32 + 5)
    dx = torch.zeros(N, D, dtype=torch.float64, device=dev)
    dq = torch.zeros(G, heads, D, dtype=torch.float64, device=dev)
    b_dx, b_dq = torch.zeros_like(dx), torch.zeros_like(dq)
    mass = torch.zeros(N, D, dtype=torch.float64, device=dev)        # sum_h p |dO_h| + |ds qt_h|, for the 2 heads fmaf chain
    ax = x.abs()
    for h in range(heads):
        q, g = qt[:, h][n2g], d_o[:, h][n2g]                          # [N, D]
        z = (x * q).sum(1)
        p = torch.exp(z - lse[:, h][n2g])
        dp = (x * g).sum(1)
        delta = (o[:, h] * d_o[:, h]).sum(1)[n2g]
        ds = p * (dp - delta)
        dx += p[:, None] * g + ds[:, None] * q
        dq[:, h] = torch.zeros(G, D, dtype=torch.float64, device=dev).index_add_(0, n2g, ds[:, None] * x)
        if not with_bound:
            continue
        e_arg = g_in * (ax * q.abs()).sum(1) + U * (z - lse[:, h][n2g]).abs()
        e_p = p * (torch.expm1(e_arg) * (1 + 4 * U) + 4 * U) + 2.0 ** -148
        e_dp = g_in * (ax * g.abs()).sum(1)
        e_delta = g_in * (o[:, h] * d_o[:, h]).abs().sum(1)[n2g]
        diff = (dp - delta).abs()
        e_ds = e_p * diff + p * (e_dp + e_delta) + 2 * U * p * diff
        b_dx += e_p[:, None] * g.abs() + e_ds[:, None] * q.abs()
        mass += p[:, None] * g.abs() + (ds[:, None] * q).abs()
        b_dq[:, h] = (torch.zeros(G, D, dtype=torch.float64, device=dev).index_add_(0, n2g, e_ds[:, None] * ax)
                      + _gamma(CHUNK + chunks) * torch.zeros(G, D, dtype=torch.float64, device=dev).index_add_(0, n2g, (ds[:, None] * x).abs()))
    if not with_bound:
        return dx, dq
    b_dx += _gamma(2 * heads) * mass
    return dx, dq, b_dx * 1.01 + 1e-37, b_dq * 1.01 + 1e-37


def kernel_backward_formula(x, qt, o, lse, d_o, n2g, G):
    """(dx [N, D], d qt [G, heads, D]) in float64 from exactly the backward kernel's inputs x, qt, o, lse and d o (o and lse those of
    the forward kernel), on x's device: per node n of graph b and head h, z = x_n . qt[b, h], p = exp(z - lse[b, h]),
    delta = o[b, h] . dO[b, h], ds = p (x_n . dO[b, h] - delta); dx_n = sum_h p dO[b, h] + ds qt[b, h], d qt[b, h] = sum_n ds x_n.
    With the exact float64 o and lse this is the gradient of sum dO . o."""
    return _kernel_backward(x, qt, o, lse, d_o, n2g, G, False)


def kernel_backward_bound(x, qt, o, lse, d_o, n2g, G):
    """Per-element bounds (dx, d qt) on |kernel - kernel_backward_formula| for the fp32 backward kernel (DESIGN.md §3.7 / §4), in
    float64, from the order of attn_readout.cu's header.  With u = 2^-24, gamma_n = n u / (1 - n u), V = D / 32 features per lane
    and k chunks in the graph:
        z      e_arg = gamma_{V+5} sum_f |x_f qt_f| + u |z - lse|         (a lane's fmaf chain of V, a five-level butterfly; - lse)
        p      e_p = p (expm1(e_arg) (1 + 4u) + 4u) + 2^-148                (expf: 2 ulp = 4u; an underflow)
        dp     e_dp = gamma_{V+5} sum_f |x_f dO_f|,   delta  e_delta = gamma_{V+5} sum_f |o_f dO_f|
        ds     e_ds = e_p |dp - delta| + p (e_dp + e_delta) + 2u p |dp - delta|
        dx     sum_h (e_p |dO_h| + e_ds |qt_h|) + gamma_{2 heads} sum_h (p |dO_h| + |ds qt_h|)   (2 heads fmafs per feature)
        d qt   sum_n e_ds |x_n| + gamma_{32+k} sum_n |ds x_n|              (a chunk's chain of <= 32 rows, then k chunk additions)
    All terms are absolute, so cancellation in dp - delta is covered.  Second-order terms: 1 % slack, plus 1e-37 absolute."""
    return _kernel_backward(x, qt, o, lse, d_o, n2g, G, True)[2:]


def _fl(t):
    return t.float().double()


def _lane_dot(u, w):
    """A warp's dot product over the last dim as the kernel forms it: lane l's fmaf chain over features l, l + 32, ..., then the
    xor butterfly (lane 0's order), emulated in float64 with a rounding to float32 after every operation."""
    V = u.shape[-1] // 32
    uu, ww = u.reshape(*u.shape[:-1], V, 32), w.reshape(*w.shape[:-1], V, 32)
    acc = torch.zeros(torch.broadcast_shapes(uu.shape, ww.shape)[:-2] + (32,), dtype=torch.float64)
    for k in range(V):
        acc = _fl(uu[..., k, :] * ww[..., k, :] + acc)
    for half in (16, 8, 4, 2, 1):
        idx = torch.arange(32) ^ half
        acc = _fl(acc + acc[..., idx])
    return acc[..., 0]


def emulate_kernel_backward(x, qt, o, lse, d_o, n2g, G, warps=3, mutant=None):
    """float32 emulation of attn_readout_backward_chunk_kernel and the chunk sum (CPU, small shapes), with ``warps`` warps walking the
    chunks c = w, w + warps, ...  ``mutant`` (the bound must reject each): "no_ds_qt" drops the ds qt term of dx; "stale_delta" and
    "stale_qt" keep delta or qt of the warp's first graph when its graph changes; "drop_last_dq" drops a graph's last chunk's d qt
    partial."""
    x, qt, o, lse, d_o = (t.float().double() for t in (x, qt, o, lse, d_o))
    N, D = x.shape
    heads = qt.shape[1]
    counts = torch.bincount(n2g, minlength=G).tolist()
    order = torch.argsort(n2g, stable=True)
    chunk_list, start = [], 0                                        # (graph, positions) in chunk order
    for b, c in enumerate(counts):
        for s in range(0, c, CHUNK):
            chunk_list.append((b, order[start + s:start + min(c, s + CHUNK)]))
        start += c
    delta_of = _lane_dot(o, d_o)                                     # [G, heads]
    dx = torch.zeros(N, D, dtype=torch.float64)
    part = [None] * len(chunk_list)
    for w in range(warps):
        first = None
        for c in range(w, len(chunk_list), warps):
            b, nodes = chunk_list[c]
            first = b if first is None else first
            q = qt[first if mutant == "stale_qt" else b]
            delta = delta_of[first if mutant == "stale_delta" else b]
            dq = torch.zeros(heads, D, dtype=torch.float64)
            for n in nodes.tolist():
                xn, acc = x[n], torch.zeros(D, dtype=torch.float64)
                for h in range(heads):
                    z = _lane_dot(xn, q[h])
                    dp = _lane_dot(xn, d_o[b, h])
                    pr = _fl(torch.exp(_fl(z - lse[b, h])))
                    ds = _fl(pr * _fl(dp - delta[h]))
                    acc = _fl(pr * d_o[b, h] + acc)
                    if mutant != "no_ds_qt":
                        acc = _fl(ds * q[h] + acc)
                    dq[h] = _fl(ds * xn + dq[h])
                dx[n] = acc
            part[c] = dq
    d_qt = torch.zeros(G, heads, D, dtype=torch.float64)
    for c, (b, _) in enumerate(chunk_list):
        last = c + 1 == len(chunk_list) or chunk_list[c + 1][0] != b
        if not (mutant == "drop_last_dq" and last):
            d_qt[b] = _fl(d_qt[b] + part[c])
    return dx.float(), d_qt.float()
