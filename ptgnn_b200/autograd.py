"""Backward of ``GatedMessagePassingLayer`` (SURVEY.md §8 row f-1, first cut): makes the layer usable under ``torch.autograd``
(`/root/reference/ptgnn/baseneuralmodel/trainer.py:221-236` calls ``loss.backward()`` through the layers).

The forward is the unchanged native forward (fused aggregation + GRU kernels).  The backward re-computes what it needs and keeps the
edge-sized work on the native kernels:

* aggregate re-computation: ``edge_messages`` + ``segment_reduce`` kernels (with the arg-max edge ids for max / min);
* GRU: gate pre-activations and the two input-gradient products on the native dense kernel (``composed.linear``), the gate
  derivatives as pointwise torch ops;
* ``d h_src``: sum / mean -- the SAME gather -> Linear -> segmented-reduce kernels run on the transposed graph (edges reversed,
  weights ``W_t^T``, states = ``d agg``); max / min -- the routed message gradients times ``W_t`` on the dense kernel, then the
  native scatter-add by source;
* parameter gradients (``dW_t``, ``dW_ih``, ``dW_hh``): plain ``[out, rows] x [rows, in]`` GEMMs with a huge K (rows = edges or
  nodes) -- library GEMMs on the tensor cores in the forward's 3xFP16 split (three cuBLAS fp16 GEMMs with fp32 accumulation per
  product, operands scaled by a power of two first); bias gradients are column sums.

``MlpMessagePassingLayer`` (default message MLP) follows the same scheme; its node-sized tail (activation, LayerNorm, dense layer:
mlpmessagepassing.py:114-117) is differentiated by a local ``torch.autograd.grad`` over library ops, and its output Dropout is a torch
op applied outside the Function.

The gated layer's training-mode dropout (a per-edge mask on the gathered rows, gatedmessagepassing.py:59) and edge features under
autograd need the gathered ``[E_t, H]`` rows to exist: they run as the reference writes the layer, with the Linear / scatter / GRUCell
as differentiable native operators (``gated_forward_composed``).  fp32 states only.  Parity: ``tests/test_gpu_backward.py`` against ``torch.autograd`` through the CPU oracle (1e-4).
"""
import threading
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F_
from torch.autograd.function import once_differentiable

from . import _native as N
from . import composed as C
from .edgeplan import plan_for
from .scatter import scatter_sum


_TLS = threading.local()


class _suppress_output_dropout:
    """Inside an autograd.Function's forward the layer is re-entered under no_grad: its output dropout is applied OUTSIDE the
    Function (a differentiable torch op on the Function's result), not in the inner call."""

    def __enter__(self):
        self.previous = getattr(_TLS, "suppress", False)
        _TLS.suppress = True

    def __exit__(self, *exc):
        _TLS.suppress = self.previous
        return False


def output_dropout_suppressed() -> bool:
    return getattr(_TLS, "suppress", False)


def needs_grad(module: torch.nn.Module, node_states: torch.Tensor) -> bool:
    return torch.is_grad_enabled() and (node_states.requires_grad or any(p.requires_grad for p in module.parameters()))


class _exact_fp16_gemms:
    """cuBLAS fp16 GEMMs with fp32 accumulation all the way (no reduced-precision split-K reductions) while the split products run."""

    def __enter__(self):
        self.previous = torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction
        torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = self.previous
        return False


def _split16(x: torch.Tensor, scaled: bool = True, index: Optional[torch.Tensor] = None):
    """fp32 [rows, cols] -> (hi, lo, inv_scale) with (hi + lo / 2048) * inv_scale ~= x[index] (index: int32 row ids, None = all rows in
    order); hi, lo fp16: the 3xFP16 split of the forward kernels (22 significant bits).  scaled: first multiply by the power of two
    that brings the largest element to ~2^10 -- gradients are routinely below fp16's normal range (states and aggregates are not: the
    forward already requires them to fit).  Gather, scaling and split are one native pass; nothing synchronises."""
    rows = x.shape[0] if index is None else int(index.shape[0])
    cols = x.shape[1]
    hi = torch.empty(rows, cols, dtype=torch.float16, device=x.device)
    lo = torch.empty(rows, cols, dtype=torch.float16, device=x.device)
    if rows == 0 or x.numel() == 0:
        return hi, lo, 1.0
    scale, inv = None, 1.0
    if scaled:
        amax = torch.linalg.vector_norm(x, ord=float("inf")).clamp(min=1e-30)
        scale = torch.exp2(torch.floor(torch.log2(1024.0 / amax))).to(torch.float32)
        inv = 1.0 / scale
    x = x.contiguous()
    if cols % 8 != 0:      # rare shapes: torch ops
        v = x if index is None else x.index_select(0, index.long())
        v = v * scale if scale is not None else v
        hi = v.half()
        return hi, torch.sub(v, hi).mul_(2048.0).half(), inv
    with torch.cuda.device(x.device):
        rc = N.lib().ptgnn_b200_gather_split_f16(N.ptr(x), N.ptr(index), rows, cols, N.ptr(scale), N.ptr(hi), N.ptr(lo), N.current_stream(x.device))
    N.check(rc, "ptgnn_b200_gather_split_f16")
    return hi, lo, inv


def _mm_t_split(a, b):
    """A^T B in fp32 accuracy on the tensor cores for A = (hi, lo, inv) [K, M], B = (hi, lo, inv) [K, N]: three library fp16 GEMMs with
    fp32 accumulation (hi*hi + 2^-11 (hi*lo + lo*hi)) -- the K = edges / nodes parameter-gradient products were 39 % of a training
    step as fp32 SIMT GEMMs."""
    a_hi, a_lo, a_inv = a
    b_hi, b_lo, b_inv = b
    main = torch.mm(a_hi.t(), b_hi, out_dtype=torch.float32)
    corr = torch.mm(a_hi.t(), b_lo, out_dtype=torch.float32)
    corr.add_(torch.mm(a_lo.t(), b_hi, out_dtype=torch.float32))
    return main.add_(corr, alpha=1.0 / 2048.0).mul_(a_inv * b_inv)


def _slice(split, lo_, hi_):
    hi, lo, inv = split
    return hi[lo_:hi_], lo[lo_:hi_], inv


def _gru_backward(g, agg, h, w_ih, w_hh, b_ih, b_hh):
    """Gradients of torch.nn.GRUCell (gate order r, z, n) w.r.t. (input, hidden, weight_ih, weight_hh, bias_ih, bias_hh): gate
    pre-activations and the two input-gradient products on the native dense kernel, the gate derivatives in one native pointwise
    kernel, the parameter gradients ([3H, N] x [N, .], K = num_nodes) as split fp16 library GEMMs."""
    gi = C.linear(agg, w_ih, b_ih)
    gh = C.linear(h, w_hh, b_hh)
    d_gi, d_gh, d_h = torch.empty_like(gi), torch.empty_like(gh), torch.empty_like(h)
    with torch.cuda.device(h.device):
        rc = N.lib().ptgnn_b200_gru_gate_grads_f32(N.ptr(gi), N.ptr(gh), N.ptr(h), N.ptr(g), h.shape[0], h.shape[1], N.ptr(d_gi), N.ptr(d_gh),
                                                  N.ptr(d_h), N.current_stream(h.device))
    N.check(rc, "ptgnn_b200_gru_gate_grads_f32")
    d_h = d_h + C.linear(d_gh, w_hh.t().contiguous())                    # direct path + through W_hh
    d_agg = C.linear(d_gi, w_ih.t().contiguous())                        # [N, D]
    with _exact_fp16_gemms():
        s_gi, s_gh = _split16(d_gi), _split16(d_gh)
        d_w_ih, d_w_hh = _mm_t_split(s_gi, _split16(agg, False)), _mm_t_split(s_gh, _split16(h, False))
    return d_agg, d_h, d_w_ih, d_w_hh, d_gi.sum(dim=0), d_gh.sum(dim=0)


class _GatedLayerFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, layer, adjacency_lists, reduce_name, h, w_ih, w_hh, b_ih, b_hh, *weights):
        with torch.no_grad():
            out = layer(h.detach(), adjacency_lists)
        ctx.save_for_backward(h, w_ih, w_hh, b_ih, b_hh, *weights)
        ctx.adjacency_lists = adjacency_lists
        ctx.reduce_name = reduce_name
        return out

    @staticmethod
    @once_differentiable          # the backward runs native kernels: no double backward
    def backward(ctx, grad_out):
        h, w_ih, w_hh, b_ih, b_hh, *weights = ctx.saved_tensors
        adj: List[Tuple[torch.Tensor, torch.Tensor]] = ctx.adjacency_lists
        reduce_name = ctx.reduce_name
        reduce = N.REDUCE[reduce_name]
        g = grad_out.contiguous().float()
        h = h.detach().contiguous()
        num_nodes, H = h.shape
        W = [w.detach().contiguous() for w in weights]
        w_ih, w_hh = w_ih.detach().contiguous(), w_hh.detach().contiguous()
        plan = plan_for(adj, num_nodes)
        E = plan.num_edges

        # ---- 1. re-compute the aggregate (and, for max / min, which edge won each (target, feature))
        arg = None
        if reduce_name in ("max", "min"):
            msg = C.edge_messages(plan, h, None, W, False)                   # [E, D], cat(types) order
            agg, arg = C.segment_reduce(msg, plan, reduce, return_arg=True)
            del msg
        else:
            agg = C.aggregate(plan, h, W, reduce)                            # the fused kernel where it takes the dimensions

        # ---- 2. GRUCell backward
        d_agg, d_h, d_w_ih, d_w_hh, d_b_ih, d_b_hh = _gru_backward(g, agg, h, w_ih, w_hh, b_ih.detach(), b_hh.detach())

        # ---- 3. aggregation + per-type Linear backward
        d_W = []
        if reduce_name in ("sum", "mean"):
            if reduce_name == "mean":
                cnt = (plan.row_ptr[1:] - plan.row_ptr[:-1]).clamp(min=1).to(torch.float32)
                d_agg = d_agg / cnt[:, None]
            with _exact_fp16_gemms():
                a_all = _split16(d_agg, True, plan.tgt32)                    # [E, D] rows of d_agg, cat(types) order
                b_all = _split16(h, False, plan.src32)                       # [E, H] source states
                for t, w in enumerate(W):
                    lo_, hi_ = plan.type_off[t], plan.type_off[t + 1]
                    d_W.append(_mm_t_split(_slice(a_all, lo_, hi_), _slice(b_all, lo_, hi_)) if hi_ > lo_ else torch.zeros_like(w))
            if E > 0:
                # d h_src[u] = sum over edges (u -> v, type t) of W_t^T d_agg[v]: the forward's aggregation on the transposed graph
                rev = [(tgt, src) for src, tgt in adj]
                rplan = plan_for(rev, num_nodes)
                d_h = d_h + C.aggregate(rplan, d_agg.contiguous(), [w.t().contiguous() for w in W], N.REDUCE["sum"])
        else:
            D = d_agg.shape[1]
            d_msg = torch.zeros(E + 1, D, dtype=torch.float32, device=h.device)      # row E takes the empty targets' sentinel
            d_msg.scatter_(0, arg, d_agg)                                            # each (edge, feature) has one target: no collisions
            with _exact_fp16_gemms():
                a_all = _split16(d_msg[:E])
                b_all = _split16(h, False, plan.src32)
            lo = 0
            for (src, tgt), w in zip(adj, W):
                e_t = src.numel()
                part = d_msg[lo:lo + e_t]
                lo += e_t
                if e_t == 0:
                    d_W.append(torch.zeros_like(w))
                    continue
                with _exact_fp16_gemms():
                    d_W.append(_mm_t_split(_slice(a_all, lo - e_t, lo), _slice(b_all, lo - e_t, lo)))
                d_h = d_h + scatter_sum(C.linear(part.contiguous(), w.t().contiguous()), src, dim=0, dim_size=num_nodes)
        return (None, None, None, d_h, d_w_ih, d_w_hh, d_b_ih, d_b_hh, *d_W)


def gated_forward_with_grad(layer, node_states, adjacency_lists, reduce_name, w_ih, w_hh, b_ih, b_hh, weights):
    return _GatedLayerFunction.apply(layer, adjacency_lists, reduce_name, node_states, w_ih, w_hh, b_ih, b_hh, *weights)


# =====================================================================================================================
# MlpMessagePassingLayer (default message MLP: one bias-free Linear per edge type; string aggregation; no edge features)
#   out = state_update(message_activation(reduce_{e -> v} W_t [h_src(e) ; h_tgt(e)]))      mlpmessagepassing.py:68-117
# =====================================================================================================================
def _node_tail(agg: torch.Tensor, message_activation, ln, dense, dense_activation) -> torch.Tensor:
    """mlpmessagepassing.py:114-117 without the trailing Dropout: node-sized pointwise ops, LayerNorm and one [N, D] x [D, H] Linear."""
    x = agg if message_activation is None else message_activation(agg)
    if ln is not None:
        x = F_.layer_norm(x, ln.normalized_shape, ln.weight, ln.bias, ln.eps)
    if dense is not None:
        x = F_.linear(x, dense.weight, dense.bias)
        if dense_activation is not None:
            x = dense_activation(x)
    return x


class _MlpLayerFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, layer, adjacency_lists, reduce_name, use_target, modules, num_tail_params, h, *params):
        with torch.no_grad(), _suppress_output_dropout():
            out = layer(h.detach(), adjacency_lists)
        ctx.save_for_backward(h, *params)
        ctx.adjacency_lists, ctx.reduce_name, ctx.use_target = adjacency_lists, reduce_name, use_target
        ctx.modules, ctx.num_tail_params = modules, num_tail_params
        return out

    @staticmethod
    @once_differentiable          # the backward runs native kernels: no double backward
    def backward(ctx, grad_out):
        h, *params = ctx.saved_tensors
        tail_params, weights = params[:ctx.num_tail_params], params[ctx.num_tail_params:]
        adj: List[Tuple[torch.Tensor, torch.Tensor]] = ctx.adjacency_lists
        reduce_name, use_target = ctx.reduce_name, ctx.use_target
        message_activation, ln, dense, dense_activation = ctx.modules
        pna = None if isinstance(reduce_name, str) else reduce_name          # the native PnaMessageAggregation module
        g = grad_out.contiguous().float()
        h = h.detach().contiguous()
        num_nodes, H = h.shape
        W = [w.detach().contiguous() for w in weights]
        plan = plan_for(adj, num_nodes)
        E = plan.num_edges

        # ---- 1. re-compute the aggregate on the native kernels (PNA: with its arg ids; the messages are kept for its backward)
        msg = C.edge_messages(plan, h, h if use_target else None, W, use_target)
        arg = None
        if pna is not None:
            from .aggregation import native_pna

            agg, arg_max, arg_min = native_pna(msg, plan, pna.delta, want_arg=True)
        elif reduce_name in ("max", "min"):
            agg, arg = C.segment_reduce(msg, plan, N.REDUCE[reduce_name], return_arg=True)
        else:
            agg = C.segment_reduce(msg, plan, N.REDUCE[reduce_name])
        if pna is None:
            del msg

        # ---- 2. node-sized tail (activation, LayerNorm, dense): local autograd over library ops
        agg_leaf = agg.detach().requires_grad_(True)
        with torch.enable_grad():
            tail = _node_tail(agg_leaf, message_activation, ln, dense, dense_activation)
            wanted = [agg_leaf] + [p for p in tail_params if p.requires_grad]
            grads = torch.autograd.grad(tail, wanted, g, allow_unused=True)
        d_agg = grads[0].contiguous()
        it = iter(grads[1:])
        d_tail = [next(it) if p.requires_grad else None for p in tail_params]

        # ---- 3. aggregation + per-type Linear backward
        d_h = torch.zeros_like(h)
        d_W = []
        Ws = [w[:, :H].contiguous() for w in W]                              # columns multiplying h_src
        Wg = [w[:, H:].contiguous() for w in W] if use_target else None      # columns multiplying h_tgt
        if pna is None and reduce_name in ("sum", "mean"):
            if reduce_name == "mean":
                cnt = (plan.row_ptr[1:] - plan.row_ptr[:-1]).clamp(min=1).to(torch.float32)
                d_agg = (d_agg / cnt[:, None]).contiguous()
            with _exact_fp16_gemms():
                a_all, b_all = _split16(d_agg, True, plan.tgt32), _split16(h, False, plan.src32)
                g_all = _split16(h, False, plan.tgt32) if use_target else None
                for t, w in enumerate(W):
                    lo_, hi_ = plan.type_off[t], plan.type_off[t + 1]
                    if hi_ == lo_:
                        d_W.append(torch.zeros_like(w))
                        continue
                    a = _slice(a_all, lo_, hi_)
                    d_w = _mm_t_split(a, _slice(b_all, lo_, hi_))                                  # [D, H]: columns multiplying h_src
                    d_W.append(torch.cat([d_w, _mm_t_split(a, _slice(g_all, lo_, hi_))], dim=1) if use_target else d_w)
            if E > 0:
                rplan = plan_for([(tgt, src) for src, tgt in adj], num_nodes)                     # transposed graph: d h_src
                d_h = d_h + C.aggregate(rplan, d_agg, [w.t().contiguous() for w in Ws], N.REDUCE["sum"])
                if use_target:                                                                     # d h_tgt: every edge sends W_g^T d_agg[v] to its own target v
                    tplan = plan_for([(tgt, tgt) for _src, tgt in adj], num_nodes)
                    d_h = d_h + C.aggregate(tplan, d_agg, [w.t().contiguous() for w in Wg], N.REDUCE["sum"])
        else:
            # per-edge message gradients: routed to the winning edges (max / min), or the PNA backward
            if pna is not None:
                from .aggregation import native_pna_backward

                d_msg = native_pna_backward(msg, plan, pna.delta, agg, arg_max, arg_min, d_agg)
                del msg
            else:
                d_msg = torch.zeros(E + 1, d_agg.shape[1], dtype=torch.float32, device=h.device)
                d_msg = d_msg.scatter_(0, arg, d_agg)[:E]
            with _exact_fp16_gemms():
                a_all, b_all = _split16(d_msg), _split16(h, False, plan.src32)
                g_all = _split16(h, False, plan.tgt32) if use_target else None
            lo = 0
            for t, ((src, tgt), w) in enumerate(zip(adj, W)):
                e_t = src.numel()
                part = d_msg[lo:lo + e_t].contiguous()
                lo += e_t
                if e_t == 0:
                    d_W.append(torch.zeros_like(w))
                    continue
                with _exact_fp16_gemms():
                    a = _slice(a_all, lo - e_t, lo)
                    d_w = _mm_t_split(a, _slice(b_all, lo - e_t, lo))
                    d_W.append(torch.cat([d_w, _mm_t_split(a, _slice(g_all, lo - e_t, lo))], dim=1) if use_target else d_w)
                d_h = d_h + scatter_sum(C.linear(part, Ws[t].t().contiguous()), src, dim=0, dim_size=num_nodes)
                if use_target:
                    d_h = d_h + scatter_sum(C.linear(part, Wg[t].t().contiguous()), tgt, dim=0, dim_size=num_nodes)
        return (None, None, None, None, None, None, d_h, *d_tail, *d_W)


def mlp_forward_with_grad(layer, node_states, adjacency_lists, reduce_name, use_target, message_activation, ln, dense, dense_activation,
                          weights):
    """``reduce_name``: "sum", "mean", "max", "min", or the layer's native ``PnaMessageAggregation`` module."""
    tail_params: List[Optional[torch.Tensor]] = []
    if ln is not None:
        tail_params += [ln.weight, ln.bias]
    if dense is not None:
        tail_params += [dense.weight] + ([dense.bias] if dense.bias is not None else [])
    return _MlpLayerFunction.apply(layer, adjacency_lists, reduce_name, bool(use_target), (message_activation, ln, dense, dense_activation),
                                   len(tail_params), node_states, *tail_params, *weights)


# =====================================================================================================================
# Differentiable stand-alone operators: the composed path (edge features, per-edge dropout) under autograd
# =====================================================================================================================
class _LinearFn(torch.autograd.Function):
    """y = x W^T (+ b) on the native dense kernel; dx on the same kernel, dW / db as library GEMM / column sum."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return C.linear(x.detach().contiguous(), weight.detach().contiguous(), None if bias is None else bias.detach())

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, weight = ctx.saved_tensors
        g = g.contiguous()
        with _exact_fp16_gemms():
            d_w = _mm_t_split(_split16(g), _split16(x.detach()))
        return C.linear(g, weight.detach().t().contiguous()), d_w, (g.sum(dim=0) if ctx.has_bias else None)


class _SegmentReduceFn(torch.autograd.Function):
    """torch_scatter.scatter(messages, targets, reduce) on the native segmented-reduce kernel; backward = gather of the target's
    gradient (sum / mean) or routing to the winning edge (max / min, torch_scatter's arg semantics)."""

    @staticmethod
    def forward(ctx, messages, plan, reduce_name):
        ctx.plan, ctx.reduce_name = plan, reduce_name
        m = messages.detach().contiguous()
        if reduce_name in ("max", "min"):
            out, arg = C.segment_reduce(m, plan, N.REDUCE[reduce_name], return_arg=True)
            ctx.save_for_backward(arg)
            return out
        return C.segment_reduce(m, plan, N.REDUCE[reduce_name])

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        plan, reduce_name = ctx.plan, ctx.reduce_name
        g = g.contiguous()
        E = plan.num_edges
        if reduce_name in ("max", "min"):
            (arg,) = ctx.saved_tensors
            d_msg = torch.zeros(E + 1, g.shape[1], dtype=g.dtype, device=g.device)
            d_msg.scatter_(0, arg, g)
            return d_msg[:E], None, None
        if reduce_name == "mean":
            cnt = (plan.row_ptr[1:] - plan.row_ptr[:-1]).clamp(min=1).to(g.dtype)
            g = g / cnt[:, None]
        return g.index_select(0, plan.tgt32.long()), None, None


class _GRUCellFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, agg, h, w_ih, w_hh, b_ih, b_hh):
        import types

        ctx.save_for_backward(agg, h, w_ih, w_hh, b_ih, b_hh)
        shim = types.SimpleNamespace(weight_ih=w_ih.detach(), weight_hh=w_hh.detach(), bias_ih=b_ih.detach(), bias_hh=b_hh.detach())
        return C.grucell(agg.detach().contiguous(), h.detach().contiguous(), shim)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        agg, h, w_ih, w_hh, b_ih, b_hh = (t.detach() for t in ctx.saved_tensors)
        return _gru_backward(g.contiguous(), agg.contiguous(), h.contiguous(), w_ih.contiguous(), w_hh.contiguous(), b_ih, b_hh)


def gated_forward_composed(layer_weights, gru, node_states, adjacency_lists, edge_features, reduce_name, dropout_p: float):
    """GatedMessagePassingLayer.forward exactly as the reference writes it (gatedmessagepassing.py:46-69) -- gather, cat with the edge
    features, Dropout on the per-edge rows, per-type Linear, scatter, GRUCell -- with the Linear / scatter / GRUCell on the native
    kernels as differentiable operators.  Used where the [E_t, H] gathered rows must exist: per-edge dropout (training mode) and
    edge features under autograd."""
    num_nodes = node_states.shape[0]
    plan = plan_for(adjacency_lists, num_nodes)
    msgs = []
    for t, ((src, _tgt), w) in enumerate(zip(adjacency_lists, layer_weights)):
        x = F_.embedding(src, node_states)
        f = None if edge_features is None else edge_features[t]
        if f is not None and f.dim() == 2 and f.shape[1] > 0:
            x = torch.cat([x, f.to(x.dtype)], dim=-1)
        x = F_.dropout(x, dropout_p, dropout_p > 0)
        msgs.append(_LinearFn.apply(x, w, None))
    agg = _SegmentReduceFn.apply(torch.cat(msgs, dim=0), plan, reduce_name)
    return _GRUCellFn.apply(agg, node_states, gru.weight_ih, gru.weight_hh, gru.bias_ih, gru.bias_hh)


# =====================================================================================================================
# GruGlobalStateUpdate (globalgraphexchange.py:13-72): readout g = reduce_{n in b} s_n x_n, dropout on g (a torch op between the two
# Functions, so autograd keeps its mask), then h' = GRUCell(g[graph(n)], h_n).  fp32 states.
# =====================================================================================================================
class _GraphReadoutFn(torch.autograd.Function):
    """g [G, H] on the native readout (weighted sum, sum, mean) or the segmented reduce with arg-max node ids (max, min)."""

    @staticmethod
    def forward(ctx, kind, plan, node_to_graph_idx, h, gate_weight):
        from .reduceops import reduce_states

        x = h.detach().contiguous()
        ctx.kind, ctx.plan = kind, plan
        if kind in ("max", "min"):
            g, arg = C.segment_reduce(x, plan, N.REDUCE[kind], return_arg=True)
            ctx.save_for_backward(arg)
            return g
        g, s = reduce_states(kind, None if gate_weight is None else gate_weight.detach(), x, node_to_graph_idx, plan, want_gates=True)
        ctx.save_for_backward(x, s, gate_weight)
        return g

    @staticmethod
    @once_differentiable
    def backward(ctx, d_g):
        kind, plan = ctx.kind, ctx.plan
        d_g = d_g.contiguous()
        if kind in ("max", "min"):
            (arg,) = ctx.saved_tensors
            num_nodes = plan.num_edges
            d_x = torch.zeros(num_nodes + 1, d_g.shape[1], dtype=d_g.dtype, device=d_g.device)   # row N takes the empty graphs' sentinel
            d_x.scatter_(0, arg, d_g)                                                            # one graph per node: no collisions
            return None, None, None, d_x[:num_nodes], None
        x, s, w = ctx.saved_tensors
        gid = plan.tgt32.long()
        d_gn = d_g.index_select(0, gid)                                  # [N, H]: the gradient of each node's graph
        if kind == "mean":
            cnt = (plan.row_ptr[1:] - plan.row_ptr[:-1]).clamp(min=1).to(torch.float32)
            return None, None, None, d_gn / cnt.index_select(0, gid)[:, None], None
        if kind == "sum":
            return None, None, None, d_gn, None
        # weighted sum: d x_n = s_n d g_b + s_n (1 - s_n) (x_n . d g_b) w ;  d w = sum_n s_n (1 - s_n) (x_n . d g_b) x_n
        q = s * (1.0 - s) * (x * d_gn).sum(dim=1)
        d_x = s[:, None] * d_gn + q[:, None] * w.detach().reshape(1, -1)
        return None, None, None, d_x, (q[None, :] @ x) if w.requires_grad else None


def graph_readout_with_grad(kind, gate_weight, node_states, node_to_graph_idx, plan):
    return _GraphReadoutFn.apply(kind, plan, node_to_graph_idx, node_states, gate_weight)


class _GlobalGruFn(torch.autograd.Function):
    """h' = GRUCell(g[graph(n)], h_n) on the table GRU kernel; backward: the GRUCell backward with the input side reduced per graph."""

    @staticmethod
    def forward(ctx, layer, plan, h, g, w_ih, w_hh, b_ih, b_hh):
        with torch.no_grad():
            out = layer.table_update(h.detach(), g.detach(), plan)
        ctx.save_for_backward(h, g, w_ih, w_hh, b_ih, b_hh)
        ctx.plan = plan
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        h, g, w_ih, w_hh, b_ih, b_hh = (t.detach().contiguous() for t in ctx.saved_tensors)
        plan = ctx.plan
        gi = C.linear(g, w_ih, b_ih).index_select(0, plan.tgt32.long())     # the [G, 3H] table, gathered per node
        gh = C.linear(h, w_hh, b_hh)
        d_gi, d_gh, d_h = torch.empty_like(gi), torch.empty_like(gh), torch.empty_like(h)
        with torch.cuda.device(h.device):
            rc = N.lib().ptgnn_b200_gru_gate_grads_f32(N.ptr(gi), N.ptr(gh), N.ptr(h), N.ptr(grad_out.contiguous()), h.shape[0], h.shape[1],
                                                      N.ptr(d_gi), N.ptr(d_gh), N.ptr(d_h), N.current_stream(h.device))
        N.check(rc, "ptgnn_b200_gru_gate_grads_f32")
        d_h = d_h + C.linear(d_gh, w_hh.t().contiguous())
        d_table = C.segment_reduce(d_gi, plan, N.REDUCE["sum"])             # [G, 3H]: per graph, in node order
        d_g = C.linear(d_table, w_ih.t().contiguous())                      # [G, S]
        with _exact_fp16_gemms():
            d_w_hh = _mm_t_split(_split16(d_gh), _split16(h, False))
        return None, None, d_h, d_g, d_table.t() @ g, d_w_hh, d_table.sum(dim=0), d_gh.sum(dim=0)


def global_gru_with_grad(layer, node_states, summaries, plan, w_ih, w_hh, b_ih, b_hh):
    return _GlobalGruFn.apply(layer, plan, node_states, summaries, w_ih, w_hh, b_ih, b_hh)


# =====================================================================================================================
# Attention readout (varsizedsummary.py:84-178): o[b, h] = sum_n softmax_n(x_n . qt[b, h]) x_n on the native kernel; the G-row products
# around it (qt from the queries and the key weight, value and output layers) are _LinearFn's.  fp32 states.
# =====================================================================================================================
class _AttentionReadoutFn(torch.autograd.Function):
    """o [G, heads, D] from x [N, D] and qt [G, heads, D]; backward: d x and d qt on the native backward kernel (p re-computed from
    the saved lse, no [N, heads] tensor kept)."""

    @staticmethod
    def forward(ctx, plan, heads, x, qt):
        from .reduceops import native_attention_readout

        xd, qd = x.detach().contiguous(), qt.detach().contiguous()
        o, lse = native_attention_readout(xd, plan, qd, heads)
        ctx.save_for_backward(xd, qd, o, lse)
        ctx.plan = plan
        return o

    @staticmethod
    @once_differentiable
    def backward(ctx, d_o):
        from .reduceops import native_attention_readout_backward

        x, qt, o, lse = ctx.saved_tensors
        d_x, d_qt = native_attention_readout_backward(x, ctx.plan, qt, o, lse, d_o.contiguous().float())
        return None, None, d_x, d_qt


def attention_readout_with_grad(plan, heads, node_states, qt):
    return _AttentionReadoutFn.apply(plan, heads, node_states, qt)


# =====================================================================================================================
# MultiHeadSelfAttentionMessagePassing (selfattmessagepassing.py:92-117): o_i = sum_j softmax_j(a_i . b_j / sqrt(dk)) v_j within the
# chunks of each graph, on the native kernel; the node-sized products around it are _LinearFn's.  fp32 states.
# =====================================================================================================================
class _SelfAttentionFn(torch.autograd.Function):
    """o [R, heads * dv] from t [R, heads * (2 dk + dv)]; backward: d t on the native backward kernels (p re-computed from the saved
    lse: no [L, L] tensor is kept)."""

    @staticmethod
    def forward(ctx, plan, heads, dk, dv, max_chunk, t):
        from .selfattention import native_selfatt

        td = t.detach().contiguous()
        o, lse = native_selfatt(td, plan, heads, dk, dv, max_chunk)
        ctx.save_for_backward(td, o, lse)
        ctx.plan, ctx.dims = plan, (heads, dk, dv, max_chunk)
        return o

    @staticmethod
    @once_differentiable
    def backward(ctx, d_o):
        from .selfattention import native_selfatt_backward

        t, o, lse = ctx.saved_tensors
        d_t = native_selfatt_backward(t, ctx.plan, *ctx.dims, o, lse, d_o.contiguous().float())
        return None, None, None, None, None, d_t


def selfatt_with_grad(plan, heads, dk, dv, max_chunk, t):
    return _SelfAttentionFn.apply(plan, heads, dk, dv, max_chunk, t)


# =====================================================================================================================
# GraphNorm (graphnorm.py:36-46): y = gamma (x - alpha mu_g) / sqrt(sigma_g^2) + bias per graph, on the native kernels.  fp32 states.
# =====================================================================================================================
class _GraphNormFn(torch.autograd.Function):
    """y [N, D] from x [N, D] and the [1, D] parameters; backward: d x and the parameter gradients on the native backward kernels
    (the normalised states are recomputed from the saved [G, D] mean and rstd: no [N, D] tensor is kept besides x)."""

    @staticmethod
    def forward(ctx, plan, eps, x, gamma, alpha, bias):
        from .graphnorm import native_graph_norm

        xd = x.detach().contiguous()
        y, mean, rstd = native_graph_norm(xd, plan, gamma, alpha, bias, eps)
        ctx.save_for_backward(xd, gamma, alpha, mean, rstd)
        ctx.plan, ctx.eps = plan, eps
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, d_y):
        from .graphnorm import native_graph_norm_backward

        x, gamma, alpha, mean, rstd = ctx.saved_tensors
        d_x, d_gamma, d_alpha, d_bias = native_graph_norm_backward(x, ctx.plan, gamma, alpha, ctx.eps, mean, rstd, d_y.contiguous().float())
        return None, None, d_x, d_gamma.reshape(gamma.shape), d_alpha.reshape(alpha.shape), d_bias.reshape(gamma.shape)


def graph_norm_with_grad(plan, eps, node_states, gamma, alpha, bias):
    return _GraphNormFn.apply(plan, eps, node_states, gamma, alpha, bias)


# =====================================================================================================================
# PnaMessageAggregation (pna_aggregation.py:27-56): [S | S p1 | S m1] per target on the native kernel.  fp32 messages.
# =====================================================================================================================
class _PnaFn(torch.autograd.Function):
    """out [N, 15 D] from messages [E, D]; backward: d messages on the native backward kernel, which reads the mean and std back from
    the saved output and the max / min winners from the saved [N, D] arg ids (no [E, D] tensor is kept besides the messages)."""

    @staticmethod
    def forward(ctx, plan, delta, messages):
        from .aggregation import native_pna

        m = messages.detach()
        out, arg_max, arg_min = native_pna(m, plan, delta, want_arg=True)
        ctx.save_for_backward(m, out, arg_max, arg_min)
        ctx.plan, ctx.delta = plan, delta
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        from .aggregation import native_pna_backward

        m, out, arg_max, arg_min = ctx.saved_tensors
        return None, None, native_pna_backward(m, ctx.plan, ctx.delta, out, arg_max, arg_min, d_out.contiguous().float())


def pna_with_grad(plan, delta, messages):
    return _PnaFn.apply(plan, delta, messages)


# =====================================================================================================================
# TokenUnitEmbedder / SubtokenUnitEmbedder (strelementrepresentationmodel.py:16-89): the pooled table rows on the native embedding-bag
# kernel.  fp32 output.
# =====================================================================================================================
class _EmbeddingBagFn(torch.autograd.Function):
    """out [B, D] from table [V, D] and ids [B, S]; backward: d table on the native sorted, atomic-free kernel.  Saves the ids, the
    lengths and (max) the [B, D] uint8 winning slots: no [B, S, D] tensor exists in either direction."""

    @staticmethod
    def forward(ctx, table, ids, lengths, mode, status):
        from .embeddings import native_embedding_bag

        out, arg = native_embedding_bag(table.detach(), ids, lengths, mode, want_arg=True, status=status)
        ctx.save_for_backward(ids, lengths, arg)     # an in-place change of the ids before the backward is then an error, not a wrong gradient
        ctx.mode, ctx.vocab = mode, table.shape[0]
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        from .embeddings import native_embedding_bag_backward

        ids, lengths, arg = ctx.saved_tensors
        d_table = native_embedding_bag_backward(d_out.contiguous().float(), ids, lengths, ctx.mode, ctx.vocab, arg)
        return d_table, None, None, None, None


def embedding_bag_with_grad(table, ids, lengths, mode, status=None):
    return _EmbeddingBagFn.apply(table, ids, lengths, mode, status)


# =====================================================================================================================
# GruCopyingDecoder (grucopydecoder.py:95-97, 122-124): the copy scores s[i, l] = c_i . o[graph(i), l] and their per-sample logsumexp
# on the native kernel.  fp32 copy representations.
# =====================================================================================================================
class _CopyAttentionFn(torch.autograd.Function):
    """(s [M, L], lse [G, L]) from c [M, H] and o [G, L, H]; backward: d c and d o on the native backward kernel (s and p re-computed
    from c, o and the saved lse: no [M, L] tensor is kept)."""

    @staticmethod
    def forward(ctx, plan, c, o):
        from .decoder import native_copy_attention

        cd, od = c.detach().contiguous(), o.detach().contiguous()
        s, lse = native_copy_attention(cd, plan, od)
        ctx.save_for_backward(cd, od, lse)
        ctx.plan = plan
        return s, lse

    @staticmethod
    @once_differentiable
    def backward(ctx, d_s, d_lse):
        from .decoder import native_copy_attention_backward

        c, o, lse = ctx.saved_tensors
        d_c, d_o = native_copy_attention_backward(c, ctx.plan, o, lse, d_s.contiguous().float(), d_lse.contiguous().float())
        return None, d_c, d_o


def copy_attention_with_grad(plan, copy_reps, o):
    return _CopyAttentionFn.apply(plan, copy_reps, o)


class _GatherByGraphFn(torch.autograd.Function):
    """x[graph(row)] [M, L] for x [G, L] and the rows of a graph plan; backward: the rows of each graph summed in row order on the native
    segmented reduce (columns padded to a multiple of 4).  The library's backward of an index gather adds with float atomics, so its
    result changes from run to run."""

    @staticmethod
    def forward(ctx, plan, index, x):
        ctx.plan = plan
        return x.index_select(0, index)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        L = g.shape[1]
        g = F_.pad(g.contiguous().float(), (0, (-L) % 4))
        return None, None, C.segment_reduce(g, ctx.plan, N.REDUCE["sum"])[:, :L]


def gather_by_graph(plan, index, x):
    return _GatherByGraphFn.apply(plan, index, x)
