"""Backward passes of the native layers and operators, so that they train under ``torch.autograd`` (the reference's trainer calls
``loss.backward()`` through the layers: ptgnn/baseneuralmodel/trainer.py:221-236).

Each Function's forward is the unchanged native forward.  Its backward re-computes what it needs and keeps the edge-sized work on the
native kernels.  The three trainable message-passing layers (gated, Mlp with the default message MLP, EGC) share one backward for
their aggregation agg = reduce_{e -> v} W_t(e) [h_src(e) ; h_tgt(e)], ``_aggregation_backward``:

* ``d h``: sum / mean -- the forward's aggregation kernels on the transposed graph (edges reversed, or from each target to itself
  for the ``h_tgt`` columns; weights ``W_t^T``; states ``d agg`` scaled by a power of two); max / min and PNA -- the per-edge message
  gradients times ``W_t`` on the dense kernel, then the native scatter-add by source (and by target for the ``h_tgt`` columns);
* parameter gradients (``dW_t``, and the GRU's ``dW_ih``, ``dW_hh``): plain ``[out, rows] x [rows, in]`` GEMMs with a huge K (rows =
  edges or nodes) -- library GEMMs on the tensor cores in the forward's 3xFP16 split (``_mm_t_split``: three cuBLAS fp16 GEMMs with
  fp32 accumulation per product, operands scaled by a power of two first); bias gradients are column sums.

The GRUs (gated layer, GruGlobalStateUpdate) take their gate pre-activations and input-gradient products on the native dense kernel
(``composed.linear``) and the gate derivatives from one native pointwise kernel (``_gru_gate_grads``).  The Mlp layer's node-sized
tail (activation, LayerNorm, dense layer: mlpmessagepassing.py:114-117) is differentiated by a local ``torch.autograd.grad`` over
library ops, and its output Dropout is a torch op applied outside the Function.

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


def _pow2_scale(x: torch.Tensor):
    """(scale, inv_scale) as fp32 device scalars: the power of two that brings the largest |element| of x to [512, 1024).  Multiplying
    by it is exact in fp32's normal range, and nothing synchronises."""
    amax = torch.linalg.vector_norm(x, ord=float("inf")).clamp(min=1e-30)
    scale = torch.exp2(torch.floor(torch.log2(1024.0 / amax))).to(torch.float32)
    return scale, 1.0 / scale


def _split16(x: torch.Tensor, index: Optional[torch.Tensor] = None, scale=None):
    """fp32 [rows, cols] -> (hi, lo, inv_scale) with (hi + lo / 2048) * inv_scale ~= x[index] (index: int32 row ids, None = all rows in
    order); hi, lo fp16: the 3xFP16 split of the forward kernels (22 significant bits) of x times ``_pow2_scale(x)``.  The scaling keeps
    gradients (routinely below fp16's normal range) and states beyond fp16's range (PTGNN_B200_FP32_MODE=tf32) at full precision.
    scale: that pair when the caller already has it.  Gather, scaling and split are one native pass; nothing synchronises."""
    rows = x.shape[0] if index is None else int(index.shape[0])
    cols = x.shape[1]
    hi = torch.empty(rows, cols, dtype=torch.float16, device=x.device)
    lo = torch.empty(rows, cols, dtype=torch.float16, device=x.device)
    if rows == 0 or x.numel() == 0:
        return hi, lo, 1.0
    scale, inv = _pow2_scale(x) if scale is None else scale
    x = x.contiguous()
    if cols % 8 != 0:      # rare shapes: torch ops
        v = x if index is None else x.index_select(0, index.long())
        v = v * scale
        hi = v.half()
        return hi, torch.sub(v, hi).mul_(2048.0).half(), inv
    N.call("ptgnn_b200_gather_split_f16", x.device, N.ptr(x), N.ptr(index), rows, cols, N.ptr(scale), N.ptr(hi), N.ptr(lo))
    return hi, lo, inv


def _add_aggregate(d_h: torch.Tensor, plan, x: torch.Tensor, weights, scale) -> torch.Tensor:
    """d_h + sum_{e -> v} W_t(e) x[src(e)] for a gradient x: ``C.aggregate`` on x times its ``_pow2_scale`` pair ``scale``, scaled back in
    the add.  The fused kernel splits its operand into fp16 pairs without scaling, which represents x only to 2^-36 absolute (no
    precision left for a gradient of 1e-8) and overflows at 65504; the power of two makes both exact in fp32's normal range."""
    s, inv = scale
    return torch.addcmul(d_h, C.aggregate(plan, x * s, weights, N.REDUCE["sum"]), inv)


def _mm_t_split(a, b):
    """A^T B in fp32 accuracy on the tensor cores for A = (hi, lo, inv) [K, M], B = (hi, lo, inv) [K, N]: three library fp16 GEMMs with
    fp32 accumulation (hi*hi + 2^-11 (hi*lo + lo*hi)) -- the K = edges / nodes parameter-gradient products were 39 % of a training
    step as fp32 SIMT GEMMs.  The GEMMs accumulate in fp32 all the way: reduced-precision split-K reductions are off while they run."""
    a_hi, a_lo, a_inv = a
    b_hi, b_lo, b_inv = b
    matmul = torch.backends.cuda.matmul
    previous = matmul.allow_fp16_reduced_precision_reduction
    matmul.allow_fp16_reduced_precision_reduction = False
    try:
        main = torch.mm(a_hi.t(), b_hi, out_dtype=torch.float32)
        corr = torch.mm(a_hi.t(), b_lo, out_dtype=torch.float32)
        corr.add_(torch.mm(a_lo.t(), b_hi, out_dtype=torch.float32))
    finally:
        matmul.allow_fp16_reduced_precision_reduction = previous
    return main.add_(corr, alpha=1.0 / 2048.0).mul_(a_inv * b_inv)


def _slice(split, lo_, hi_):
    hi, lo, inv = split
    return hi[lo_:hi_], lo[lo_:hi_], inv


def _mean_divisor(plan) -> torch.Tensor:
    """[segments] fp32: each segment's length (a target's in-degree, a graph's node count), at least 1 -- what mean divides by."""
    return (plan.row_ptr[1:] - plan.row_ptr[:-1]).clamp(min=1).to(torch.float32)


def _route_to_arg(g: torch.Tensor, arg: torch.Tensor, rows: int) -> torch.Tensor:
    """Backward of a max / min reduction over ``rows`` input rows: [rows, C] zeros with each element g[v, c] at row arg[v, c].  Empty
    segments point at the sentinel row ``rows``, which is dropped; every (row, column) belongs to one segment, so nothing collides."""
    return torch.zeros(rows + 1, g.shape[1], dtype=g.dtype, device=g.device).scatter_(0, arg, g)[:rows]


def _gru_gate_grads(g, gi, gh, h, w_hh):
    """(d gi, d gh, d h) of torch.nn.GRUCell (gate order r, z, n) from its gate pre-activations gi, gh: the gate derivatives in one native
    pointwise kernel; d h is the direct path plus the product through W_hh on the native dense kernel."""
    d_gi, d_gh, d_h = torch.empty_like(gi), torch.empty_like(gh), torch.empty_like(h)
    N.call("ptgnn_b200_gru_gate_grads_f32", h.device, N.ptr(gi), N.ptr(gh), N.ptr(h), N.ptr(g), h.shape[0], h.shape[1], N.ptr(d_gi),
           N.ptr(d_gh), N.ptr(d_h))
    return d_gi, d_gh, d_h + C.linear(d_gh, w_hh.t().contiguous())


def _gru_backward(g, agg, h, w_ih, w_hh, b_ih, b_hh):
    """Gradients of torch.nn.GRUCell w.r.t. (input, hidden, weight_ih, weight_hh, bias_ih, bias_hh): gate pre-activations and the two
    input-gradient products on the native dense kernel, the parameter gradients ([3H, N] x [N, .], K = num_nodes) as split fp16
    library GEMMs."""
    d_gi, d_gh, d_h = _gru_gate_grads(g, C.linear(agg, w_ih, b_ih), C.linear(h, w_hh, b_hh), h, w_hh)
    d_agg = C.linear(d_gi, w_ih.t().contiguous())                        # [N, D]
    d_w_ih, d_w_hh = _mm_t_split(_split16(d_gi), _split16(agg)), _mm_t_split(_split16(d_gh), _split16(h))
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
        g = grad_out.contiguous().float()
        h = h.detach().contiguous()
        W = [w.detach().contiguous() for w in weights]
        w_ih, w_hh = w_ih.detach().contiguous(), w_hh.detach().contiguous()
        plan = plan_for(adj, h.shape[0])
        agg, arg = _recompute_aggregate(plan, h, W, ctx.reduce_name)
        d_agg, d_h, d_w_ih, d_w_hh, d_b_ih, d_b_hh = _gru_backward(g, agg, h, w_ih, w_hh, b_ih.detach(), b_hh.detach())
        d_W, d_h = _aggregation_backward(plan, adj, h, W, d_agg, ctx.reduce_name, arg, d_h)
        return (None, None, None, d_h, d_w_ih, d_w_hh, d_b_ih, d_b_hh, *d_W)


def _recompute_aggregate(plan, h, W, reduce_name):
    """(agg, arg) of agg = reduce_{e -> v} W_t(e) h[src(e)]: arg, for max / min, is which edge won each (target, feature), from the
    messages and the segmented reduce; sum / mean run the fused kernel where it takes the dimensions, and arg is None."""
    if reduce_name in ("max", "min"):
        msg = C.edge_messages(plan, h, None, W, False)                       # [E, D], cat(types) order
        return C.segment_reduce(msg, plan, N.REDUCE[reduce_name], return_arg=True)
    return C.aggregate(plan, h, W, N.REDUCE[reduce_name]), None


def _aggregation_backward(plan, adj, h, W, d_agg, reduce_name, arg, d_h, b_all=None, *, W_tgt=None, d_msg=None):
    """Backward of agg = reduce_{e -> v} W_t(e) [h[src(e)] ; h[tgt(e)]] (bias-free per-type Linear, then sum / mean / max / min) from
    d_agg [N, D]: returns (d_W per type, d_h + the h part).  W: the columns of W_t that multiply h_src; W_tgt: those that multiply h_tgt
    (None: the messages read h_src only), and d_W[t] is then [d W_src ; d W_tgt] along dim 1.  arg: the winning edge ids of max / min
    ([N, D], E for empty targets).  d_msg: the per-edge message gradients [E, D] when the caller has them (PNA's backward); they replace
    the routing of d_agg through arg.  b_all: the 3xFP16 split of the gathered source states, ``_split16(h, plan.src32)``, when the
    caller reuses it across calls.
    sum / mean: split fp16 GEMMs over edges, and the forward's aggregation with W_t^T on the transposed graph (and, for h_tgt, on the
    graph of each edge's target to itself); otherwise: split fp16 GEMMs over the message gradients, and per type the native linear
    with W_t^T and scatter-add by source (and by target)."""
    num_nodes = h.shape[0]
    E = plan.num_edges
    dense = d_msg is None and reduce_name in ("sum", "mean")
    if dense:
        if reduce_name == "mean":
            d_agg = d_agg / _mean_divisor(plan)[:, None]
        d_agg = d_agg.contiguous()
        scale = _pow2_scale(d_agg)                                       # one scale for a_all and the transposed aggregations
        a_all = _split16(d_agg, plan.tgt32, scale)                       # [E, D] rows of d_agg, cat(types) order
    else:
        if d_msg is None:
            d_msg = _route_to_arg(d_agg, arg, E)
        a_all = _split16(d_msg)
    if b_all is None:
        b_all = _split16(h, plan.src32)                                  # [E, H] source states
    g_all = None if W_tgt is None else _split16(h, plan.tgt32)           # [E, H] target states
    d_W = []
    for t, ((src, tgt), w) in enumerate(zip(adj, W)):
        lo, hi = plan.type_off[t], plan.type_off[t + 1]
        if hi == lo:
            d_W.append(w.new_zeros(w.shape[0], w.shape[1] + (0 if W_tgt is None else W_tgt[t].shape[1])))
            continue
        a = _slice(a_all, lo, hi)
        d_w = _mm_t_split(a, _slice(b_all, lo, hi))
        d_W.append(d_w if W_tgt is None else torch.cat([d_w, _mm_t_split(a, _slice(g_all, lo, hi))], dim=1))
        if not dense:
            part = d_msg[lo:hi].contiguous()
            d_h = d_h + scatter_sum(C.linear(part, w.t().contiguous()), src, dim=0, dim_size=num_nodes)
            if W_tgt is not None:
                d_h = d_h + scatter_sum(C.linear(part, W_tgt[t].t().contiguous()), tgt, dim=0, dim_size=num_nodes)
    if dense and E > 0:
        # d h_src[u] = sum over edges (u -> v, type t) of W_t^T d_agg[v]: the forward's aggregation on the transposed graph
        rplan = plan_for([(tgt, src) for src, tgt in adj], num_nodes)
        d_h = _add_aggregate(d_h, rplan, d_agg, [w.t().contiguous() for w in W], scale)
        if W_tgt is not None:      # d h_tgt: every edge sends W_tgt^T d_agg[v] to its own target v
            tplan = plan_for([(tgt, tgt) for _src, tgt in adj], num_nodes)
            d_h = _add_aggregate(d_h, tplan, d_agg, [w.t().contiguous() for w in W_tgt], scale)
    return d_W, d_h


def gated_forward_with_grad(layer, node_states, adjacency_lists, reduce_name, w_ih, w_hh, b_ih, b_hh, weights):
    return _GatedLayerFunction.apply(layer, adjacency_lists, reduce_name, node_states, w_ih, w_hh, b_ih, b_hh, *weights)


# =====================================================================================================================
# EGCMessagePassingLayer (egcmessagepassing.py:54-91) on its fused slabs (DESIGN.md §3.14):
#   out[n, o] = sum_b w[n, hd bases + b] A[n, r(o, b)],  w = h Wc^T + bc,  A = reduce_{e -> n} W_t(e) h[src(e)],  r(o, b) = (hd bases + b) dh + c
# =====================================================================================================================
def egc_slab_rows(s: int, out: int, heads: int, bases: int, device) -> torch.Tensor:
    """Reference rows of bases[t].weight in slab s: position p = j bases + b <- row r(o, b), o = s 128 / bases + j."""
    p = torch.arange(128, device=device)
    o = s * (128 // bases) + p // bases
    dh = out // heads
    return ((o // dh) * bases + p % bases) * dh + o % dh


class _EgcLayerFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, layer, adjacency_lists, reduce_name, dims, h, coeff_weight, coeff_bias, *weights):
        with torch.no_grad():
            out = layer(h.detach(), adjacency_lists)
        ctx.save_for_backward(h, coeff_weight, coeff_bias, *weights)
        ctx.adjacency_lists, ctx.reduce_name, ctx.dims = adjacency_lists, reduce_name, dims
        return out

    @staticmethod
    @once_differentiable          # the backward runs native kernels: no double backward
    def backward(ctx, grad_out):
        h, cw, cb, *weights = (t.detach() for t in ctx.saved_tensors)
        adj = ctx.adjacency_lists
        reduce_name = ctx.reduce_name
        _in_dim, out, heads, bases = ctx.dims
        g = grad_out.contiguous().float()
        h, cw = h.contiguous(), cw.contiguous()
        W = [w.contiguous() for w in weights]
        num_nodes = h.shape[0]
        plan = plan_for(adj, num_nodes)
        per, dh = 128 // bases, out // heads

        # 1. the coefficients, on the native dense kernel as in the forward
        w = C.linear(h, cw, cb).view(num_nodes, heads, bases)
        prod = torch.empty(num_nodes, out, bases, dtype=torch.float32, device=h.device)       # G[n, o] A[n, r(o, b)], node-sized
        d_h = torch.zeros_like(h)
        d_slabs = [[] for _ in W]
        b_all = _split16(h, plan.src32)                                  # the gathered source states, once for every slab
        for s in range(bases * out // 128):
            rows = egc_slab_rows(s, out, heads, bases, h.device)
            Ws = [wt.index_select(0, rows) for wt in W]                 # [128, H]: the slab's rows, in slab order
            # 2. the slab's aggregate A_s [N, 128] (and, for max / min, which edge won each (target, feature))
            agg, arg = _recompute_aggregate(plan, h, Ws, reduce_name)
            # 3. node-side terms: the slab's columns o = s per + j, their heads and coefficient rows
            cols = slice(s * per, (s + 1) * per)
            hd = torch.arange(s * per, (s + 1) * per, device=h.device) // dh
            g_s = g[:, cols].unsqueeze(-1)                                       # [N, per, 1]
            prod[:, cols] = g_s * agg.view(num_nodes, per, bases)
            d_agg = (w.index_select(1, hd) * g_s).reshape(num_nodes, 128)        # dA_s[n, j bases + b] = w[n, hd(j), b] G[n, o]
            # 4. the slab's weight gradients and its part of d h
            d_Ws, d_h = _aggregation_backward(plan, adj, h, Ws, d_agg, reduce_name, arg, d_h, b_all)
            for t, d in enumerate(d_Ws):
                d_slabs[t].append(d)
        # 5. slab order -> the reference's row order
        inv = torch.argsort(torch.cat([egc_slab_rows(s, out, heads, bases, h.device) for s in range(bases * out // 128)]))
        d_W = [torch.cat(ds, dim=0).index_select(0, inv) for ds in d_slabs]
        # 6. the coefficient Linear
        d_w = prod.view(num_nodes, heads, dh, bases).sum(dim=2).reshape(num_nodes, heads * bases)
        d_cw = _mm_t_split(_split16(d_w), _split16(h))
        d_h = d_h + C.linear(d_w.contiguous(), cw.t().contiguous())
        return (None, None, None, None, d_h, d_cw, d_w.sum(dim=0), *d_W)


def egc_forward_with_grad(layer, node_states, adjacency_lists, reduce_name, coeff_weight, coeff_bias, weights):
    return _EgcLayerFunction.apply(layer, adjacency_lists, reduce_name, layer._dims, node_states, coeff_weight, coeff_bias, *weights)


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

        # ---- 3. aggregation + per-type Linear backward (PNA: from the per-edge message gradients of its own backward)
        d_msg = None
        if pna is not None:
            from .aggregation import native_pna_backward

            d_msg = native_pna_backward(msg, plan, pna.delta, agg, arg_max, arg_min, d_agg)
            del msg
        Ws = [w[:, :H].contiguous() for w in W]                              # columns multiplying h_src
        Wg = [w[:, H:].contiguous() for w in W] if use_target else None      # columns multiplying h_tgt
        d_W, d_h = _aggregation_backward(plan, adj, h, Ws, d_agg, reduce_name, arg, torch.zeros_like(h), W_tgt=Wg, d_msg=d_msg)
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
        if reduce_name in ("max", "min"):
            (arg,) = ctx.saved_tensors
            return _route_to_arg(g, arg, plan.num_edges), None, None
        if reduce_name == "mean":
            g = g / _mean_divisor(plan)[:, None]
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
            return None, None, None, _route_to_arg(d_g, arg, plan.num_edges), None      # the plan's edges are the nodes
        x, s, w = ctx.saved_tensors
        gid = plan.tgt32.long()
        d_gn = d_g.index_select(0, gid)                                  # [N, H]: the gradient of each node's graph
        if kind == "mean":
            return None, None, None, d_gn / _mean_divisor(plan).index_select(0, gid)[:, None], None
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
        d_gi, d_gh, d_h = _gru_gate_grads(grad_out.contiguous(), gi, C.linear(h, w_hh, b_hh), h, w_hh)
        d_table = C.segment_reduce(d_gi, plan, N.REDUCE["sum"])             # [G, 3H]: per graph, in node order
        d_g = C.linear(d_table, w_ih.t().contiguous())                      # [G, S]
        d_w_hh = _mm_t_split(_split16(d_gh), _split16(h))
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
# CharUnitEmbedder (strelementrepresentationmodel.py:100-142): the character CNN on the native kernel.  fp32.
# =====================================================================================================================
CHAR_BACKWARD_CHUNK = 4096      # tokens per backward chunk: the backward's workspace is bounded by this, not by B


def _col2im(y: torch.Tensor, Bc: int, L_out: int, w: int, F: int, L_in: int) -> torch.Tensor:
    """d input [Bc, L_in, F] of a convolution from y [Bc L_out, w F] = d out W_tap for every tap: the taps added in tap order."""
    yv = y.view(Bc, L_out, w, F)
    d = torch.zeros(Bc, L_in, F, dtype=torch.float32, device=y.device)
    for tap in range(w):
        d[:, tap:tap + L_out] += yv[:, :, tap]
    return d


def _char_cnn_backward(d_out, chars, arg, prepared, shape, w2, w3):
    """Gradients of (W1, b1, W2, b2, W3) from d_out [B, D] fp32, in chunks of CHAR_BACKWARD_CHUNK tokens whose results are added in
    chunk order.  Per chunk: the kernel's materialise mode gives a1 and a2; d_out goes to its winning positions; dW3 and dW2 are split
    fp16 library GEMMs over the im2col of a2 and a1; d a2 and d a1 are native ``linear`` products followed by a col2im that adds the taps
    in a fixed order; dW1 is the table gradient of an embedding bag over the (token, position) rows.  No float atomics."""
    from .embeddings import native_char_cnn_materialise, native_embedding_bag_backward

    V, F1, k1, F2, k2, D, k3 = shape
    B, L = chars.shape
    L1, L2 = L - k1 + 1, L - k1 - k2 + 2
    L3 = L2 - k3 + 1
    dev = d_out.device
    f32 = dict(dtype=torch.float32, device=dev)
    d_t1, d_b1 = torch.zeros(V * k1, F1, **f32), torch.zeros(F1, **f32)
    d_w2, d_b2, d_w3 = torch.zeros(F2, F1 * k2, **f32), torch.zeros(F2, **f32), torch.zeros(D, F2 * k3, **f32)
    w3cat = w3.detach().permute(2, 1, 0).reshape(k3 * F2, D).contiguous()      # [tap F2 + k, d] = W3[d, k, tap]
    w2cat = w2.detach().permute(2, 1, 0).reshape(k2 * F1, F2).contiguous()
    taps = torch.arange(k1, device=dev)
    for c0 in range(0, B, CHAR_BACKWARD_CHUNK):
        ch = chars[c0:c0 + CHAR_BACKWARD_CHUNK]
        Bc = ch.shape[0]
        a1, a2 = native_char_cnn_materialise(ch, shape, prepared)
        dl3 = torch.zeros(Bc, L3, D, **f32)
        dl3.scatter_(1, arg[c0:c0 + Bc].long().unsqueeze(1), d_out[c0:c0 + Bc].unsqueeze(1))
        dl3 = dl3.view(Bc * L3, D)
        x3 = a2.view(Bc, L2, F2).unfold(1, k3, 1).reshape(Bc * L3, F2 * k3)
        d_w3 += _mm_t_split(_split16(dl3), _split16(x3))
        dl2 = _col2im(C.linear(dl3, w3cat), Bc, L3, k3, F2, L2).mul_(a2.view(Bc, L2, F2) > 0).view(Bc * L2, F2)
        d_b2 += dl2.sum(dim=0)
        x2 = a1.view(Bc, L1, F1).unfold(1, k2, 1).reshape(Bc * L2, F1 * k2)
        d_w2 += _mm_t_split(_split16(dl2), _split16(x2))
        dl1 = _col2im(C.linear(dl2, w2cat), Bc, L2, k2, F1, L1).mul_(a1.view(Bc, L1, F1) > 0).view(Bc * L1, F1)
        d_b1 += dl1.sum(dim=0)
        valid = (ch >= 0) & (ch < V)        # the kernel read an out-of-range id as character 0: so does its gradient
        ids = (torch.where(valid, ch, torch.zeros_like(ch)).unfold(1, k1, 1) * k1 + taps).reshape(Bc * L1, k1)
        d_t1 += native_embedding_bag_backward(dl1, ids, None, "sum", V * k1)
    d_w1 = d_t1.view(V, k1, F1).permute(2, 0, 1).contiguous()
    return d_w1, d_b1, d_w2.view(F2, F1, k2), d_b2, d_w3.view(D, F2, k3)


class _CharCnnFn(torch.autograd.Function):
    """out [B, D] fp32 from chars [B, L] and the five parameters; saves the ids and the [B, D] uint8 winning positions only."""

    @staticmethod
    def forward(ctx, chars, shape, prepared, status, w1, b1, w2, b2, w3):
        from .embeddings import native_char_cnn

        out, arg = native_char_cnn(chars, shape, prepared, want_arg=True, status=status)
        ctx.save_for_backward(chars, arg, w2, w3)
        ctx.shape, ctx.prepared = shape, prepared
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        chars, arg, w2, w3 = ctx.saved_tensors
        grads = _char_cnn_backward(d_out.contiguous().float(), chars, arg, ctx.prepared, ctx.shape, w2, w3)
        return (None, None, None, None) + grads


def char_cnn_with_grad(chars, shape, prepared, status, w1, b1, w2, b2, w3):
    return _CharCnnFn.apply(N.require_cuda(chars, "chars", torch.int64), shape, prepared, status, w1, b1, w2, b2, w3)


# =====================================================================================================================
# LinearFeatureEmbedder (linearmapembedding.py:13-29): act(x W^T) on the native feature-embedding kernel.  fp32.
# =====================================================================================================================
class _FeatureEmbedFn(torch.autograd.Function):
    """out [N, D] from x [N, F] and W [D, F].  act' is read from what torch's own backward reads, so nothing is recomputed: the output
    for ReLU and Tanh (already kept as the result), the pre-activation for GELU (one more [N, D] fp32 write in the same launch, cheaper
    than re-running the GEMM, which reads x again); None needs neither.  Backward: d pre on one native pointwise pass, dW = d pre^T x as
    split fp16 library GEMMs (K = N), dx on the native dense kernel only when x requires a gradient."""

    @staticmethod
    def forward(ctx, x, weight, prepared, act, status):
        from .embeddings import native_feature_embed

        out, _, pre = native_feature_embed(x.detach(), prepared, weight.shape[0], act, want_pre=act == N.ACT_GELU, status=status)
        ctx.act = act
        ctx.save_for_backward(x, weight, pre if act == N.ACT_GELU else (None if act == N.ACT_NONE else out))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        from .embeddings import native_activation_grad

        x, weight, saved = ctx.saved_tensors
        g = g.contiguous().float()
        d_pre = g if ctx.act == N.ACT_NONE else native_activation_grad(ctx.act, g, saved)
        d_w = _mm_t_split(_split16(d_pre), _split16(x.detach())) if ctx.needs_input_grad[1] else None
        d_x = C.linear(d_pre, weight.detach().t().contiguous()) if ctx.needs_input_grad[0] else None
        return d_x, d_w, None, None, None


def feature_embed_with_grad(x, weight, prepared, act, status=None):
    return _FeatureEmbedFn.apply(x, weight, prepared, act, status)


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


# =====================================================================================================================
# VarMisuse candidate selection (varmisuse.py:76-91): the per-slot log-softmax of the candidate scores and the mean NLL of the correct
# candidates, on the native kernels.  fp32 states.
# =====================================================================================================================
class _VarMisuseFn(torch.autograd.Function):
    """loss [] from h [N, H] and the score weight [1, 2H]; backward: d h and d w on the native backward kernels (the softmax re-computed
    from the saved [K] scores and [J] logsumexps).  ``ops``: ``heads.varmisuse_inputs``."""

    @staticmethod
    def forward(ctx, ops, hits, h, weight):
        from .heads import native_varmisuse

        loss, score, lse, _ = native_varmisuse(*ops, hits=hits)
        ctx.ops = ops
        ctx.save_for_backward(score, lse)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        from .heads import native_varmisuse_backward

        score, lse = ctx.saved_tensors
        d_h, d_w = native_varmisuse_backward(*ctx.ops, score, lse, g.contiguous().float())
        return None, None, d_h, d_w.view(1, -1)


def varmisuse_with_grad(ops, hits, node_states, weight):
    return _VarMisuseFn.apply(ops, hits, node_states, weight)


# =====================================================================================================================
# Classification heads (graph2class.py:63-102, ppi.py:13-62): the Linear and its cross-entropy or BCE loss on the native kernel.  fp32.
# =====================================================================================================================
class _ClassifyFn(torch.autograd.Function):
    """loss [] from h [N, H], W [C, H] and b [C]; backward: d logits from one launch that recomputes the logits (from the saved [R] lse
    and valid-row count for CE), then ``heads.classify_input_grads``.  ``ops``: ``heads.ClassifyOps``."""

    @staticmethod
    def forward(ctx, ops, hits, metrics, h, weight, bias):
        from .heads import native_classify

        loss, lse, _, valid, _, _, safe_idx = native_classify(ops, weight.shape[0], hits=hits, metrics=metrics)
        ctx.ops, ctx.safe_idx = ops, safe_idx
        ctx.save_for_backward(weight, lse, valid)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        from .heads import classify_input_grads, native_classify_backward

        weight, lse, valid = ctx.saved_tensors
        d_logits = native_classify_backward(ctx.ops, weight.shape[0], lse, valid, g.contiguous().float())
        d_h, d_w, d_b = classify_input_grads(ctx.ops, ctx.safe_idx, weight, d_logits, *ctx.needs_input_grad[3:6])
        return None, None, None, d_h, d_w, d_b


def classify_with_grad(ops, hits, metrics, node_states, weight, bias):
    return _ClassifyFn.apply(ops, hits, metrics, node_states, weight, bias)


class _ClassifyLogitsFn(torch.autograd.Function):
    """logits [R, C] (Graph2ClassModule._logits) with the head's backward for an upstream d logits."""

    @staticmethod
    def forward(ctx, ops, h, weight, bias):
        from .heads import native_classify

        _, _, _, _, _, logits, safe_idx = native_classify(ops, weight.shape[0], want_logits=True)
        ctx.ops, ctx.safe_idx = ops, safe_idx
        ctx.save_for_backward(weight)
        return logits

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        from .heads import classify_input_grads

        (weight,) = ctx.saved_tensors
        d_h, d_w, d_b = classify_input_grads(ctx.ops, ctx.safe_idx, weight, g.contiguous().float(), *ctx.needs_input_grad[1:4])
        return None, d_h, d_w, d_b


def classify_logits_with_grad(ops, node_states, weight, bias):
    return _ClassifyLogitsFn.apply(ops, node_states, weight, bias)
