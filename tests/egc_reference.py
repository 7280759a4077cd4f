"""Float64 restatement of ``EGCMessagePassingLayer`` (egcmessagepassing.py:54-91) with an error bound for every output element,
and a bf16 emulation of the reference under autocast.  Built on ``fused_reference`` (messages, aggregate, check_bound).

Notation: w = h Wc^T + bc [N, heads * bases], A = the aggregate of the [E, bases * out] messages, and
out[n, o] = sum_b w[n, hd * bases + b] A[n, (hd * bases + b) * dh + c] for o = hd * dh + c.

fp32 path.  The kernel's aggregate A~ is within ``fused_reference.aggregate``'s bound err_A of A (3xFP16 messages, fp32 reduction).
The coefficients come from the native dense kernel (3xTF32: fp32 operands to ~2^-21, fp32 accumulation over K):
|w~ - w| <= err_w = (2 K + 16) u (|h| |Wc|^T + |bc|).  The combination rounds each product and adds them in base order, so

    |out~ - out| <= sum_b (|w_b| err_A_b + |A_b| err_w_b + err_A_b err_w_b) + (bases + 1) u sum_b (|w_b| + err_w_b)(|A_b| + err_A_b).

Targets without in-edges have A = 0 with a zero bound: their output must be exactly 0.

bf16 path (autocast).  The states are bf16; the coefficient Linear rounds its weight and bias to bf16, accumulates in fp32 and rounds
its output to bf16; the aggregate is the fp32 reduction of bf16 messages, rounded back to bf16 (``_aggregate_messages`` casts to the
message dtype); each product bf16(A) bf16(w) is rounded to bf16; the sum over the bases is taken in fp32 and rounded to bf16 once.
``emulate_bf16`` does exactly that with float64 sums rounded where autocast rounds.  ``bf16_kernel_reference`` states the same
arithmetic in the kernel's order with a per-element bound: an fp32 accumulation (message, reduction, coefficient Linear) that lands
within its error of a bf16 rounding midpoint may round either way, which moves that value by one bf16 ulp and is carried through the
products and the sum; everywhere else the bound is 0 and the kernel must match exactly.
"""
from typing import Sequence

import torch

import fused_reference as R
from helpers import split_f16

U = R.U


def rel_l2(x: torch.Tensor, ref: torch.Tensor) -> float:
    x, ref = x.detach().cpu().double(), ref.detach().cpu().double()
    return float((x - ref).norm() / ref.norm().clamp(min=1e-300))


def slab_rows(s: int, out: int, heads: int, bases: int) -> torch.Tensor:
    """Reference rows of ``bases[t].weight`` in slab s (DESIGN.md §3.14): position p = j bases + b <- row ((o // dh) bases + b) dh + o % dh,
    o = s 128 / bases + j."""
    p = torch.arange(128)
    o = s * (128 // bases) + p // bases
    dh = out // heads
    return ((o // dh) * bases + p % bases) * dh + o % dh


def _bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).to(torch.bfloat16).double()


def _combine(A: torch.Tensor, w: torch.Tensor, heads: int, bases: int) -> torch.Tensor:
    """[N, bases * out] (reference row order) x [N, heads * bases] -> the per-base products [N, heads, bases, dh]."""
    n = A.shape[0]
    return A.view(n, heads, bases, -1) * w.view(n, heads, bases, 1)


def forward_torch(h, adj, weights: Sequence[torch.Tensor], cw, cb, reduce: str, heads: int, bases: int) -> torch.Tensor:
    """The layer in the inputs' dtype with differentiable torch ops (float64 inputs: the restatement autograd differentiates)."""
    n = h.shape[0]
    out_dim = weights[0].shape[0] // bases
    w = h @ cw.T + cb
    m = torch.cat([h[s] @ W.T for (s, _t), W in zip(adj, weights)])
    tgt = torch.cat([t for _s, t in adj])
    zeros = torch.zeros(n, m.shape[1], dtype=h.dtype)
    if reduce in ("max", "min"):
        A = zeros.scatter_reduce(0, tgt[:, None].expand_as(m), m, "amax" if reduce == "max" else "amin", include_self=False)
    else:
        A = zeros.index_add(0, tgt, m)
        if reduce == "mean":
            cnt = torch.zeros(n, dtype=h.dtype).index_add_(0, tgt, torch.ones(tgt.shape[0], dtype=h.dtype))
            A = A / cnt.clamp(min=1)[:, None]
    return _combine(A, w, heads, bases).sum(2).reshape(n, out_dim)


def forward64(h, adj, weights: Sequence[torch.Tensor], cw, cb, reduce: str, heads: int, bases: int):
    """-> (out [N, out] float64, bound [N, out] float64) for fp32 states on the fused path."""
    n, K = h.shape
    out_dim = weights[0].shape[0] // bases
    h64 = h.double()
    w = h64 @ cw.double().T + cb.double()
    err_w = (2 * K + 16) * U * (h64.abs() @ cw.double().abs().T + cb.double().abs())
    tgt, m, err = R.messages(h, adj, weights, False, False)
    A, err_A, _ = R.aggregate(tgt, m, err, n, reduce, False)
    ref = _combine(A, w, heads, bases).sum(2).reshape(n, out_dim)
    Aa, eA = A.abs().view(n, heads, bases, -1), err_A.view(n, heads, bases, -1)
    wa, ew = w.abs().view(n, heads, bases, 1), err_w.view(n, heads, bases, 1)
    bnd = (wa * eA + Aa * ew + eA * ew).sum(2) + (bases + 1) * U * ((wa + ew) * (Aa + eA)).sum(2)
    return ref, bnd.reshape(n, out_dim)


def emulate_f32(h, adj, weights, cw, cb, reduce: str, heads: int, bases: int, correction: bool = True, mean_division: bool = True):
    """The fp32 path as the kernel computes it, in float32 arithmetic: 3xFP16 messages (without the two correction products if
    ``correction`` is False -- a mutant for the bound's teeth), the sequential fp32 reduction, the mean division (dropped if
    ``mean_division`` is False), the products rounded to fp32 and added in base order.  For the CPU checks of the bound."""
    n = h.shape[0]
    out_dim = weights[0].shape[0] // bases

    def split(x):
        hi, lo = split_f16(x)
        return hi.float(), lo.float()

    hh, hl = split(h.float())
    tgts, msgs = [], []
    for (s, t), W in zip(adj, weights):
        wh, wl = split(W.float())
        xh, xl = hh[s].double(), hl[s].double()
        m = xh @ wh.double().T
        if correction:
            m = m + (xh @ wl.double().T + xl @ wh.double().T) / 2048.0
        msgs.append(m.float())
        tgts.append(t)
    tgt = torch.cat(tgts)
    m32 = torch.cat(msgs) if msgs else torch.zeros(0, weights[0].shape[0])
    cnt = torch.zeros(n).index_add_(0, tgt, torch.ones(tgt.shape[0]))
    if reduce in ("max", "min"):
        init = float("-inf") if reduce == "max" else float("inf")
        A = torch.full((n, m32.shape[1]), init).scatter_reduce_(0, tgt[:, None].expand_as(m32), m32, "amax" if reduce == "max" else "amin")
        A = torch.where((cnt == 0)[:, None], torch.zeros_like(A), A)
    else:
        A = torch.from_numpy(R._seq_sum_f32(tgt, m32.numpy(), n))
        if reduce == "mean" and mean_division:
            A = A / cnt.clamp(min=1)[:, None]
    w = (h.double() @ cw.double().T + cb.double()).float()
    p = _combine(A, w, heads, bases)
    s = p[:, :, 0]
    for b in range(1, bases):
        s = s + p[:, :, b]
    return s.reshape(n, out_dim).double()


def emulate_bf16(h, adj, weights, cw, cb, reduce: str, heads: int, bases: int) -> torch.Tensor:
    """The reference under autocast bf16 (see the module docstring), float64 sums rounded where autocast rounds -> [N, out] float64
    holding bf16 values."""
    n = h.shape[0]
    out_dim = weights[0].shape[0] // bases
    hb = _bf16(h)
    w = _bf16(hb @ _bf16(cw).T + _bf16(cb))
    tgt, m, err = R.messages(hb.float(), adj, weights, False, True)
    A, _, _ = R.aggregate(tgt, m, torch.zeros_like(err), n, reduce, True)
    p = _bf16(_combine(A, w, heads, bases))
    return _bf16(p.sum(2).reshape(n, out_dim))


def _bf16_window(x: torch.Tensor, e: torch.Tensor):
    """-> (bf16(x), how far another bf16 rounding of a value within e of x lies from it): 0 unless [x - e, x + e] holds a midpoint."""
    b = _bf16(x)
    return b, torch.where(e > 0, torch.maximum(_bf16(x + e) - b, b - _bf16(x - e)), torch.zeros_like(b))


def bf16_kernel_reference(h, adj, weights, cw, cb, reduce: str, heads: int, bases: int, mutant: str = None):
    """The fused bf16 path element by element -> (ref [N, out], bound [N, out]) float64; ref holds bf16 values.

    Nominal values: the coefficients bf16(fp32 sum of bf16 products + bf16 bias); the aggregate of ``fused_reference.aggregate``
    before its output rounding, then rounded to bf16; each product rounded to bf16; their fp32 sum in base order (the kernel's
    order) rounded to bf16.  The bound follows the only freedoms the arithmetic leaves: an fp32 accumulation (message, reduction,
    coefficient Linear) that lands within its error of a bf16 midpoint may round either way -- one bf16 ulp of that value, carried
    through the products and the sum.  Elsewhere the bound is 0 and the kernel must match exactly.  ``mutant``: ``"no_round_ap"``
    leaves A and the products unrounded, ``"no_round_coef"`` the coefficients (kernels that drop those roundings must fail)."""
    n, K = h.shape
    out_dim = weights[0].shape[0] // bases
    hb = _bf16(h)
    cwb, cbb = _bf16(cw), _bf16(cb)
    w_exact = hb @ cwb.T + cbb
    e_w = (2 * K + 16) * U * (hb.abs() @ cwb.abs().T + cbb.abs())
    w, err_w = _bf16_window(w_exact, e_w)
    if mutant == "no_round_coef":
        w, err_w = w_exact.to(torch.float32).double(), e_w
    tgt, m, err = R.messages(hb.float(), adj, weights, False, True)
    pre, bnd, _ = R.aggregate(tgt, m, err, n, reduce, True, round_bf16=False)
    A, err_A = _bf16_window(pre, bnd)
    if mutant == "no_round_ap":
        A, err_A = pre, bnd
    Av, eA = A.view(n, heads, bases, -1), err_A.view(n, heads, bases, -1)
    wv, ew = w.view(n, heads, bases, 1), err_w.view(n, heads, bases, 1)
    exact = Av * wv
    e_p = Av.abs() * ew + wv.abs() * eA + eA * ew
    if mutant == "no_round_ap":
        p, err_p = exact.to(torch.float32).double(), e_p + U * exact.abs()
    else:
        p, err_p = _bf16_window(exact, e_p)
    s = p[:, :, 0].to(torch.float32)
    for b in range(1, bases):
        s = s + p[:, :, b].to(torch.float32)
    s = s.double()
    spread = err_p.sum(2)
    e_s = torch.where(spread > 0, spread + (bases + 1) * U * (p.abs() + err_p).sum(2), torch.zeros_like(spread))
    ref, bound = _bf16_window(s, e_s)
    return ref.reshape(n, out_dim), bound.reshape(n, out_dim)


def params_of(sd, num_types: int):
    """(bases weights, coefficient weight, coefficient bias) from a state_dict with the reference's keys."""
    p = "_EGCMessagePassingLayer__"
    return [sd[f"{p}bases.{t}.weight"] for t in range(num_types)], sd[p + "weight_coeffs.weight"], sd[p + "weight_coeffs.bias"]


def n2_bars(out: torch.Tensor, autocast_ref: torch.Tensor, fp32_ref: torch.Tensor):
    """DESIGN.md §4, N2: rel. L2 <= 1e-2 against the reference's autocast output, and at least as close to the fp32 result as the
    reference's autocast path is (mean error <= 1.1x, fraction within 1e-2 >= the reference's - 0.002)."""
    out, ac, f = (x.detach().cpu().double() for x in (out, autocast_ref, fp32_ref))
    err, err_ref = (out - f).abs(), (ac - f).abs()
    return {"rel_l2": rel_l2(out, ac) <= 1e-2, "mean": float(err.mean()) <= 1.1 * float(err_ref.mean()),
            "within": float((err <= 1e-2).double().mean()) >= float((err_ref <= 1e-2).double().mean()) - 0.002}
