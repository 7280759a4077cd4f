"""Float64 references of the fp32 layer backward passes (``ptgnn_b200/autograd.py``), with an error bound for every element of
each native stage, and float64 restatements of the gated and Mlp layers for end-to-end gradients.

Stages and their bounds (u = 2^-24):

* ``gather_split`` (csrc/gru_grad.cu): out row r = split(x[index[r]] * s), hi = fp16(v), lo = fp16((v - hi) * 2048), v = x * s
  in fp32, round to nearest even.  Emulated bit for bit on the CPU (IEEE fp32 products, the CPU's RNE fp32 -> fp16).

* ``gru_gate_grads`` (csrc/gru_grad.cu): the GRUCell gate derivatives from the fp32 pre-activations.  The bound follows each fp32
  operation of the kernel: a sum, product or difference rounds to u of its magnitude (an fma contraction rounds less, so the
  bound holds either way); expf and tanhf are within 2 ulp = 4u relative (CUDA C Programming Guide, single-precision
  functions); sigmoid = 1 / (1 + expf(-a)) then errs by 4u (1 - r) + 2u <= 6u of r (the add and the IEEE division), and a
  rounding of its argument moves it by r (1 - r) of that.  tanh(c) errs by 4u |n| plus (1 - n^2) times its argument's error.
  Errors propagate to first order with the local slope, widened by ``SLACK`` for the dropped second-order terms, plus
  ``TINY`` absolute per operation for results below fp32's normal range.  ``GATE_REL`` holds the function constants.

* ``_mm_t_split``: A^T B from the 3xFP16 splits of A [K, M] and B [K, N], each operand first scaled by its power of two s.  The
  split represents a scaled element x to 4u |x| plus 2^-36 absolute (``fused_reference``), the dropped lo*lo product is 4u of
  |a b|, combining the main and correction products costs 2u and the inverse scales are exact.  The three library GEMMs add
  K products in fp32 in some order: gamma_K of the mass.  So |got - ref| <= (C_SPLIT + gamma_K) |A|^T |B| + 2^-36 (|A|^T 1 / s_b
  + 1^T |B| / s_a).

* Transposed aggregation (d h_src = sum over edges u -> v of W_t^T d_agg[v], and the Mlp's target-side term): the forward's
  aggregation on the operands (s d_agg, W^T), with s = ``pow2_scale(d_agg)``; value and bound of ``fused_reference`` (fused
  path) or ``unfused_reference`` (3xTF32 path), divided by s.  The absolute 2^-36 term then scales with amax(d_agg).
"""
import math
from typing import Dict, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F_

import fused_reference as FR
import unfused_reference as UR
from helpers import split_f16

U = FR.U
ABS_F16 = FR.ABS_F16
SLACK = 1.01                        # second-order terms dropped by the first-order propagation below
TINY = 2.0 ** -120                  # per operation: results that leave fp32's normal range
GATE_REL = {"sigmoid": 6 * U, "tanh": 4 * U}
C_SPLIT = (4 + 4 + 4 + 2) * U       # two operand splits, the dropped lo*lo product, the combination of the three products


def pow2_scale(x: torch.Tensor) -> float:
    """The power of two the backward scales x by before a 3xFP16 split: 2^floor(log2(1024 / amax(x)))."""
    amax = max(float(x.abs().max()) if x.numel() else 0.0, 1e-30)
    return 2.0 ** math.floor(math.log2(1024.0 / amax))


# ---- gather_split ------------------------------------------------------------------------------------------------------
def gather_split(x: torch.Tensor, index: Optional[torch.Tensor], scale: Optional[float]):
    """-> (hi, lo) fp16 on the CPU, bit for bit what the kernel writes."""
    v = x.float().cpu()
    if index is not None:
        v = v.index_select(0, index.cpu().long())
    if scale is not None:
        v = v * torch.tensor(scale, dtype=torch.float32)
    return split_f16(v)


def split_value(x: torch.Tensor, scale: float = 1.0, index: Optional[torch.Tensor] = None) -> torch.Tensor:
    """What the 3xFP16 product sees of x: (hi + lo / 2048) / scale in float64, with the split of ``gather_split``."""
    hi, lo = gather_split(x, index, scale if scale != 1.0 else None)
    return (hi.double() + lo.double() / 2048.0) / scale


# ---- gru_gate_grads ----------------------------------------------------------------------------------------------------
def _mul(a, ea, b, eb):
    v = a * b
    e = a.abs() * eb + b.abs() * ea + ea * eb
    return v, e + U * (v.abs() + e) + TINY


def _sub(a, ea, b, eb):
    v = a - b
    e = ea + eb
    return v, e + U * (v.abs() + e) + TINY


def gru_gate_grads(gi: torch.Tensor, gh: torch.Tensor, h: torch.Tensor, g: torch.Tensor):
    """-> {name: (ref, bound)} for d_gi, d_gh and d_h_direct (float64, CPU) from the fp32 inputs."""
    gi, gh, h, g = (t.detach().cpu().double() for t in (gi, gh, h, g))
    H = h.shape[1]
    ir, iz, in_ = gi[:, :H], gi[:, H:2 * H], gi[:, 2 * H:]
    hr, hz, hn = gh[:, :H], gh[:, H:2 * H], gh[:, 2 * H:]
    zero = torch.zeros_like(h)

    def sigmoid(a):
        ea = U * a.abs()                                              # the fp32 sum of the two pre-activations
        s = torch.sigmoid(a)
        return s, SLACK * s * (1 - s) * ea + GATE_REL["sigmoid"] * s + TINY

    r, er = sigmoid(ir + hr)
    z, ez = sigmoid(iz + hz)
    rhn, erhn = _mul(r, er, hn, zero)
    c = in_ + rhn
    ec = erhn + U * (c.abs() + erhn)
    n = torch.tanh(c)
    en = SLACK * (1 - n * n) * ec + GATE_REL["tanh"] * n.abs() + TINY
    one = torch.ones_like(h)
    omz, eomz = _sub(one, zero, z, ez)
    omr, eomr = _sub(one, zero, r, er)
    nn2, enn2 = _mul(n, en, n, en)
    omn, eomn = _sub(one, zero, nn2, enn2)
    dn, edn = _mul(*_mul(g, zero, omz, eomz), omn, eomn)
    hmn, ehmn = _sub(h, zero, n, en)
    dz, edz = _mul(*_mul(*_mul(g, zero, hmn, ehmn), z, ez), omz, eomz)
    dr, edr = _mul(*_mul(*_mul(dn, edn, hn, zero), r, er), omr, eomr)
    dnr, ednr = _mul(dn, edn, r, er)
    dh, edh = _mul(g, zero, z, ez)
    return {"d_gi": (torch.cat([dr, dz, dn], 1), SLACK * torch.cat([edr, edz, edn], 1)),
            "d_gh": (torch.cat([dr, dz, dnr], 1), SLACK * torch.cat([edr, edz, ednr], 1)),
            "d_h": (dh, SLACK * edh)}


# ---- _mm_t_split -------------------------------------------------------------------------------------------------------
def mm_t_split(a: torch.Tensor, b: torch.Tensor, sa: Optional[float] = None, sb: Optional[float] = None):
    """-> (ref [M, N], bound [M, N]) for A^T B, A [K, M], B [K, N] fp32 (float64 on the CPU).  sa, sb: the operands' scales when they
    were taken over larger tensors than these rows (default: ``pow2_scale`` of A and B)."""
    a64, b64 = a.detach().cpu().double(), b.detach().cpu().double()
    K = a64.shape[0]
    ref = a64.t() @ b64
    if K == 0:
        return ref, torch.zeros_like(ref)
    sa = pow2_scale(a64) if sa is None else sa
    sb = pow2_scale(b64) if sb is None else sb
    aa, ab = a64.abs(), b64.abs()
    bound = (C_SPLIT + UR.gamma(K)) * (aa.t() @ ab) + ABS_F16 * (aa.sum(0)[:, None] / sb + ab.sum(0)[None, :] / sa)
    return ref, SLACK * bound


# ---- transposed aggregation --------------------------------------------------------------------------------------------
def transposed_aggregate(x: torch.Tensor, adj, weights: Sequence[torch.Tensor], num_nodes: int, fused: bool, scaled: bool = True):
    """-> (ref, bound) of d[u] = sum over edges (u -> v, type t) of W_t^T x[v] (x = d_agg [N, D], W_t [D, H]) on the fused (3xFP16) or
    unfused (3xTF32) aggregation, with x scaled by ``pow2_scale(x)`` first (``scaled``) as the backward does."""
    x64 = x.detach().cpu().double()
    s = pow2_scale(x64) if scaled else 1.0
    rev = [(t.cpu(), s_.cpu()) for s_, t in adj]
    wt = [w.detach().cpu().double().t().contiguous() for w in weights]
    xs = x64 * s
    if fused:
        tgt, m, err = FR.messages(xs, rev, wt, False, False)
    else:
        tgt, m, err = UR.fp32_messages(xs.float(), rev, [w.float() for w in wt], False)
        err = err + U * m.abs()                                       # the unfused messages are stored as fp32 before the reduce
    ref, bnd, _ = FR.aggregate(tgt, m, err, num_nodes, "sum", False)
    return ref / s, bnd / s


def emulate_transposed_aggregate(x: torch.Tensor, adj, weights: Sequence[torch.Tensor], num_nodes: int, scale: float) -> torch.Tensor:
    """The fused kernel's 3xFP16 arithmetic on the CPU (float64 sums): x * scale and the weights split into (hi, lo') as the kernels
    do, hi*hi + 2^-11 (hi*lo' + lo'*hi) per message, the sum divided by scale.  ``scale`` 1 is the unscaled split."""
    xh, xl = (v.double() for v in gather_split(x, None, scale if scale != 1.0 else None))
    out = torch.zeros(num_nodes, weights[0].shape[1], dtype=torch.float64)
    for (src, tgt), w in zip(adj, weights):
        wh, wl = (v.double() for v in gather_split(w.detach().float().t().contiguous(), None, None))
        m = xh[tgt] @ wh.t() + (xh[tgt] @ wl.t() + xl[tgt] @ wh.t()) / 2048.0
        out.index_add_(0, src, m)
    return out / scale


# ---- float64 layer restatements ----------------------------------------------------------------------------------------
def _reduce(m: torch.Tensor, tgt: torch.Tensor, n: int, reduce: str) -> torch.Tensor:
    zeros = torch.zeros(n, m.shape[1], dtype=m.dtype)
    if reduce in ("max", "min"):
        return zeros.scatter_reduce(0, tgt[:, None].expand_as(m), m, "amax" if reduce == "max" else "amin", include_self=False)
    agg = zeros.index_add(0, tgt, m)
    if reduce == "mean":
        cnt = torch.zeros(n, dtype=m.dtype).index_add_(0, tgt, torch.ones(tgt.shape[0], dtype=m.dtype))
        agg = agg / cnt.clamp(min=1)[:, None]
    return agg


def messages64(h: torch.Tensor, adj, weights: Sequence[torch.Tensor], use_target: bool) -> torch.Tensor:
    parts = [(torch.cat([h[s], h[t]], 1) if use_target else h[s]) @ w.t() for (s, t), w in zip(adj, weights)]
    return torch.cat(parts) if parts else torch.zeros(0, weights[0].shape[0], dtype=h.dtype)


def gated_forward64(h, adj, p: Dict[str, torch.Tensor], reduce: str):
    """GatedMessagePassingLayer (gather, per-type Linear, scatter, GRUCell) in float64; p: the layer's parameters by name."""
    pre = "_GatedMessagePassingLayer__"
    W = [p[f"{pre}edge_message_transformation_layers.{t}.weight"] for t in range(len(adj))]
    tgt = torch.cat([t for _s, t in adj])
    agg = _reduce(messages64(h, adj, W, False), tgt, h.shape[0], reduce)
    gi = agg @ p[pre + "state_update.weight_ih"].t() + p[pre + "state_update.bias_ih"]
    gh = h @ p[pre + "state_update.weight_hh"].t() + p[pre + "state_update.bias_hh"]
    ir, iz, in_ = gi.chunk(3, 1)
    hr, hz, hn = gh.chunk(3, 1)
    r, z = torch.sigmoid(ir + hr), torch.sigmoid(iz + hz)
    n = torch.tanh(in_ + r * hn)
    return (1 - z) * n + z * h, agg


def mlp_forward64(layer, h, adj, p: Dict[str, torch.Tensor], reduce: str, use_target: bool):
    """MlpMessagePassingLayer with the default message MLP (one bias-free Linear per type): messages, scatter, message activation,
    LayerNorm, dense layer and its activation, in float64; the activation modules are the layer's own."""
    pre = "_MlpMessagePassingLayer__"
    W = [p[f"{pre}edge_message_transformation_layers.{t}._MLP__mlp_modules.1.weight"] for t in range(len(adj))]
    tgt = torch.cat([t for _s, t in adj])
    agg = _reduce(messages64(h, adj, W, use_target), tgt, h.shape[0], reduce)
    act = getattr(layer, pre + "message_activation")
    x = agg if act is None else act(agg)
    for i, m in enumerate(getattr(layer, pre + "state_update")):
        if isinstance(m, torch.nn.LayerNorm):
            x = F_.layer_norm(x, m.normalized_shape, p[f"{pre}state_update.{i}.weight"], p[f"{pre}state_update.{i}.bias"], m.eps)
        elif isinstance(m, torch.nn.Linear):
            x = F_.linear(x, p[f"{pre}state_update.{i}.weight"], p.get(f"{pre}state_update.{i}.bias"))
        elif not isinstance(m, torch.nn.Dropout):
            x = m(x)
    return x, agg


def leaves64(layer) -> Dict[str, torch.Tensor]:
    return {k: v.detach().cpu().double().requires_grad_(True) for k, v in layer.named_parameters()}


# ---- graphs ------------------------------------------------------------------------------------------------------------
def dedup(adj):
    """Each (source, target) pair at most once per edge type: no two edges of a type carry the same message."""
    out = []
    for s, t in adj:
        n = int(max(int(s.max()), int(t.max())) + 1) if s.numel() else 1
        key = torch.unique(s * n + t)
        out.append((key // n, key % n))
    return out


def tie_gap(m: torch.Tensor, tgt: torch.Tensor, n: int, reduce: str) -> float:
    """Smallest distance between the winning message of a (target, feature) and its runner-up, over targets with >= 2 edges."""
    if reduce not in ("max", "min") or m.shape[0] == 0:
        return math.inf
    x = (m if reduce == "max" else -m).detach()
    order = torch.argsort(tgt, stable=True)
    ts, xs = tgt[order].numpy(), x[order].numpy()
    starts = np.flatnonzero(np.r_[True, ts[1:] != ts[:-1]])
    best = math.inf
    for a, b in zip(starts, np.r_[starts[1:], ts.shape[0]]):
        if b - a >= 2:
            part = np.sort(xs[a:b], axis=0)
            best = min(best, float((part[-1] - part[-2]).min()))
    return best


def check_scaled(got: torch.Tensor, ref: torch.Tensor, what: str):
    """-> (max|err| / max|ref|, relative L2, max|err|) with no floor on the reference's magnitude."""
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} != {tuple(ref.shape)}"
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite gradient"
    err = (got - ref).abs()
    amax = float(ref.abs().max()) if ref.numel() else 0.0
    if amax == 0.0:
        assert bool((got == 0).all()), f"{what}: the gradient must be exactly 0"
        return 0.0, 0.0, 0.0
    return float(err.max()) / amax, float((got - ref).norm() / ref.norm()), float(err.max())
