"""Float64 restatement of the reference's ``CharUnitEmbedder`` (strelementrepresentationmodel.py:128-142) and a per-element error bound
for the native kernel (ptgnn_b200/csrc/char_cnn.cu, DESIGN.md §3.13), derived from the kernel's order of operations.

Bound (fp32 path).  With u = 2^-24 and the absolute-value forward m1 = |b1| + sum |W1| (the gathered terms), m2 = |b2| + conv(|a1|, |W2|),
m3 = conv(|a2|, |W3|) (exact, from the float64 activations):
  e1 = (w1 + 1) u m1                                     b1 and the w1 gathered rows added in fp32
  e2 = conv(e1, |W2|) + c(F1 w2) m2,   e3 = conv(e2, |W3|) + c(F2 w3) m3
  c(K) = 3 2^-22 + (K + 16) 2^-23    the 3xFP16 split (|lo'| rounding 2^-11 of a 2^-11 residual, the dropped lo' lo' term) on both
                                     operands, and the tensor core's fp32 accumulation of K products with a margin for its truncation
and the max moves by at most the largest e3 of the token's positions (|max a - max b| <= max |a - b|).  ReLU does not increase an error.
bf16 path: the weights, biases, a1, the layer-2 output and the output are rounded to bf16 (relative 2^-9 each), so every layer adds
3 2^-9 of its magnitude: e1 = 2 2^-9 m1, e_l = conv(e_{l-1}, |W|) + 3 2^-9 m_l.

The element bounds are worst cases and do not see a precision defect (a kernel without the 3xFP16 correction products, or a bf16
kernel without a bias, stays inside them).  So the tests also hold the whole output to relative-L2 bars that such defects miss:
* fp32: rel. L2 <= FP32_REL_L2 against float64.  ``emulate_split`` (the 3xFP16 products) is at ~1e-7 on the fixtures, the same
  emulation without the correction products at ~3e-4.
* bf16: within BF16_EMU_REL_L2 of ``emulate_bf16`` (float64 sums rounded to bf16 where autocast rounds) and the N2 bars of DESIGN.md
  §4 against the reference's autocast output (``n2_bars``).
"""
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from helpers import split_f16

PRE = "_CharUnitEmbedder__"
FP32_REL_L2 = 1e-5
BF16_EMU_REL_L2 = 2e-3


def rel_l2(x: torch.Tensor, ref: torch.Tensor) -> float:
    x, ref = x.double(), ref.double()
    return float((x - ref).norm() / ref.norm().clamp(min=1e-300))


def params_of(state: Dict[str, np.ndarray], D: int = None):
    """(W1, b1, W2, b2, W3) float tensors from a fixture's ``sd::`` arrays (W3 cut to its first D rows)."""
    g = lambda k: torch.from_numpy(np.asarray(state["sd::" + PRE + k]))
    w3 = g("conv_l3.weight")
    return g("conv_l1.weight"), g("conv_l1.bias"), g("conv_l2.weight"), g("conv_l2.bias"), (w3 if D is None else w3[:D])


def layers(chars: torch.Tensor, w1, b1, w2, b2, w3, dtype=torch.float64) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(a1, a2, l3) of the reference's formulation in ``dtype``: a1 [B, F1, L1], a2 [B, F2, L2] post-ReLU, l3 [B, D, L3]."""
    C = w1.shape[1]
    x = F.one_hot(chars, C).transpose(1, 2).to(dtype)
    a1 = F.relu(F.conv1d(x, w1.to(dtype), b1.to(dtype)))
    a2 = F.relu(F.conv1d(a1, w2.to(dtype), b2.to(dtype)))
    return a1, a2, F.conv1d(a2, w3.to(dtype))


def forward(chars, w1, b1, w2, b2, w3, dtype=torch.float64) -> torch.Tensor:
    return layers(chars, w1, b1, w2, b2, w3, dtype)[2].max(dim=-1).values


def bound(chars, w1, b1, w2, b2, w3, bf16: bool = False) -> torch.Tensor:
    """[B, D] float64: the largest |kernel - exact| the kernel's order allows (module docstring)."""
    C = w1.shape[1]
    d = torch.float64
    a1, a2, l3 = layers(chars, w1, b1, w2, b2, w3)
    x = F.one_hot(chars, C).transpose(1, 2).to(d)
    m1 = F.conv1d(x, w1.abs().to(d), b1.abs().to(d))
    m2 = F.conv1d(a1, w2.abs().to(d), b2.abs().to(d))
    m3 = F.conv1d(a2, w3.abs().to(d))
    if bf16:
        r = 2.0 ** -9
        e1 = 2 * r * m1
        e2 = F.conv1d(e1, w2.abs().to(d)) + 3 * r * m2
        e3 = F.conv1d(e2, w3.abs().to(d)) + 3 * r * m3
    else:
        u = 2.0 ** -24
        c = lambda K: 3 * 2.0 ** -22 + (K + 16) * 2.0 ** -23
        e1 = (w1.shape[2] + 1) * u * m1
        e2 = F.conv1d(e1, w2.abs().to(d)) + c(w2.shape[1] * w2.shape[2]) * m2
        e3 = F.conv1d(e2, w3.abs().to(d)) + c(w3.shape[1] * w3.shape[2]) * m3
    return e3.max(dim=-1).values


def gradients(chars, w1, b1, w2, b2, w3, grad_out, decisions=None) -> Tuple[torch.Tensor, ...]:
    """float64 autograd gradients of (out * grad_out).sum() w.r.t. the five parameters.  ``decisions`` = (a1 > 0 [B, F1, L1], a2 > 0
    [B, F2, L2], arg [B, D]): the ReLU masks and max positions to use instead of float64's own.  A pre-activation within rounding of 0,
    or two positions within rounding of each other, may legitimately go the other way in fp32; with the kernel's decisions the
    comparison measures the arithmetic only."""
    ps = [p.detach().to(torch.float64).requires_grad_(True) for p in (w1, b1, w2, b2, w3)]
    if decisions is None:
        out = forward(chars, *ps)
    else:
        m1, m2, arg = decisions
        x = F.one_hot(chars, w1.shape[1]).transpose(1, 2).to(torch.float64)
        a1 = F.conv1d(x, ps[0], ps[1]) * m1
        a2 = F.conv1d(a1, ps[2], ps[3]) * m2
        out = F.conv1d(a2, ps[4]).gather(-1, arg.long().unsqueeze(-1)).squeeze(-1)
    (out * grad_out.to(torch.float64)).sum().backward()
    return tuple(p.grad for p in ps)


def _rb(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def emulate_bf16(chars, w1, b1, w2, b2, w3, drop_bias: Optional[int] = None) -> torch.Tensor:
    """[B, D] float64 holding bf16 values: weights and biases rounded to bf16, each conv summed exactly and rounded to bf16 where
    autocast's conv1d rounds (a1, the layer-2 output, the output).  ``drop_bias`` = 1 or 2: the mutant without that bias."""
    W1, B1, W2, B2, W3 = (_rb(p.double()) for p in (w1, b1, w2, b2, w3))
    B1 = B1 * 0 if drop_bias == 1 else B1
    B2 = B2 * 0 if drop_bias == 2 else B2
    x = F.one_hot(chars, w1.shape[1]).transpose(1, 2).to(torch.float64)
    a1 = F.relu(_rb(F.conv1d(x, W1, B1)))
    a2 = F.relu(_rb(F.conv1d(a1, W2, B2)))
    return _rb(F.conv1d(a2, W3)).max(dim=-1).values


def _split(x: torch.Tensor):
    hi, lo = split_f16(x)
    return hi.double(), lo.double()


def emulate_split(chars, w1, b1, w2, b2, w3, correction: bool = True) -> torch.Tensor:
    """[B, D] of the kernel's fp32 arithmetic: a1 in fp32, layers 2 and 3 as 3xFP16 products (hi hi + 2^-11 (hi lo' + lo' hi)) of the
    split operands, summed in float64.  ``correction=False``: the mutant with only the hi hi products."""
    x = F.one_hot(chars, w1.shape[1]).transpose(1, 2).to(torch.float32)
    a = F.relu(F.conv1d(x.double(), w1.double(), b1.double()).float())

    def conv(a, w, b):
        ah, al = _split(a)
        wh, wl = _split(w)
        out = F.conv1d(ah, wh)
        if correction:
            out = out + (F.conv1d(ah, wl) + F.conv1d(al, wh)) / 2048.0
        return (out if b is None else out + b.double()[:, None]).float()

    a = F.relu(conv(a, w2, b2))
    return conv(a, w3, None).double().max(dim=-1).values


def n2_bars(out: torch.Tensor, autocast_ref: torch.Tensor, fp32_ref: torch.Tensor) -> Dict[str, bool]:
    """DESIGN.md §4, N2: rel. L2 <= 1e-2 against the reference's autocast output, and at least as close to the fp32 result as the
    reference's autocast path is (mean error <= 1.1x, fraction within 1e-2 >= the reference's - 0.002)."""
    out, ac, f = out.double(), autocast_ref.double(), fp32_ref.double()
    err, err_ref = (out - f).abs(), (ac - f).abs()
    return {"rel_l2": rel_l2(out, ac) <= 1e-2, "mean": float(err.mean()) <= 1.1 * float(err_ref.mean()),
            "within": float((err <= 1e-2).double().mean()) >= float((err_ref <= 1e-2).double().mean()) - 0.002}
