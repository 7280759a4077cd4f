"""Float64 restatement of the reference's ``LinearFeatureEmbedder`` (linearmapembedding.py:13-29): ``act(x W^T)``, its backward, the
per-element error bounds of the native kernel (ptgnn_b200/csrc/feature_embed.cu) and an emulation of that kernel's arithmetic.

* ``forward`` / ``gradients``: float64 (d W = d pre^T x, d x = d pre W, d pre = g act'(pre)).
* ``bound``: |kernel - forward| per element.  fp32 (3xFP16 split): the split leaves 2^-22 |x| |w| per product (dropped lo' lo' term,
  rounding of lo') plus 2^-36 per operand for values below fp16's normal range; the accumulator takes one k16 MMA per 16 columns of
  K = F padded to 16, each adding at most 2 fp32 roundings of sum |x| |w|: (K / 8 + 8) 2^-23 sum |x| |w| in all; |act'| <= 1.13 carries that to the output, and tanhf / erff / the GELU product add a few fp32 ulps.  bf16:
  the same against the float64 result of bf16-rounded inputs, plus the bf16 roundings of the pre-activation and of the output.
* ``emulate_split``: the kernel's split products in float64 (with ``correction=False``: the hi products only, a mutant the bound must
  reject).
"""
import math

import torch

from helpers import split_f16

ACTIVATIONS = ("none", "relu", "tanh", "gelu")
ACT_SLOPE = 1.13          # max |GELU'(x)| (1.129 at x = 2.42); ReLU, Tanh: 1


def act64(pre: torch.Tensor, act: str) -> torch.Tensor:
    if act == "relu":
        return pre.clamp(min=0.0)
    if act == "tanh":
        return torch.tanh(pre)
    if act == "gelu":
        return 0.5 * pre * (1.0 + torch.erf(pre / math.sqrt(2.0)))
    return pre


def act_grad64(pre: torch.Tensor, act: str) -> torch.Tensor:
    if act == "relu":
        return (pre > 0).double()
    if act == "tanh":
        return 1.0 - torch.tanh(pre) ** 2
    if act == "gelu":
        return 0.5 * (1.0 + torch.erf(pre / math.sqrt(2.0))) + pre * torch.exp(-0.5 * pre * pre) / math.sqrt(2.0 * math.pi)
    return torch.ones_like(pre)


def bf16_round(t: torch.Tensor) -> torch.Tensor:
    return t.float().to(torch.bfloat16).double()


def forward(x: torch.Tensor, w: torch.Tensor, act: str, bf16: bool = False) -> torch.Tensor:
    x, w = x.double(), w.double()
    if bf16:
        x, w = bf16_round(x), bf16_round(w)
    return act64(x @ w.t(), act)


def gradients(x: torch.Tensor, w: torch.Tensor, act: str, grad_out: torch.Tensor):
    """(d W, d x) of (act(x W^T) * grad_out).sum() in float64."""
    x, w, g = x.double(), w.double(), grad_out.double()
    d_pre = g * act_grad64(x @ w.t(), act)
    return d_pre.t() @ x, d_pre @ w


def bound(x: torch.Tensor, w: torch.Tensor, act: str, bf16: bool = False) -> torch.Tensor:
    x, w = x.double(), w.double()
    if bf16:
        x, w = bf16_round(x), bf16_round(w)
    K = (x.shape[1] + 15) // 16 * 16
    mag = x.abs() @ w.abs().t()
    pre = x @ w.t()
    b_pre = (K / 8 + 8) * 2.0 ** -23 * mag
    if not bf16:
        b_pre = b_pre + 2.0 ** -22 * mag + 2.0 ** -36 * (x.abs().sum(1, keepdim=True) + w.abs().sum(1).unsqueeze(0))
    else:
        b_pre = b_pre + 2.0 ** -8 * pre.abs()          # the bf16 pre-activation
    y = act64(pre, act)
    b = ACT_SLOPE * b_pre + 2.0 ** -21 * (y.abs() + pre.abs()) + 2.0 ** -40
    if bf16:
        b = b + 2.0 ** -8 * (y.abs() + b)               # the bf16 output
    return b


def _split(t: torch.Tensor):
    hi, lo = split_f16(t)
    return hi.double(), lo.double()


def emulate_split(x: torch.Tensor, w: torch.Tensor, act: str, correction: bool = True) -> torch.Tensor:
    xh, xl = _split(x)
    wh, wl = _split(w)
    pre = xh @ wh.t()
    if correction:
        pre = pre + (xh @ wl.t() + xl @ wh.t()) / 2048.0
    return act64(pre, act)


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp(min=1e-300))
