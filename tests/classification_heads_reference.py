"""Float64 restatement of the reference's classification heads: ``Graph2ClassModule`` (graph2class.py:63-102: ``CrossEntropyLoss`` of
``Linear(h[supernodes])`` and the argmax accuracy) and ``PPIClassification`` (ppi.py:13-62: BCE-with-logits summed per node and averaged,
TP / FP / FN of ``sigmoid(x) >= 0.5`` and the fp32 metric formulas), their gradients and the error bounds of the native kernel
(ptgnn_b200/csrc/classify.cu).

* ``logits``: float64 ``rows W^T + b`` (bf16: of bf16-rounded rows, weight and bias, then rounded to bf16 as autocast's Linear).
* ``logit_bound``: the feature embedder's 3xFP16 (or bf16) bound of ``rows W^T`` (feature_embedding_reference.bound) plus the fp32
  roundings of the bias add, and with bf16 the rounding of the logit itself.
* ``ce`` / ``bce``: per-row terms, loss, argmax, counts and their bounds: a term moves by at most twice the largest logit error of its row
  (CE) or the sum of its logit errors (BCE), plus a few fp32 ulps of expf / logf / log1pf; the loss adds the fixed-order sums' roundings.
* ``ppi_metrics``: precision, recall and fscore as ppi.py:50-52 computes them in fp32, from integer counts.
"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import feature_embedding_reference as FE  # noqa: E402

IGNORE_INDEX = -100
SUM_DEPTH = 96            # fp32 additions any loss partial goes through (per-thread columns, quad, blocks, rows, CTA and final trees)


def rows_of(h: torch.Tensor, idx) -> torch.Tensor:
    return h if idx is None else h[idx]


def logits(h, idx, w, b, bf16: bool = False) -> torch.Tensor:
    x, w, b = rows_of(h, idx).double(), w.double(), b.double()
    if bf16:
        x, w, b = FE.bf16_round(x), FE.bf16_round(w), FE.bf16_round(b)
    out = x @ w.t() + b
    return FE.bf16_round(out) if bf16 else out


def logit_bound(h, idx, w, b, bf16: bool = False) -> torch.Tensor:
    x = rows_of(h, idx)
    bb = FE.bf16_round(b) if bf16 else b.double()
    pre = FE.bound(x, w, "none", bf16)
    v = logits(h, idx, w, b, bf16).abs()
    out = pre + 2.0 ** -23 * (v + bb.abs()) + 2.0 ** -40
    if bf16:
        out = out + 2.0 ** -8 * (v + out)                 # the rounding of the logit may go the other way
    return out


def ce(z: torch.Tensor, zb: torch.Tensor, target: torch.Tensor):
    """(loss, loss bound, lse [S], argmax [S], hits, valid rows) of nn.CrossEntropyLoss() (mean over non-ignored rows) on logits z
    [S, C] with per-element bounds zb."""
    z = z.double()
    lse = torch.logsumexp(z, dim=1) if z.shape[1] else torch.zeros(0, dtype=torch.float64)
    arg = z.argmax(dim=1) if z.shape[0] else torch.zeros(0, dtype=torch.int64)
    valid = target != IGNORE_INDEX
    n = int(valid.sum())
    if n == 0:
        return float("nan"), 0.0, lse, arg, int((arg == target).sum()), 0
    t = z[valid].gather(1, target[valid].unsqueeze(1)).squeeze(1)
    terms = lse[valid] - t
    rb = 2.0 * zb[valid].max(dim=1).values + 2.0 ** -20 * (lse[valid].abs() + t.abs() + 1.0)
    loss = float(terms.mean())
    bound = float(rb.mean()) + SUM_DEPTH * 2.0 ** -24 * float(terms.abs().mean()) + 2.0 ** -23 * abs(loss)
    return loss, bound, lse, arg, int((arg == target).sum()), n


def ce_grad(z: torch.Tensor, target: torch.Tensor, g: float = 1.0) -> torch.Tensor:
    """d loss / d logits [S, C]."""
    z = z.double()
    valid = target != IGNORE_INDEX
    p = torch.softmax(z, dim=1)
    onehot = torch.zeros_like(p)
    onehot[valid] = torch.nn.functional.one_hot(target[valid], z.shape[1]).double()
    return g * (p - onehot) * valid.unsqueeze(1).double() / max(int(valid.sum()), 1)


def sigmoid_predict(z: torch.Tensor, bf16: bool = False) -> torch.Tensor:
    """torch's ``sigmoid(x) >= 0.5`` for fp32 logits (1 / (1 + exp(-x)) rounded to fp32, or to bf16)."""
    p = (1.0 / (1.0 + torch.exp(-z.double()))).float()
    if bf16:
        p = p.to(torch.bfloat16).float()
    return p >= 0.5


def bce(z: torch.Tensor, zb: torch.Tensor, t: torch.Tensor):
    """(loss, loss bound, tp, fp, fn) of binary_cross_entropy_with_logits(reduction="none").sum(-1).mean() and the counts of the
    float64 decision z >= 0 (equal to torch's where |z| is above the threshold's rounding, see ``threshold_margin``)."""
    z, tf = z.double(), t.double()
    terms = z.clamp(min=0) - z * tf + torch.log1p(torch.exp(-z.abs()))
    R = z.shape[0]
    loss = float(terms.sum(dim=1).mean()) if R else float("nan")
    bound = (float((zb + 2.0 ** -21 * (terms.abs() + 1.0)).sum(dim=1).mean()) + SUM_DEPTH * 2.0 ** -24 * float(terms.sum(dim=1).mean())
             + 2.0 ** -23 * abs(loss)) if R else 0.0
    p = z >= 0
    return loss, bound, int((p & t).sum()), int((p & ~t).sum()), int((~p & t).sum())


def ce_hits_decidable(z: torch.Tensor, zb: torch.Tensor) -> bool:
    """No row has a runner-up logit within the two logits' bounds of its maximum: every argmax is decided by the bounds."""
    if z.shape[1] < 2 or z.shape[0] == 0:
        return True
    top2 = z.topk(2, dim=1)
    bmax = zb.max(dim=1).values
    return bool(((top2.values[:, 0] - top2.values[:, 1]) > 2 * bmax).all())


def bce_counts_decidable(z: torch.Tensor, zb: torch.Tensor, bf16: bool = False) -> bool:
    """No logit lies within its bound (plus the sigmoid's rounding band: 2^-23, or 2^-8 in bf16) of the threshold 0."""
    band = 2.0 ** -7 if bf16 else 2.0 ** -22
    return bool((z.abs() > zb + band).all())


def ppi_metrics(tp: int, fp: int, fn: int):
    """(precision, recall, fscore) as fp32 tensors, exactly as ppi.py:50-52 computes them."""
    tp_, fp_, fn_ = (torch.tensor(float(v), dtype=torch.float32) for v in (tp, fp, fn))
    precision = tp_ / (tp_ + fp_ + 1e-10)
    recall = tp_ / (tp_ + fn_ + 1e-10)
    fscore = 2 * precision * recall / (precision + recall + 1e-10)
    return precision, recall, fscore


def param_grads(h, idx, w, d_logits):
    """(d h [N, H], d W, d b) in float64 for d logits [R, C]."""
    x = rows_of(h, idx).double()
    d_rows = d_logits.double() @ w.double()
    d_h = torch.zeros(h.shape, dtype=torch.float64)
    if idx is None:
        d_h = d_rows
    else:
        d_h.index_add_(0, idx, d_rows)
    return d_h, d_logits.double().t() @ x, d_logits.double().sum(0)


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-300)) if b.numel() else 0.0


def emulate_logits(h, idx, w, b, correction: bool = True) -> torch.Tensor:
    """The kernel's fp32 split products in float64 plus the bias (``correction=False``: the hi products only, a mutant)."""
    return FE.emulate_split(rows_of(h, idx), w, "none", correction) + b.double()


def mutants_exceed(h, idx, w, b) -> dict:
    """{mutant: whether some logit leaves its bound}: a 2^-12 relative weight error, and the kernel without its correction products."""
    ref, zb = logits(h, idx, w, b), logit_bound(h, idx, w, b)
    w_err = w.double() * (1.0 + 2.0 ** -12)
    return {"weight_2^-12": bool(((logits(h, idx, w_err, b) - ref).abs() > zb).any()),
            "no_correction": bool(((emulate_logits(h, idx, w, b, correction=False) - ref).abs() > zb).any())}


def nan_or_close(a: float, b: float, tol: float) -> bool:
    return (math.isnan(a) and math.isnan(b)) or abs(a - b) <= tol
