"""Float64 restatement of the reference's VarMisuse head (implementations/varmisuse/varmisuse.py:58-91), and the per-element error bounds
the native kernels are held to (DESIGN.md §3.16).

* ``varmisuse(h, cand, slot_of, slot_nodes, correct, w)`` -> dict of loss [], score [K], lse [J], argmax [J] (first maximum; K for a slot
  without candidates) and hits (slots whose argmax is their correct candidate), all float64 / int64.
* ``varmisuse_gradients(...)`` -> (d h [N, H], d w [1, 2H]) of ``g * loss`` by autograd in float64.
* ``score_bound`` / ``lse_bound`` / ``loss_bound``: |fp32 kernel - float64| per element.  A score is a dot product of length 2H, computed
  as two fmaf chains of H / 4 terms per lane and a 32-lane butterfly: |err| <= gamma_{2H + 2} sum_i |w_i x_i| with gamma_n = n u / (1 - n u),
  u = 2^-24.  A slot's logsumexp adds its scores' error to the relative error of the online sum of exponentials, (c + 8) u for c
  candidates (expf and logf are within 2 ulp).  The loss is a mean of S terms score - lse summed in fp32.
* ``bf16=True`` rounds h and w to bf16 first, as the kernel does for bf16 states.
"""
import torch

U = 2.0 ** -24


def _gamma(n):
    return n * U / (1 - n * U)


def _bf16(t):
    return t.to(torch.bfloat16).to(torch.float64)


def _operands(h, w, bf16):
    h, w = h.to(torch.float64), w.reshape(-1).to(torch.float64)
    return (_bf16(h), _bf16(w)) if bf16 else (h, w)


def _loss(h, cand, slot_of, slot_nodes, correct, w):
    H = h.shape[1]
    J = slot_nodes.shape[0]
    score = h[cand] @ w[:H] + h[slot_nodes][slot_of] @ w[H:]
    mx = torch.full((J,), -torch.inf, dtype=score.dtype).scatter_reduce(0, slot_of, score.detach(), "amax", include_self=True)
    shift = torch.where(torch.isinf(mx), torch.zeros_like(mx), mx)
    total = torch.zeros(J, dtype=score.dtype).scatter_add(0, slot_of, (score - shift[slot_of]).exp())
    lse = total.log() + shift
    loss = -(score[correct] - lse[slot_of[correct]]).mean()
    return loss, score, lse


def varmisuse(h, cand, slot_of, slot_nodes, correct, w, bf16=False):
    h, w = _operands(h, w, bf16)
    loss, score, lse = _loss(h, cand, slot_of, slot_nodes, correct, w)
    K, J = cand.shape[0], slot_nodes.shape[0]
    arg = torch.full((J,), K, dtype=torch.int64)
    for j in range(J):
        ks = (slot_of == j).nonzero().flatten()
        if ks.numel():
            arg[j] = ks[int(torch.argmax(score[ks]))]           # torch.argmax returns the first maximum
    hits = int((arg == correct).sum()) if correct.shape[0] == J else 0
    return dict(loss=loss, score=score, lse=lse, argmax=arg, hits=hits)


def varmisuse_gradients(h, cand, slot_of, slot_nodes, correct, w, g=1.0):
    hd = h.to(torch.float64).clone().requires_grad_(True)
    wd = w.reshape(1, -1).to(torch.float64).clone().requires_grad_(True)
    loss, _, _ = _loss(hd, cand, slot_of, slot_nodes, correct, wd.reshape(-1))
    (loss * g).backward()
    return hd.grad, wd.grad


def score_bound(h, cand, slot_of, slot_nodes, w, bf16=False):
    h, w = _operands(h, w, bf16)
    H = h.shape[1]
    a = h.abs()
    return _gamma(2 * H + 2) * (a[cand] @ w[:H].abs() + a[slot_nodes][slot_of] @ w[H:].abs())


def lse_bound(h, cand, slot_of, slot_nodes, w, bf16=False):
    J = slot_nodes.shape[0]
    sb = score_bound(h, cand, slot_of, slot_nodes, w, bf16)
    worst = torch.zeros(J, dtype=torch.float64).scatter_reduce(0, slot_of, sb, "amax", include_self=True)
    count = torch.zeros(J, dtype=torch.float64).scatter_add(0, slot_of, torch.ones_like(sb))
    return worst + (count + 8) * U


def loss_bound(h, cand, slot_of, slot_nodes, correct, w, bf16=False):
    ref = varmisuse(h, cand, slot_of, slot_nodes, correct, w, bf16)
    terms = ref["score"][correct] - ref["lse"][slot_of[correct]]
    S = correct.shape[0]
    per = score_bound(h, cand, slot_of, slot_nodes, w, bf16)[correct] + lse_bound(h, cand, slot_of, slot_nodes, w, bf16)[slot_of[correct]]
    return float(per.sum() / S + _gamma(S + 2) * terms.abs().sum() / S)
