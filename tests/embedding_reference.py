"""Float restatement of the reference's TokenUnitEmbedder / SubtokenUnitEmbedder (strelementrepresentationmodel.py:16-89), written from
their semantics, a float32 emulation of the native kernels' order (DESIGN.md §3.12) and the per-element error bounds derived from it.

``module_forward`` runs in the dtype of its inputs: in float32 it reproduces the reference's outputs and autograd gradients bit for bit
(the same library ops in the same order), in float64 it is the accuracy reference.  ``emulate_forward`` / ``emulate_backward`` repeat
the kernels' float32 operations one by one (every kernel operation is an explicit round-to-nearest intrinsic, and torch's float32 CPU
add and divide round the same way), so the kernels must match them bit for bit.
"""
import math

import torch
import torch.nn.functional as F

CHUNK = 32              # pergraph::CHUNK: occurrences per warp chunk of the backward
U = 2.0 ** -24          # unit roundoff of fp32
U_BF16 = 2.0 ** -8      # of one rounding to bf16 (8 significand bits)


def clamp_lengths(ids, lengths):
    S = ids.shape[1]
    return torch.full((ids.shape[0],), S, dtype=torch.int64) if lengths is None else lengths.clamp(0, S)


def pool(embedded, lengths, kind):
    """The reference's pooling of embedded [B, S, D] over the first lengths[i] slots."""
    S = embedded.shape[1]
    mask = torch.arange(S).unsqueeze(0) < lengths.unsqueeze(-1)
    if kind == "mean":
        embedded = embedded * mask.unsqueeze(-1).to(embedded.dtype)
        return embedded.sum(dim=-2) / (lengths.unsqueeze(-1).to(embedded.dtype) + 1e-10)
    if kind == "sum":
        return (embedded * mask.unsqueeze(-1).to(embedded.dtype)).sum(dim=-2)
    if kind == "max":
        return embedded.masked_fill(~mask.unsqueeze(-1), -math.inf).max(dim=-2)[0]
    raise ValueError(kind)


def module_forward(table, ids, lengths=None, kind="sum", weight=None):
    """Eval-mode forward of TokenUnitEmbedder (ids [B], lengths None) or SubtokenUnitEmbedder (ids [B, S]); weight: the dense output
    layer's [D, D] or None."""
    if ids.dim() == 1:
        return F.embedding(ids, table)
    out = pool(F.embedding(ids, table), lengths, kind)
    return out if weight is None else F.linear(out, weight)


# ---- the kernels' order ----------------------------------------------------------------------------------------------------------
def emulate_forward(table, ids, lengths=None, kind="sum", out_dtype=torch.float32, ignore_lengths=False, mean_by_slots=False):
    """(out [B, D], arg [B, D] uint8) of the bag kernel: the valid slots added in slot order in float32, mean divided by
    fl(len) + 1e-10, max by strict compare (lowest slot wins), rounded once to ``out_dtype``.  ``ignore_lengths`` / ``mean_by_slots``:
    mutants the bound must reject (every slot taken as valid; mean divided by S)."""
    if ids.dim() == 1:
        ids = ids.unsqueeze(1)
    table = table.float()
    B, S = ids.shape
    D = table.shape[1]
    lens = clamp_lengths(ids, None if ignore_lengths else lengths)
    acc = torch.full((B, D), -math.inf if kind == "max" else 0.0, dtype=torch.float32)
    arg = torch.zeros(B, D, dtype=torch.uint8)
    for s in range(S):
        m = lens > s
        x = table[ids[m, s]]
        if kind == "max":
            win = x > acc[m]
            acc[m] = torch.where(win, x, acc[m])
            arg[m] = torch.where(win, torch.tensor(s, dtype=torch.uint8), arg[m])
        else:
            acc[m] = acc[m] + x
    if kind == "mean":
        den = torch.full((B,), float(S)) if mean_by_slots else clamp_lengths(ids, lengths).float() + torch.tensor(1e-10, dtype=torch.float32)
        acc = acc / den[:, None]
    return acc.to(out_dtype), arg


def occurrences(ids, lengths, V):
    """(row, slot, token) of the valid slots in the plan's order: by token, then by (row, slot); ids outside [0, V) count as token 0."""
    if ids.dim() == 1:
        ids = ids.unsqueeze(1)
    B, S = ids.shape
    lens = clamp_lengths(ids, lengths)
    valid = (torch.arange(S)[None, :] < lens[:, None]).flatten()
    e = torch.arange(B * S)[valid]
    tok = ids.flatten()[valid]
    tok = torch.where((tok < 0) | (tok >= V), torch.zeros_like(tok), tok)
    order = torch.argsort(tok, stable=True)
    e, tok = e[order], tok[order]
    return e // S, e % S, tok


def emulate_backward(d_out, ids, lengths, kind, V, arg=None):
    """d table [V, D] in the backward kernel's order: every token's occurrences in plan order, CHUNK of them added sequentially into
    one partial (mean: each term divided by fl(len) + 1e-10 first; max: only where arg == slot), the partials added in chunk order."""
    d_out = d_out.float()
    D = d_out.shape[1]
    row, slot, tok = occurrences(ids, lengths, V)
    term = d_out[row]
    if kind == "mean":
        lens = clamp_lengths(ids if ids.dim() == 2 else ids.unsqueeze(1), lengths)
        term = term / (lens[row].float() + torch.tensor(1e-10, dtype=torch.float32))[:, None]
    elif kind == "max":
        term = torch.where(arg[row] == slot[:, None].to(torch.uint8), term, torch.zeros(()))
    counts = torch.bincount(tok, minlength=V)
    start = torch.cumsum(counts, 0) - counts
    within = torch.arange(tok.numel()) - start[tok]          # position of the occurrence among its token's
    chunk_of, t_in = within // CHUNK, within % CHUNK
    nchunks = (counts + CHUNK - 1) // CHUNK
    chunk_base = torch.cumsum(nchunks, 0) - nchunks
    cid = chunk_base[tok] + chunk_of
    partial = torch.zeros(int(nchunks.sum()), D, dtype=torch.float32)
    for t in range(CHUNK):
        m = t_in == t
        partial[cid[m]] = partial[cid[m]] + term[m]
    d_table = torch.zeros(V, D, dtype=torch.float32)
    for j in range(int(nchunks.max()) if V else 0):
        m = nchunks > j
        d_table[m] = d_table[m] + partial[chunk_base[m] + j]
    return d_table


# ---- bounds ----------------------------------------------------------------------------------------------------------------------
def linear_bound(x_abs, w_abs):
    """|fl(x W^T) - x W^T| for the native fp32 dense operator: (K + 4) u |x| |W|^T (K products and additions in some order)."""
    return (x_abs.shape[1] + 4) * U * (x_abs @ w_abs.T)


def bound(table, ids, lengths=None, kind="sum", weight=None, table_first=False, out_dtype=torch.float32):
    """Per-element bound on |out_native - out_exact| in float64.  With n = len_i valid slots:
        bag over rows known to e_T:   sum  (n - 1) u sum_s |T| + sum_s e_T;  mean: that / den + 2u |mean| (den and the division);
                                      max  max_s e_T (no rounding)
        pool first:   e_T = 0, then the dense operator on the pooled rows p: e_p |W|^T + linear_bound(|p|, |W|)
        table first:  T = table W^T, e_T = linear_bound(|table|, |W|), then the bag
        bf16 output:  + 2^-8 (|out| + bound) for the one rounding at the store.  A row whose exact value is infinite (max of no slot)
        must be reproduced exactly: its bound is 0."""
    if ids.dim() == 1:
        ids = ids.unsqueeze(1)
    table = table.double()
    lens = clamp_lengths(ids, lengths)
    S = ids.shape[1]
    mask = (torch.arange(S)[None, :] < lens[:, None]).unsqueeze(-1).double()
    w = None if weight is None else weight.double()

    def bag(T, e_T):
        rows, e_rows = T[ids], e_T[ids]
        if kind == "max":
            return (e_rows * mask).amax(dim=1)
        n = lens.double()[:, None]
        b = (n - 1).clamp(min=0) * U * (rows.abs() * mask).sum(1) + (e_rows * mask).sum(1)
        if kind == "mean":
            den = n + 1e-10
            b = b / den + 2 * U * ((rows * mask).sum(1) / den).abs()
        return b

    if w is None:
        b = bag(table, torch.zeros_like(table))
        exact = module_forward(table, ids, lens, kind)
    elif table_first:
        b = bag(table @ w.T, linear_bound(table.abs(), w.abs()))
        exact = module_forward(table, ids, lens, kind, w)
    else:
        pooled = module_forward(table, ids, lens, kind)
        finite = torch.where(torch.isfinite(pooled), pooled, torch.zeros(()).double())
        b = bag(table, torch.zeros_like(table)) @ w.abs().T + linear_bound(finite.abs(), w.abs())
        exact = module_forward(table, ids, lens, kind, w)
    if out_dtype == torch.bfloat16:
        b = b + U_BF16 * (torch.where(torch.isfinite(exact), exact, torch.zeros(()).double()).abs() + b)
    b = torch.where(torch.isfinite(exact), b * 1.01 + 1e-30, torch.zeros(()).double())
    return b


def backward_bound(d_out, ids, lengths, kind, V, arg=None):
    """Per-element bound on |d_table_native - d_table_exact|: a token with n occurrences in k chunks adds at most CHUNK + k terms along
    any path, and mean divides each term first: (CHUNK + k + 2) u sum |term|."""
    d_out = d_out.double()
    row, slot, tok = occurrences(ids, lengths, V)
    term = d_out[row].abs()
    if kind == "mean":
        lens = clamp_lengths(ids if ids.dim() == 2 else ids.unsqueeze(1), lengths)
        term = term / (lens[row].double() + 1e-10)[:, None]
    elif kind == "max":
        term = torch.where(arg[row] == slot[:, None].to(torch.uint8), term, torch.zeros(()).double())
    counts = torch.bincount(tok, minlength=V)
    k = ((counts + CHUNK - 1) // CHUNK).double()[:, None]
    total = torch.zeros(V, d_out.shape[1], dtype=torch.float64).index_add(0, tok, term)
    return (CHUNK + k + 2) * U * total * 1.01 + 1e-30
