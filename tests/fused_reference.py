"""Float64 reference of the fused aggregation kernel (csrc/fused_mp.cu) with an error bound for every output element, and
graphs built to drive that kernel through each of its structural branches.

The layer under test is ``MlpMessagePassingLayer(K, 128, 128, T, agg, message_activation=act, use_layer_norm=False,
use_dense_layer=False)``: its fused output is the kernel's aggregate itself (fp32 ``out_mode`` 0, bf16 ``out_mode`` 1),
optionally through an activation.  Message e of type t is m_e = W_t x_e, x_e = h[src] (or [h[src]; h[tgt]]), and the
aggregate of target v reduces the messages of v in plan order (type-major, then list order).

Error model, fp32 path (3xFP16).  u = 2^-24.  Each operand x is split into fp16 hi = fl16(x) and lo' = fl16(2^11 (x - hi));
hi + 2^-11 lo' represents x to 4u |x| (|x - hi| <= 2^-11 |x|, lo' is rounded to 2^-11 of that), plus 2^-36 absolute when
lo' is an fp16 subnormal (|x| below fp16's normal range).  The kernel computes hi*hi + 2^-11 (hi*lo' + lo'*hi) and drops
2^-22 lo'*lo' (<= 4u |x w|).  The products are exact on the tensor cores; each of the S = NSEG*K/16 k-steps adds one
wgmma block into an fp32 accumulator, which we allow 2u of the step's mass (one ulp: truncating alignment); the correction
accumulator's own rounding is 2^-11 smaller (1u for all of it) and the final fma combining the two costs 1u.  So per
message and feature

    |m~ - m| <= C_S * mass + 2^-36 * (sum_k |w_k| + sum_k |x_k|),   C_S = (8 + 4 + 2 S + 1 + 1) u = (14 + 2 S) u,

with mass = sum_k |w_k x_k|.  S <= 16 (K = 128, NSEG = 2) gives C_S <= 46 u < 2^-18; running hi*hi alone errs by ~2^-12
sqrt(K) of the mass and fails (``tests/test_fused_reference_cpu.py`` checks that).  The sum / mean reduction is a
sequential fp32 sum of n messages: + gamma_n sum_e (|m_e| + err_e), gamma_n = n u / (1 - n u); the mean's division adds u
of the result.  Max / min move by at most the largest message perturbation.  Targets without messages must be exactly 0.

bf16 path.  Inputs and weights are bf16, their products exact, each message is the fp32 tensor-core sum rounded once to
bf16; the reduction is fp32 in plan order, then the output is rounded to bf16.  The reference emulates exactly that, with
one freedom: a message may be the bf16 rounding of any value within the fp32 accumulation error e = (4 S + 4) u of its mass.
Where [m - e, m + e] contains no bf16 rounding midpoint that is exactly bf16(m); near a midpoint it is +-1 bf16 ulp; a
message that cancels to far below its mass (|m| < e) may be several of its own ulps off.  Such messages widen the bound of
their aggregate by that distance (plus the fp32 re-rounding of a sum that saw them).  The output may differ by 1 bf16 ulp.

An activation after the aggregate propagates the bound through its Lipschitz constant (GELU 1.13, ReLU 1; tanh: its largest
slope within the bound) and adds its own fp32 evaluation error, 8u (|x| + |act(x)|).
"""
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from oracle import ptgnn_oracle as O

U = 2.0 ** -24
ABS_F16 = 2.0 ** -36
LIPSCHITZ = {None: 1.0, "gelu": 1.13, "tanh": 1.0, "relu": 1.0}


def fp32_message_constant(K: int, nseg: int) -> float:
    S = nseg * K // 16
    c = (14 + 2 * S) * U
    assert c <= 2.0 ** -18, "the fp32 message bound must stay at or below 2^-18 of the mass"
    return c


def bf16_window_constant(K: int, nseg: int) -> float:
    return (4 * (nseg * K // 16) + 4) * U


# ---- messages ---------------------------------------------------------------------------------------------------------
def _bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).to(torch.bfloat16).double()


def messages(h: torch.Tensor, adj, weights: Sequence[torch.Tensor], use_target: bool, bf16: bool, chunk: int = 8192):
    """-> (tgt [E] int64, m [E, D] float64, err [E, D] float64) in concatenated (type-major) edge order.

    fp32: m = exact W x, err = the per-message bound above.  bf16: m = the nominal bf16 message (round-to-nearest of the
    exact value), err = how far another bf16 rounding within the accumulation error lies from it (0 for most messages)."""
    h64 = h.double()
    K = h.shape[1]
    nseg = 2 if use_target else 1
    tgts, ms, errs = [], [], []
    for (s, t), w in zip(adj, weights):
        W = (w.to(torch.bfloat16) if bf16 else w).double()
        Wa = W.abs()
        wsum = Wa.sum(1)
        for a in range(0, s.shape[0], chunk):
            ss, tt = s[a:a + chunk], t[a:a + chunk]
            X = torch.cat([h64[ss], h64[tt]], 1) if use_target else h64[ss]
            m = X @ W.T
            mass = X.abs() @ Wa.T
            if bf16:
                # the kernel's message is the bf16 rounding of some value within e of m; widened by 2^-22 |m| so that the
                # double rounding float64 -> fp32 -> bf16 used here cannot narrow the interval
                e = 1.01 * bf16_window_constant(K, nseg) * mass + 2.0 ** -22 * m.abs()
                b = _bf16(m)
                err = torch.maximum(_bf16(m + e) - b, b - _bf16(m - e))
                m = b
            else:
                err = fp32_message_constant(K, nseg) * mass + ABS_F16 * (X.abs().sum(1, keepdim=True) + wsum[None, :])
            ms.append(m)
            errs.append(err)
        tgts.append(t)
    return torch.cat(tgts), torch.cat(ms), torch.cat(errs)


# ---- reductions -------------------------------------------------------------------------------------------------------
def _seq_sum_f32(tgt: torch.Tensor, m32: np.ndarray, n: int) -> np.ndarray:
    """fp32 sum of each target's messages, one message at a time in edge order, starting from 0 (the kernel's order)."""
    tg = tgt.numpy()
    order = np.argsort(tg, kind="stable")
    ts = tg[order]
    first = np.searchsorted(ts, ts, side="left")
    rank = np.arange(ts.shape[0]) - first
    acc = np.zeros((n, m32.shape[1]), dtype=np.float32)
    for r in range(int(rank.max()) + 1 if rank.size else 0):
        sel = order[rank == r]
        acc[tg[sel]] = acc[tg[sel]] + m32[sel]
    return acc


def _act64(x: torch.Tensor, act: Optional[str]) -> torch.Tensor:
    if act is None:
        return x
    if act == "gelu":
        return torch.nn.functional.gelu(x)
    if act == "tanh":
        return torch.tanh(x)
    if act == "relu":
        return torch.relu(x)
    raise ValueError(act)


def _bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    a = x.abs().clamp(min=2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def activation_bound(pre: torch.Tensor, bnd: torch.Tensor, act: Optional[str]):
    """-> (act(pre), bound): ``bnd`` through the activation's slope plus its fp32 evaluation error.  The slope is the
    Lipschitz constant, except for tanh: its largest slope on [pre - bnd, pre + bnd], 1 - tanh^2(max(|pre| - bnd, 0)) (a
    saturated tanh must not pass a bf16 ulp of its input on unchanged)."""
    ref = _act64(pre, act)
    if act is None:
        return ref, bnd
    slope = 1 - torch.tanh((pre.abs() - bnd).clamp(min=0)) ** 2 if act == "tanh" else LIPSCHITZ[act]
    return ref, slope * bnd + 8 * U * (pre.abs() + ref.abs())


def aggregate(tgt, m, err, num_nodes: int, reduce: str, bf16: bool, act: Optional[str] = None, round_bf16: bool = True):
    """-> (ref [N, D] float64, bound [N, D] float64, pre [N, D] float64): the expected output, the allowed |got - ref| per
    element, and the aggregate before the activation (for epilogues checked elsewhere, e.g. LayerNorm).  bf16 with
    round_bf16=False: the fp32 value before the output's rounding to bf16 (for an epilogue that rounds later)."""
    N, D = num_nodes, m.shape[1]
    cnt = torch.zeros(N, dtype=torch.float64).index_add_(0, tgt, torch.ones(tgt.shape[0], dtype=torch.float64))
    empty = (cnt == 0)[:, None].expand(N, D)
    c = cnt.clamp(min=1)[:, None]
    idx = tgt[:, None].expand_as(m)
    if reduce in ("max", "min"):
        init = -np.inf if reduce == "max" else np.inf
        pre = torch.full((N, D), init, dtype=torch.float64).scatter_reduce_(0, idx, m, "amax" if reduce == "max" else "amin")
        pre = torch.where(empty, torch.zeros_like(pre), pre)
        bnd = torch.zeros(N, D, dtype=torch.float64).scatter_reduce_(0, idx, err, "amax")
    else:
        n = cnt[:, None]
        gamma = n * U / (1 - n * U)
        mag = torch.zeros(N, D, dtype=torch.float64).index_add_(0, tgt, m.abs() + err)
        berr = torch.zeros(N, D, dtype=torch.float64).index_add_(0, tgt, err)
        if bf16:      # exact emulation of the fp32 sum of the nominal messages; ambiguous messages add their ulp and a re-rounding
            pre = torch.from_numpy(_seq_sum_f32(tgt, m.to(torch.float32).numpy(), N)).double()
            bnd = berr + torch.where(berr > 0, 2 * gamma * mag, torch.zeros_like(mag))
            if reduce == "mean":
                pre = (pre.float() / c.float()).double()
                bnd = bnd / c + torch.where(bnd > 0, 2 * U * pre.abs() + bnd / c * U, torch.zeros_like(bnd))
        else:
            pre = torch.zeros(N, D, dtype=torch.float64).index_add_(0, tgt, m)
            bnd = berr + gamma * mag
            if reduce == "mean":
                pre = pre / c
                bnd = bnd / c + U * (pre.abs() + bnd / c)
    ref, bnd = activation_bound(pre, bnd, act)
    if bf16 and round_bf16:
        ref_b = ref.to(torch.float32).to(torch.bfloat16).double()
        bnd = bnd + _bf16_ulp(ref_b.abs() + bnd)
        ref = ref_b
    bnd = torch.where(empty, torch.zeros_like(bnd), bnd)
    return ref, bnd, pre


def check_bound(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str) -> float:
    """Every element within its bound; returns the largest error / bound ratio (elements with a zero bound must be exact)."""
    got = got.detach().cpu().double()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} != {tuple(ref.shape)}"
    err = (got - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        rows, cols = torch.nonzero(bad, as_tuple=True)
        ex = ", ".join(f"[{int(r)},{int(c)}] got {got[r, c].item():.9g} ref {ref[r, c].item():.9g} bound {bound[r, c].item():.3g}"
                       for r, c in zip(rows[:4].tolist(), cols[:4].tolist()))
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside their bound, in {int(rows.unique().numel())} rows: {ex}")
    pos = bound > 0
    return float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0


# ---- structured graphs ------------------------------------------------------------------------------------------------
GROUP_SIZES = (1, 2, 15, 16, 17, 31, 32, 33, 47, 48, 49, 63, 64, 65, 128, 129, 200)
SPLITS = (0, 1, 15, 16, 17, 48, 63, 64)        # lower-half column counts of a 64-edge sub-group (64 = all of it)
EMPTY_TYPE = 1                                 # a type without any edge, between non-empty ones


def structured_graph(B: int, T: int, num_blocks: int, num_edges: int = 50_000, seed: int = 0):
    """Deterministic graph for target-block size B and T >= 3 edge types -> (adjacency list, num_nodes).

    Reserved blocks each hold one designed case (only their own edges): (block, type) groups of every size in GROUP_SIZES;
    64-edge groups with every lower-half count in SPLITS, using rows 0, B/2 - 1, B/2 and B - 1; segments that cross the
    16-column batches and the 64-edge sub-groups, and a hub spanning four sub-groups; targets with several types; groups whose
    lower half ends on row B/2 with an empty upper half (the lower walk is the last to finish).  Runs of empty blocks sit
    between them, the last block is partial, and the remaining blocks get random filler edges with self-loops, duplicate
    edges and sources 0 and N - 1.  ``tests/test_fused_reference_cpu.py`` checks through the block plan that every case occurs."""
    assert T >= 3 and B % 8 == 0
    rng = np.random.RandomState(seed)
    half = B // 2
    N = num_blocks * B - (half + 1)               # the last block has B/2 - 1 rows
    live = [t for t in range(T) if t != EMPTY_TYPE]
    srcs: List[List[int]] = [[] for _ in range(T)]
    tgts: List[List[int]] = [[] for _ in range(T)]
    reserved = set()
    cursor = [0]
    n_case = [0]

    def block():
        b = cursor[0]
        cursor[0] += 1
        reserved.add(b)
        n_case[0] += 1
        if n_case[0] % 5 == 0:                    # a run of empty blocks after every fifth case
            for _ in range(1 + n_case[0] % 3):
                reserved.add(cursor[0])
                cursor[0] += 1
        return b

    def add(t, rows_local, b):
        for r in rows_local:
            srcs[t].append(int(rng.randint(0, N)))
            tgts[t].append(b * B + int(r))

    def layout(t, b, spec):                       # spec: [(row, count)] -> that many edges of type t to each row
        add(t, [r for r, k in spec for _ in range(k)], b)

    for i, n in enumerate(GROUP_SIZES):           # group sizes; the rows are random, both halves
        add(live[i % len(live)], rng.randint(0, B, n), block())
    for i, s in enumerate(SPLITS):                # lower-half column counts of one 64-edge group
        lo = list(rng.randint(0, half, s))
        hi = list(rng.randint(half, B, 64 - s))
        if s >= 2:
            lo[:2] = [0, half - 1]
        elif s == 1:
            lo = [half - 1]
        if 64 - s >= 2:
            hi[:2] = [half, B - 1]
        elif 64 - s == 1:
            hi = [B - 1]
        add(live[(i + 1) % len(live)], lo + hi, block())
    q = max(half - 1, 1)
    t0, t1 = live[0], live[-1]
    # segments across batches: lower rows 0|1|2 = cols 0-9 | 10-21 (15->16) | 22-26, upper B/2 | B-1 = 27-36 (31->32) | 37-63 (47->48)
    layout(t0, block(), [(0, 10), (1, 12), (min(2, half - 1), 5), (half, 10), (B - 1, 27)])
    # a segment across the sub-groups: cols 50-79 (63->64), then an upper-half tail
    layout(t1, block(), [(0, 50), (min(2, half - 1), 30), (half + 1, 20)])
    # hubs: cols 5-194 of one lower-half target (sub-groups 0-3), and an upper-half one over 150 columns
    layout(t0, block(), [(0, 5), (q, 190), (B - 1, 10)])
    layout(t1, block(), [(half, 3), (B - 1, 150)])
    # targets receiving several types (a live type empty in this block), repeated on a few blocks
    for k in range(4):
        b = block()
        for t in live:
            if t == live[1 + k % (len(live) - 1)]:
                continue
            layout(t, b, [(r, 1 + (r + t) % 3) for r in range(B)])
    # last group of the block: lower half ending on row B/2 - 1 and B/2 (as the walk sees it), nothing above; many copies
    for k in range(24):
        b = block()
        layout(t0, b, [(r, 2) for r in range(half)])
        layout(t1, b, [(r, 1) for r in range(0, half, max(1, half // 8))] + [(half - 1, 24), (half, 20)])
    # partial last block: all its rows, several types; the last node is also a source
    last = num_blocks - 1
    reserved.add(last)
    rows_last = N - last * B
    for t in live[:3]:
        add(t, list(range(rows_last)) * 3, last)
    srcs[t0][-1] = N - 1
    assert cursor[0] < last
    # filler: random edges over the remaining blocks (about one block in twelve left empty)
    free = np.array([b for b in range(num_blocks) if b not in reserved and rng.rand() > 1 / 12], dtype=np.int64)
    left = num_edges - sum(len(x) for x in srcs) - 80
    for _ in range(max(left, 0) // 8):
        b = int(free[rng.randint(0, free.shape[0])])
        add(live[rng.randint(0, len(live))], rng.randint(0, B, 8), b)
    v = free[rng.randint(0, free.shape[0], 20)] * B + rng.randint(0, B, 20)
    for k, x in enumerate(v):                     # self-loops, duplicated edges, sources 0 and N - 1
        t = live[k % len(live)]
        srcs[t].append(int(x)); tgts[t].append(int(x))
        for _ in range(3):
            srcs[t].append(int((x * 7 + 3) % N)); tgts[t].append(int(x))
    for t in live[:2]:
        srcs[t] += [0, N - 1]
        tgts[t] += [int(v[0]), int(v[1])]
    adj = []
    for t in range(T):
        perm = rng.permutation(len(srcs[t]))      # list order is not target order
        adj.append((torch.tensor(np.asarray(srcs[t], dtype=np.int64)[perm]), torch.tensor(np.asarray(tgts[t], dtype=np.int64)[perm])))
    return adj, N


def structure_facts(adj, num_nodes: int, B: int) -> Dict[str, object]:
    """What the fused kernel will see on this graph at block size B, recomputed from ``oracle.block_plan``."""
    T = len(adj)
    bp = O.block_plan(adj, num_nodes, B)
    go, tl = bp["group_off"].astype(np.int64), bp["tl_f"].astype(np.int64)
    nblk = (num_nodes + B - 1) // B
    half = B // 2
    f = dict(group_sizes=set(), nb=set(), splits=set(), split_is_n=False, rows=set(), batch_cross=set(), upper_batch_cross=False,
             max_subgroups_per_segment=0, multi_type_targets=0, empty_types=[], empty_type_in_nonempty_block=False,
             empty_block_between=False, max_empty_run=0)
    block_nonempty = np.zeros(nblk, dtype=bool)
    for b in range(nblk):
        for t in range(T):
            e0, e1 = int(go[b * T + t]), int(go[b * T + t + 1])
            n = e1 - e0
            if n == 0:
                continue
            block_nonempty[b] = True
            f["group_sizes"].add(n)
            rows = tl[e0:e1]
            f["rows"].update(int(r) for r in rows if r in (0, half - 1, half, B - 1))
            # segments: runs of equal rows; sub-groups of 64 columns
            starts = np.flatnonzero(np.r_[True, rows[1:] != rows[:-1]])
            ends = np.r_[starts[1:], n]
            for s0, s1 in zip(starts, ends):
                f["max_subgroups_per_segment"] = max(f["max_subgroups_per_segment"], (s1 - 1) // 64 - s0 // 64 + 1)
            for g0 in range(0, n, 64):
                sub = rows[g0:g0 + 64]
                ns = sub.shape[0]
                f["nb"].add((ns + 15) // 16)
                split = int((sub < half).sum())
                f["splits"].add(split)
                f["split_is_n"] |= split == ns and ns > 16
                for c in range(15, ns - 1, 16):
                    if sub[c] == sub[c + 1]:
                        f["batch_cross"].add(c)
                        f["upper_batch_cross"] |= bool(sub[c] >= half)
    counts = [int(a[0].shape[0]) for a in adj]
    sizes = np.diff(go).reshape(nblk, T)
    f["empty_type_in_nonempty_block"] = bool((sizes[block_nonempty][:, np.array(counts) > 0] == 0).any())
    f["empty_types"] = [t for t in range(T) if counts[t] == 0]
    src = np.concatenate([a[0].numpy() for a in adj])
    tgt = np.concatenate([a[1].numpy() for a in adj])
    et = np.repeat(np.arange(T), counts)
    pairs = np.unique(np.stack([tgt, et]), axis=1)
    f["multi_type_targets"] = int((np.bincount(pairs[0], minlength=num_nodes) >= 2).sum())
    run = best = 0
    for b in range(nblk):
        run = 0 if block_nonempty[b] else run + 1
        best = max(best, run)
        if b > 0 and not block_nonempty[b] and block_nonempty[:b].any() and block_nonempty[b + 1:].any():
            f["empty_block_between"] = True
    f["max_empty_run"] = best
    f["partial_last_block"] = num_nodes % B != 0 and bool(block_nonempty[-1])
    f["last_row_target"] = bool((tgt == num_nodes - 1).any())
    f["self_loops"] = int((src == tgt).sum())
    keys = np.unique(np.stack([src, tgt, et]), axis=1)
    f["duplicates"] = int(src.shape[0] - keys.shape[1])
    f["sources_0_and_last"] = bool((src == 0).any() and (src == num_nodes - 1).any())
    f["num_blocks"] = nblk
    return f
