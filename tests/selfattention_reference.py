"""Float restatement of the reference's MultiHeadSelfAttentionMessagePassing (selfattmessagepassing.py:59-128), written from its
semantics, and the per-element error bound of the native attention kernel (DESIGN.md §3.8 / §4).

``attention`` and ``layer_forward`` run in the dtype of their inputs: in float32 they reproduce the reference's own outputs bit for bit
(the same torch ops in the same order), in float64 they are the accuracy reference.  ``emulate_kernel`` is a float32 emulation of the
kernel's order (3xFP16 split operands, 64-key blocks with an online softmax); ``corrections=False`` drops the two correction products.
"""
import math

import torch
import torch.nn.functional as F

from helpers import split_f16

PREFIX = "_MultiHeadSelfAttentionMessagePassing__"
U = 2.0 ** -24          # unit roundoff of fp32


def chunks(n2g: torch.Tensor, max_num_nodes: int):
    """(start, end) row ranges: graph g owns [off_g, off_g + c_g) with c_g the number of ids g, cut into max_num_nodes-row chunks."""
    counts = torch.bincount(n2g.cpu()).tolist() if n2g.numel() else []
    out, off = [], 0
    for c in counts:
        for s in range(0, c, max_num_nodes):
            out.append((off + s, off + min(s + max_num_nodes, c)))
        off += c
    return out


def split_heads(t: torch.Tensor, heads: int, dk: int):
    t = t.reshape(t.shape[0], heads, -1)
    return t[:, :, :dk], t[:, :, dk:2 * dk], t[:, :, 2 * dk:]


def attention(t: torch.Tensor, n2g: torch.Tensor, heads: int, dk: int, max_num_nodes: int) -> torch.Tensor:
    """o [R, heads * dv] from t [R, heads * (2 dk + dv)]: row i attends with its a_i over the b_j of its chunk."""
    a, b, v = split_heads(t, heads, dk)
    outs = []
    for s, e in chunks(n2g, max_num_nodes):
        scores = torch.einsum("khd,vhd->khv", a[s:e], b[s:e]) / (dk ** 0.5)
        outs.append(torch.einsum("khv,vhd->khd", torch.softmax(scores, dim=-1), v[s:e]))
    o = torch.cat(outs, dim=0) if outs else v[:0]
    return o.reshape(o.shape[0], -1)


def layer_forward(x, n2g, sd, heads, dk, max_num_nodes):
    """The layer's forward (eval mode) on the state_dict ``sd`` (reference keys)."""
    w = lambda n: sd[PREFIX + n]  # noqa: E731
    t = F.linear(x, w("selfatt_head_transforms.weight"))
    o = attention(t, n2g, heads, dk, max_num_nodes)
    out = F.linear(o, w("summarization_layer.weight"))
    d = out.shape[1]
    y1 = F.layer_norm(out + x, (d,), w("layer_norm1.weight"), w("layer_norm1.bias"))
    hidden = F.relu(F.linear(y1, w("intermediate_layer.weight"), w("intermediate_layer.bias")))
    out = F.linear(hidden, w("output_layer.weight"), w("output_layer.bias"))
    return F.layer_norm(out + y1, (d,), w("layer_norm2.weight"), w("layer_norm2.bias"))


def bound(t: torch.Tensor, n2g: torch.Tensor, heads: int, dk: int, max_num_nodes: int) -> torch.Tensor:
    """Per-element bound on |o_kernel - o_exact| for the fp32 kernel (DESIGN.md §4), computed in float64 from t:
        logit  e_s,ij = (3 + ceil(dk / 16) + 1) 2^-22 A_ij + 2^-24 |s_ij| + 2^-30 sum_k (|a_ik| + |b_jk|),  A_ij = sum_k |a_ik b_jk| / sqrt(dk)
               (operand splits 2^-22 each side and the dropped lo'·lo' term; one truncating accumulate per k16 wgmma; the division)
        weight r_ij  = e_s,ij + 2^-22 (3 + |s_ij - m_i| / 4 + n_blocks)     (expf, P split, argument rounding, one rescale per key block)
        o_i:   |d o_i| <= S_i (2 max_j r_ij + (n / 16 + 4) 2^-22 + (n / 4 + 4) 2^-24) + 2^-34,   S_i = sum_j p_ij |v_j|
               (softmax sensitivity; V split and one truncating accumulate per k16 wgmma over n keys; per-thread l sums of n / 4 terms
               and the quad reduction; combine and division)."""
    t = t.double()
    a, b, v = split_heads(t, heads, dk)
    out = torch.empty(t.shape[0], heads, v.shape[2], dtype=torch.float64, device=t.device)
    for s, e in chunks(n2g, max_num_nodes):
        n = e - s
        nb = math.ceil(n / 64)
        aa, bb, vv = a[s:e], b[s:e], v[s:e]
        sc = torch.einsum("khd,vhd->khv", aa, bb) / math.sqrt(dk)
        A = torch.einsum("khd,vhd->khv", aa.abs(), bb.abs()) / math.sqrt(dk)
        tiny = aa.abs().sum(-1)[:, :, None] + bb.abs().sum(-1).transpose(0, 1)[None]
        e_s = (4 + math.ceil(dk / 16)) * 2.0 ** -22 * A + U * sc.abs() + 2.0 ** -30 * tiny
        m = sc.max(dim=-1, keepdim=True).values
        r = e_s + 2.0 ** -22 * (3 + (m - sc) / 4 + nb)
        p = torch.softmax(sc, dim=-1)
        S = torch.einsum("khv,vhd->khd", p, vv.abs())
        rel = 2 * r.max(dim=-1, keepdim=True).values + (n / 16 + 4) * 2.0 ** -22 + (n / 4 + 4) * U
        out[s:e] = S * rel + 2.0 ** -34
    return out.reshape(t.shape[0], -1)


def _split16(x: torch.Tensor):
    hi, lo = split_f16(x)
    return hi.float(), lo.float()


def emulate_kernel(t: torch.Tensor, n2g: torch.Tensor, heads: int, dk: int, max_num_nodes: int, corrections: bool = True) -> torch.Tensor:
    """float32 emulation of the forward kernel's order: split operands, 64-key blocks, online softmax, P split, fp32 accumulators
    (products summed exactly by float64 einsums and rounded once per block, which the bound's accumulate terms cover)."""
    t = t.float()
    a, b, v = split_heads(t, heads, dk)
    (ah, al), (bh, bl), (vh, vl) = _split16(a), _split16(b), _split16(v)
    out = torch.empty(t.shape[0], heads, v.shape[2], dtype=torch.float32)
    mm = lambda eq, x, y: torch.einsum(eq, x.double(), y.double()).float()  # noqa: E731
    sqrt_dk = torch.tensor(math.sqrt(dk), dtype=torch.float32)
    for s, e in chunks(n2g, max_num_nodes):
        m = torch.full((e - s, heads, 1), -math.inf)
        l = torch.zeros(e - s, heads, 1)
        om = torch.zeros(e - s, heads, v.shape[2])
        oc = torch.zeros_like(om)
        for j0 in range(s, e, 64):
            j1 = min(j0 + 64, e)
            sm = mm("khd,vhd->khv", ah[s:e], bh[j0:j1])
            if corrections:
                sc = mm("khd,vhd->khv", ah[s:e], bl[j0:j1]) + mm("khd,vhd->khv", al[s:e], bh[j0:j1])
                sm = sm + sc / 2048.0
            sv = sm / sqrt_dk
            mx = torch.maximum(m, sv.max(dim=-1, keepdim=True).values)
            r = torch.exp(m - mx)
            l, om, oc, m = l * r, om * r, oc * r, mx
            p = torch.exp(sv - m)
            l = l + p.sum(dim=-1, keepdim=True)
            ph, pl = _split16(p)
            om = om + mm("khv,vhd->khd", ph, vh[j0:j1])
            if corrections:
                oc = oc + mm("khv,vhd->khd", ph, vl[j0:j1]) + mm("khv,vhd->khd", pl, vh[j0:j1])
        out[s:e] = (om + oc / 2048.0) / l
    return out.reshape(t.shape[0], -1)


# ---- backward ---------------------------------------------------------------------------------------------------------------
def _gamma(n):
    return n * U / (1 - n * U)


def _chunk_batches(n2g: torch.Tensor, max_num_nodes: int, heads: int, budget: int = 1 << 24):
    """The chunks of ``chunks`` in groups padded to the group's longest chunk: (row index [C, n], valid [C, n]) with at most about
    ``budget`` elements in a [C, heads, n, n] tensor."""
    group, longest = [], 0
    for s, e in chunks(n2g, max_num_nodes) + [(None, None)]:
        if group and (s is None or (len(group) + 1) * heads * max(longest, e - s) ** 2 > budget):
            ar = torch.arange(longest)
            starts = torch.tensor([a for a, _ in group])[:, None]
            valid = ar[None] < torch.tensor([b - a for a, b in group])[:, None]
            yield torch.where(valid, starts + ar[None], torch.zeros((), dtype=torch.int64)), valid
            group, longest = [], 0
        if s is not None:
            group.append((s, e))
            longest = max(longest, e - s)


def _backward(t, o, lse, d_o, n2g, heads, dk, max_num_nodes, with_bound):
    """float64 (d t, its bound or None) per chunk group, on t's device."""
    dev = t.device
    R = t.shape[0]
    t, o, lse, d_o = (z.double() for z in (t, o, lse, d_o))
    a, b, v = split_heads(t, heads, dk)
    dv_ = v.shape[2]
    o, d_o = o.reshape(R, heads, dv_), d_o.reshape(R, heads, dv_)
    lse = lse.reshape(R, heads)
    rt = math.sqrt(dk)
    out = torch.zeros(R, heads, 2 * dk + dv_, dtype=torch.float64, device=dev)
    bnd = torch.zeros_like(out) if with_bound else None
    for idx, valid in _chunk_batches(n2g, max_num_nodes, heads):
        idx, valid = idx.to(dev), valid.to(dev)
        n = int(valid.sum(1).max())
        m = valid[:, :, None, None].double()                            # [C, n, 1, 1]
        A, B, V, dO, O = (z[idx] * m for z in (a, b, v, d_o, o))        # [C, n, heads, d]
        ls = lse[idx] * valid[:, :, None]                               # [C, n, heads]
        pair = (valid[:, None, :, None] & valid[:, None, None, :]).double()     # [C, 1, i, j]
        s = torch.einsum("cihk,cjhk->chij", A, B) / rt
        p = torch.exp(s - ls.permute(0, 2, 1)[..., None]) * pair
        dp = torch.einsum("cihk,cjhk->chij", dO, V)
        delta = (dO * O).sum(-1).permute(0, 2, 1)[..., None]            # [C, h, i, 1]
        ds = p * (dp - delta)
        g_v = torch.einsum("chij,cihk->cjhk", p, dO)
        g_b = torch.einsum("chij,cihk->cjhk", ds, A) / rt
        g_a = torch.einsum("chij,cjhk->cihk", ds, B) / rt
        rows, ok = idx[valid], valid
        out[rows] = torch.cat((g_a, g_b, g_v), dim=-1)[ok]
        if not with_bound:
            continue
        absum = torch.einsum("cihk,cjhk->chij", A.abs(), B.abs())
        arg = _gamma(dk) * absum / rt + 2 * U * s.abs() + U * (s - ls.permute(0, 2, 1)[..., None]).abs()
        e_p = (p * (torch.expm1(arg) * (1 + 4 * U) + 4 * U) + 2.0 ** -148) * pair
        e_dp = _gamma(dv_) * torch.einsum("cihk,cjhk->chij", dO.abs(), V.abs())
        e_delta = _gamma(dv_) * (dO * O).abs().sum(-1).permute(0, 2, 1)[..., None]
        diff = (dp - delta).abs()
        e_ds = (e_p * diff + p * (e_dp + e_delta) + 2 * U * p * diff) * pair
        gn = _gamma(n)
        b_v = torch.einsum("chij,cihk->cjhk", e_p, dO.abs()) + gn * torch.einsum("chij,cihk->cjhk", p, dO.abs())
        b_b = (torch.einsum("chij,cihk->cjhk", e_ds, A.abs()) + gn * torch.einsum("chij,cihk->cjhk", ds.abs(), A.abs())) / rt + 2 * U * g_b.abs()
        b_a = (torch.einsum("chij,cjhk->cihk", e_ds, B.abs()) + gn * torch.einsum("chij,cjhk->cihk", ds.abs(), B.abs())) / rt + 2 * U * g_a.abs()
        bnd[rows] = torch.cat((b_a, b_b, b_v), dim=-1)[ok]
    out = out.reshape(R, -1)
    return out, (bnd.reshape(R, -1) * 1.01 + 1e-37 if with_bound else None)


def backward_formula(t, o, lse, d_o, n2g, heads, dk, max_num_nodes):
    """d t [R, heads (2 dk + dv)] in float64 from exactly the backward kernels' inputs t, o, lse and d o (o and lse those of the
    forward kernel), on t's device: per chunk and head, s_ij = a_i . b_j / sqrt(dk), p_ij = exp(s_ij - lse_i), delta_i = dO_i . o_i,
    ds_ij = p_ij (dO_i . v_j - delta_i); dv_j = sum_i p_ij dO_i, db_j = sum_i ds_ij a_i / sqrt(dk), da_i = sum_j ds_ij b_j / sqrt(dk).
    With the exact float64 o and lse this is the gradient of ``attention``."""
    return _backward(t, o, lse, d_o, n2g, heads, dk, max_num_nodes, False)[0]


def backward_bound(t, o, lse, d_o, n2g, heads, dk, max_num_nodes):
    """Per-element bound on |d t_kernel - backward_formula| for the fp32 backward kernels (DESIGN.md §3.8 / §4), in float64, from
    the order of selfatt.cu's header.  With u = 2^-24, gamma_n = n u / (1 - n u) and n the chunk's rows:
        s      e_arg = gamma_dk sum_k |a_ik b_jk| / sqrt(dk) + 2u |s_ij| + u |s_ij - lse_i|     (the fmaf chain over dk, sqrtf and the
               division, the subtraction of lse)
        p      e_p = p (expm1(e_arg) (1 + 4u) + 4u) + 2^-148                        (expf: 2 ulp = 4u; an underflow to 0 or a subnormal)
        dp     e_dp = gamma_dv sum_k |dO_ik v_jk|,   delta  e_delta = gamma_dv sum_k |dO_ik o_ik|   (the fmaf chains over dv)
        ds     e_ds = e_p |dp - delta| + p (e_dp + e_delta) + 2u p |dp - delta|      (the difference and the product)
        dv_j   sum_i e_p |dO_i| + gamma_n sum_i p |dO_i|                             (the fmaf chain over the chunk's rows, in order)
        db_j   (sum_i e_ds |a_i| + gamma_n sum_i |ds a_i|) / sqrt(dk) + 2u |db_j|    (the chain, then sqrtf and the division)
        da_i   (sum_j e_ds |b_j| + gamma_n sum_j |ds b_j|) / sqrt(dk) + 2u |da_i|
    All terms are absolute (sums of |terms|), so cancellation in dp - delta is covered.  Second-order terms: 1 % slack, plus 1e-37
    absolute for subnormal products."""
    return _backward(t, o, lse, d_o, n2g, heads, dk, max_num_nodes, True)[1]


def _fl(x):
    return x.float().double()


def emulate_backward(t, o, lse, d_o, n2g, heads, dk, max_num_nodes, mutant=None):
    """float32 emulation of the backward kernels' order (CPU, small shapes): fmaf as a float64 multiply-add rounded to float32, expf
    as float64 exp rounded to float32.  ``mutant`` (the bound must reject each): "no_delta" drops delta; "db_unscaled" leaves db
    undivided by sqrt(dk); "kv_own_tile" limits the key-side kernel's query loop to the key's own 64-row tile; "q_short" ends the
    query-side kernel's key loop one row early."""
    R = t.shape[0]
    t, o, lse, d_o = (z.float().double() for z in (t, o, lse, d_o))
    a, b, v = split_heads(t, heads, dk)
    dv_ = v.shape[2]
    o, d_o = o.reshape(R, heads, dv_), d_o.reshape(R, heads, dv_)
    lse = lse.reshape(R, heads)
    rt = _fl(torch.tensor(math.sqrt(dk)))
    out = torch.zeros(R, heads, 2 * dk + dv_, dtype=torch.float64)
    delta_all = torch.zeros(R, heads, dtype=torch.float64)
    for k in range(dv_):
        delta_all = _fl(d_o[:, :, k] * o[:, :, k] + delta_all)
    if mutant == "no_delta":
        delta_all = torch.zeros_like(delta_all)
    for s0, e0 in chunks(n2g, max_num_nodes):
        A, B, V, dO = a[s0:e0], b[s0:e0], v[s0:e0], d_o[s0:e0]
        n = e0 - s0
        s = torch.zeros(heads, n, n, dtype=torch.float64)
        for k in range(dk):
            s = _fl(A[:, :, k].T[:, :, None] * B[:, :, k].T[:, None, :] + s)
        dp = torch.zeros_like(s)
        for k in range(dv_):
            dp = _fl(dO[:, :, k].T[:, :, None] * V[:, :, k].T[:, None, :] + dp)
        p = _fl(torch.exp(_fl(_fl(s / rt) - lse[s0:e0].T[:, :, None])))
        ds = _fl(p * _fl(dp - delta_all[s0:e0].T[:, :, None]))
        gv = torch.zeros(heads, n, dv_, dtype=torch.float64)           # [h, j, .]
        gb = torch.zeros(heads, n, dk, dtype=torch.float64)
        tile = torch.arange(n) // 64
        for i in range(n):
            use = (tile == tile[i]) if mutant == "kv_own_tile" else torch.ones(n, dtype=torch.bool)
            upd_v = _fl(p[:, i, :, None] * dO[i][:, None, :] + gv)
            upd_b = _fl(ds[:, i, :, None] * A[i][:, None, :] + gb)
            gv = torch.where(use[None, :, None], upd_v, gv)
            gb = torch.where(use[None, :, None], upd_b, gb)
        ga = torch.zeros(heads, n, dk, dtype=torch.float64)            # [h, i, .]
        for j in range(n - 1 if mutant == "q_short" else n):
            ga = _fl(ds[:, :, j, None] * B[j][:, None, :] + ga)
        gb = gb if mutant == "db_unscaled" else _fl(gb / rt)
        out[s0:e0] = torch.cat((_fl(ga / rt), gb, gv), dim=-1).permute(1, 0, 2)
    return out.reshape(R, -1).float()
