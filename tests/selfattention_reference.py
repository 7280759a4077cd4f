"""Float restatement of the reference's MultiHeadSelfAttentionMessagePassing (selfattmessagepassing.py:59-128), written from its
semantics, and the per-element error bound of the native attention kernel (DESIGN.md §3.8 / §4).

``attention`` and ``layer_forward`` run in the dtype of their inputs: in float32 they reproduce the reference's own outputs bit for bit
(the same torch ops in the same order), in float64 they are the accuracy reference.  ``emulate_kernel`` is a float32 emulation of the
kernel's order (3xFP16 split operands, 64-key blocks with an online softmax); ``corrections=False`` drops the two correction products.
"""
import math

import torch
import torch.nn.functional as F

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
    hi = x.half().float()
    return hi, ((x - hi) * 2048.0).half().float()


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
