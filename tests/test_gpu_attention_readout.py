"""Attention reducers on the GPU: the attention readout kernel against float64 with per-element bounds, the reducer modules against
the float64 restatement and the reference's fixtures, bf16 against the reference's autocast fixture, no host synchronisation, peak
memory at graph2seq's shape, and training against torch.autograd through the float64 restatement.  Every case runs twice and must
be bit-identical.

Kernel bound (DESIGN.md §3.7 gives the order).  With u = 2^-24 and gamma_k = k u / (1 - k u):
* a logit z is a per-lane fmaf chain over D / 32 features and a five-level butterfly: |dz| <= eps = gamma_{D/32+5} sum_f |x_f qt_f|.
  With E the graph's largest eps, the softmax of the computed logits differs from the exact one by a factor in [e^{-2E}, e^{2E}].
* every node's weight e^{z - M} is formed by its own expf, at most CHUNK - 1 rescales (expf and a product) and the combine's expf:
  4 + 5 (CHUNK - 1) + 4 roundings (expf: 2 ulp = 4 u), plus the arguments' subtractions, whose errors add up to at most (M - z) u
  along the running maxima.  The chunk's sum adds CHUNK roundings, the combine over k chunks k, so numerator and denominator carry
  relative errors of at most gamma_K with K = 4 + 5 (CHUNK - 1) + 4 + CHUNK + k + (M - min z).  The division adds u, and a quotient of
  two sums with relative errors gamma_K deviates by at most 2 gamma_K sum_n p_n |x_n|:
      |do| <= (e^{2E} - 1 + 2 gamma_K + u) sum_n p_n |x_n|
  and |dlse| <= E + gamma_K + 4 u |log L| + u |lse| (logf: 1 ulp).  The float64 p is used for the computed one: 1 % slack."""
import math
import os

import numpy as np
import pytest
import torch

import attention_readout_reference as AR
import global_exchange_reference as GX
from helpers import assert_close, gated_oracle_args
from oracle import ptgnn_oracle as O

pytestmark = pytest.mark.gpu

CHUNK = 32
U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
K_WEIGHT = 4 + 5 * (CHUNK - 1) + 4 + CHUNK


def gamma(k):
    return k * U / (1 - k * U)


def _n2g_layout(name, gen):
    """(node_to_graph_idx [N] int64, num_graphs): the layouts of test_gpu_global_exchange.py."""
    if name == "sizes":            # graphs of 1, CHUNK - 1, CHUNK, CHUNK + 1 and 3 CHUNK + 5 nodes, in node order
        sizes = [1, CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 5]
        return torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes)), len(sizes)
    if name == "one_big":          # 40,000 nodes in one graph
        return torch.zeros(40_000, dtype=torch.int64), 1
    if name == "config2":          # 80 x 2,560 (graph2seq's minibatch shape)
        return torch.repeat_interleave(torch.arange(80), 2560), 80
    if name == "unsorted_gaps":    # shuffled ids, graphs 2 and 7 empty, two trailing empty graphs (num_graphs > max + 1)
        ids = torch.tensor([0, 1, 3, 4, 5, 6, 8])[torch.randint(0, 7, (3000,), generator=gen)]
        ids[:2] = torch.tensor([0, 8])
        return ids, 11
    raise ValueError(name)


def _kernel_ref(x64, n2g, G, qt64):
    """float64 (o [G, heads, D], lse [G, heads], bound_o, bound_lse, z [N, heads]) on the device of x64."""
    N, D = x64.shape
    heads = qt64.shape[1]
    dev = x64.device
    ax = x64.abs()
    count = torch.bincount(n2g, minlength=G).to(torch.float64)
    chunks = torch.ceil(count / CHUNK)
    o = torch.zeros(G, heads, D, dtype=torch.float64, device=dev)
    mass = torch.zeros_like(o)
    lse = torch.full((G, heads), -math.inf, dtype=torch.float64, device=dev)
    E = torch.zeros(G, heads, dtype=torch.float64, device=dev)
    spread = torch.zeros(G, heads, dtype=torch.float64, device=dev)
    logL = torch.zeros(G, heads, dtype=torch.float64, device=dev)
    zs = []
    for h in range(heads):
        qn = qt64[n2g, h]                                                   # [N, D]
        z = (x64 * qn).sum(1)
        eps = gamma(D // 32 + 5) * (ax * qn.abs()).sum(1)
        del qn
        M = torch.full((G,), -math.inf, dtype=torch.float64, device=dev).scatter_reduce_(0, n2g, z, "amax", include_self=True)
        Mn = torch.full((G,), math.inf, dtype=torch.float64, device=dev).scatter_reduce_(0, n2g, z, "amin", include_self=True)
        e = torch.exp(z - M[n2g])
        L = torch.zeros(G, dtype=torch.float64, device=dev).index_add_(0, n2g, e)
        p = e / L[n2g]
        o[:, h] = torch.zeros(G, D, dtype=torch.float64, device=dev).index_add_(0, n2g, x64 * p[:, None])
        mass[:, h] = torch.zeros(G, D, dtype=torch.float64, device=dev).index_add_(0, n2g, ax * p[:, None])
        E[:, h] = torch.zeros(G, dtype=torch.float64, device=dev).scatter_reduce_(0, n2g, eps, "amax", include_self=True)
        has = count.to(dev) > 0
        spread[:, h] = torch.where(has, M - Mn, torch.zeros_like(M))
        logL[:, h] = torch.where(has, torch.log(L), torch.zeros_like(L))
        lse[:, h] = torch.where(has, M + torch.log(L), lse[:, h])
        zs.append(z)
    K = K_WEIGHT + chunks.to(dev)[:, None] + torch.ceil(spread)
    gK = K * U / (1 - K * U)
    bound_o = ((torch.exp(2 * E) - 1 + 2 * gK + U)[:, :, None] * mass + 1e-30 * mass) * 1.01
    bound_lse = (E + gK + 4 * U * logL.abs() + U * lse.abs().nan_to_num(0, 0, 0)) * 1.01
    return o, lse, bound_o, bound_lse, torch.stack(zs, 1)


def _native_kernel(x, n2g, G, qt, heads):
    from ptgnn_b200.reduceops import graph_plan, native_attention_readout

    plan = graph_plan(n2g.cuda(), G)
    o1, l1 = native_attention_readout(x.cuda(), plan, qt.cuda(), heads)
    o2, l2 = native_attention_readout(x.cuda(), plan, qt.cuda(), heads)
    plan.validate()
    assert torch.equal(o1, o2) and torch.equal(l1, l2), "attention readout is not run-to-run bit-identical"
    return o1.double(), l1.double()


def _check(got_o, got_lse, ref_o, ref_lse, bound_o, bound_lse, what):
    err = (got_o - ref_o).abs()
    ratio = float((err / bound_o.clamp(min=1e-300)).max())
    assert bool((err <= bound_o).all()), f"{what}: o error / bound {ratio:.3f}"
    fin = torch.isfinite(ref_lse)
    assert bool((got_lse[~fin] == -math.inf).all()), f"{what}: a graph without nodes must give lse = -inf"
    lerr = (got_lse[fin] - ref_lse[fin]).abs()
    assert bool((lerr <= bound_lse[fin]).all()), f"{what}: lse error / bound {float((lerr / bound_lse[fin]).max()):.3f}"


def _chunk_mutants(x64, n2g, G, z, heads):
    """float64 outputs of two broken kernels: (a) each graph's last partial chunk dropped, (b) in the first graph with several chunks,
    the chunk of smallest maximum combined without its e^{m_c - M} rescale.  None where a layout has no such graph."""
    D = x64.shape[1]
    count = torch.bincount(n2g, minlength=G).tolist()
    order = torch.argsort(n2g, stable=True)
    starts = np.concatenate([[0], np.cumsum(count)])
    dropped = torch.zeros(G, heads, D, dtype=torch.float64, device=x64.device)
    any_partial, rescale = False, None
    for b in range(G):
        nodes = order[starts[b]:starts[b + 1]].to(x64.device)
        if len(nodes) == 0:
            continue
        keep = nodes[:(len(nodes) // CHUNK) * CHUNK] if len(nodes) % CHUNK and len(nodes) > CHUNK else nodes
        any_partial |= len(keep) < len(nodes)
        zk = z[keep]
        p = torch.softmax(zk, 0)
        dropped[b] = torch.einsum("nh,nd->hd", p, x64[keep])
        if rescale is None and len(nodes) > CHUNK:
            zb, xb = z[nodes], x64[nodes]
            M = zb.max(0).values
            parts = []
            for c0 in range(0, len(nodes), CHUNK):
                zc, xc = zb[c0:c0 + CHUNK], xb[c0:c0 + CHUNK]
                m = zc.max(0).values
                e = torch.exp(zc - m)
                parts.append((m, e.sum(0), torch.einsum("nh,nd->hd", e, xc)))
            worst = min(range(len(parts)), key=lambda i: float(parts[i][0].min()))
            num = torch.zeros(heads, D, dtype=torch.float64, device=x64.device)
            den = torch.zeros(heads, dtype=torch.float64, device=x64.device)
            for i, (m, l, acc) in enumerate(parts):
                s = torch.ones_like(m) if i == worst else torch.exp(m - M)
                num += s[:, None] * acc
                den += s * l
            rescale = (b, num / den[:, None])
    return (dropped if any_partial else None), rescale


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("heads", [1, 4, 8])
@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("layout", ["sizes", "one_big", "config2", "unsorted_gaps"])
def test_kernel_against_float64(layout, D, heads, dtype):
    gen = torch.Generator().manual_seed(len(layout) * 1000 + D + heads)
    n2g, G = _n2g_layout(layout, gen)
    x = (torch.randn(n2g.shape[0], D, generator=gen) * 0.5).to(dtype)
    qt = torch.randn(G, heads, D, generator=gen) * (4.0 / D ** 0.5)
    got_o, got_lse = _native_kernel(x, n2g, G, qt, heads)
    x64, n2g_d = x.cuda().double(), n2g.cuda()
    ref_o, ref_lse, bound_o, bound_lse, z = _kernel_ref(x64, n2g_d, G, qt.cuda().double())
    what = f"{layout} D={D} heads={heads} {dtype}"
    _check(got_o, got_lse, ref_o, ref_lse, bound_o, bound_lse, what)
    empty = torch.bincount(n2g, minlength=G) == 0
    assert bool((got_o[empty.cuda()] == 0).all()), "graphs without nodes must be exactly 0"
    # the bound rejects a kernel that drops a graph's last partial chunk, and one that skips a chunk's rescale
    dropped, rescale = _chunk_mutants(x64, n2g_d, G, z, heads)
    if dropped is not None:
        assert not bool(((dropped - ref_o).abs() <= bound_o).all()), f"{what}: the bound does not reject a dropped last chunk"
    if rescale is not None:
        b, mut = rescale
        assert not bool(((mut - ref_o[b]).abs() <= bound_o[b]).all()), f"{what}: the bound does not reject a skipped rescale"


@pytest.mark.parametrize("heads", [1, 4, 8])
@pytest.mark.parametrize("case", ["extreme", "equal"])
def test_kernel_logit_extremes(case, heads):
    """Logits in [-100, 100] with every graph's maximum in its last row (the last chunk's last row), and all-equal logits."""
    D = 64
    gen = torch.Generator().manual_seed(heads)
    n2g, G = _n2g_layout("sizes", gen)
    x = torch.randn(n2g.shape[0], D, generator=gen) * 0.5
    qt = torch.zeros(G, heads, D)
    if case == "extreme":
        for h in range(heads):
            qt[:, h, h] = 1.0                       # z_{n,h} = x_n[h]
        x[:, :heads] = torch.rand(n2g.shape[0], heads, generator=gen) * 200 - 100
        last = torch.cumsum(torch.bincount(n2g, minlength=G), 0) - 1
        x[last, :heads] = 100.0
    got_o, got_lse = _native_kernel(x, n2g, G, qt, heads)
    assert bool(torch.isfinite(got_o).all() and torch.isfinite(got_lse).all()), "non-finite output"
    ref = _kernel_ref(x.cuda().double(), n2g.cuda(), G, qt.cuda().double())
    _check(got_o, got_lse, *ref[:4], f"{case} heads={heads}")


# ---- modules ----------------------------------------------------------------------------------------------------------------
def _module(kind, D, hidden, out, heads, value, query, seed):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    q = P.WeightedSumVarSizedElementReduce(D) if query == "weighted" else P.SimpleVarSizedElementReduce(query)
    if kind == "self":
        return P.SelfAttentionVarSizedElementReduce(D, hidden, out, q)
    return P.MultiheadSelfAttentionVarSizedElementReduce(D, hidden, out, heads, q, use_value_layer=value)


def _restated(module, x, n2g, G, params=None):
    """The float64 restatement with the module's parameters (``params``: name -> tensor, by default the module's, in float64)."""
    import ptgnn_b200 as P

    sd = params if params is not None else {k: v.detach().cpu().double() for k, v in module.state_dict().items()}
    self_attn = isinstance(module, P.SelfAttentionVarSizedElementReduce)
    p = "_SelfAttentionVarSizedElementReduce__" if self_attn else "_MultiheadSelfAttentionVarSizedElementReduce__"
    query = module._SelfAttentionVarSizedElementReduce__query_layer if self_attn else module._MultiheadSelfAttentionVarSizedElementReduce__query_layer
    if isinstance(query, P.WeightedSumVarSizedElementReduce):
        queries = GX.graph_readout(x, n2g, G, "weighted", sd[p + "query_layer._WeightedSumVarSizedElementReduce__weights_layer.weight"])
    else:
        queries = GX.graph_readout(x, n2g, G, query._SimpleVarSizedElementReduce__summarization_type)
    if self_attn:
        return AR.self_attention_forward(x, n2g, G, queries, sd[p + "key_layer.weight"], sd[p + "output_layer.weight"])
    heads = module._MultiheadSelfAttentionVarSizedElementReduce__num_heads
    return AR.multihead_self_attention_forward(x, n2g, G, queries, sd[p + "key_layer.weight"], heads, sd[p + "output_layer.weight"],
                                               sd.get(p + "value_layer.weight"))


def _call(module, x, n2g, G):
    from ptgnn_b200 import ElementsToSummaryRepresentationInput as In

    return module(In(x, n2g, G))


def _twice(module, x, n2g, G):
    with torch.no_grad():
        a = _call(module, x.cuda(), n2g.cuda(), G)
        b = _call(module, x.cuda(), n2g.cuda(), G)
    assert torch.equal(a, b), "module output is not run-to-run bit-identical"
    return a.float().cpu()


def _graphs(N, gen, per_graph=500):
    G = max(1, (N + per_graph - 1) // per_graph)
    n2g = torch.randint(0, G, (N,), generator=gen)
    return n2g, int(n2g.max()) + 1


# (class, D, hidden, output size, heads, value layer, query summarizer); the Simple and WeightedSum queries are D wide, so hidden = D
MODULE_CASES = [("multi", 256, 256, 128, 8, False, "max"), ("multi", 64, 64, 32, 1, False, "max"), ("multi", 64, 64, 32, 1, True, "mean"),
                ("multi", 128, 128, 64, 4, True, "weighted"), ("multi", 128, 128, 64, 4, False, "sum"), ("self", 64, 64, 32, 1, False, "weighted"),
                ("self", 256, 256, 64, 1, False, "min")]


@pytest.mark.parametrize("case", MODULE_CASES, ids=lambda c: "-".join(map(str, c)))
def test_module_fp32_against_float64(case):
    kind, D, hidden, out, heads, value, query = case
    gen = torch.Generator().manual_seed(D + hidden + heads)
    n2g, G = _graphs(5000, gen)
    x = torch.randn(5000, D, generator=gen) * 0.5
    module = _module(kind, D, hidden, out, heads, value, query, D + heads).cuda().eval()
    assert_close(_twice(module, x, n2g, G), _restated(module, x.double(), n2g, G), tol=1e-5, what=f"{case}")


@pytest.mark.parametrize("name", ["attn_mh1", "attn_mh1_value", "attn_mh4", "attn_mh4_value", "attn_mh8", "attn_mh8_value", "attn_self_weighted"])
def test_module_fp32_vs_reference_golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    D, heads, value = z["x"].shape[1], int(z["heads"]), bool(z["value"])
    kind = "self" if str(z["cls"]) == "self" else "multi"
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    hidden = sd[next(k for k in sd if k.endswith("key_layer.weight"))].shape[0]
    out = sd[next(k for k in sd if k.endswith("output_layer.weight"))].shape[0]
    module = _module(kind, D, hidden, out, heads, value, str(z["query"]), 0)
    module.load_state_dict(sd)
    n2g = torch.from_numpy(z["n2g"])
    got = _twice(module.cuda().eval(), torch.from_numpy(z["x"]), n2g, int(n2g.max()) + 1)
    assert_close(got, torch.from_numpy(z["out"]), tol=1e-5, what=name)
    assert bool((got[3] == 0).all()), "the graph without nodes gives 0"


def test_module_bf16_vs_reference_autocast():
    """DESIGN §4 bf16 rule: rel. L2 <= 1e-2 against the reference's autocast output, and at least as close to the fp32 result as the
    reference's autocast path is."""
    z = np.load(os.path.join(GOLDEN, "attn_mh8_bf16ac.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    D = z["x"].shape[1]
    module = _module("multi", D, D, sd["_MultiheadSelfAttentionVarSizedElementReduce__output_layer.weight"].shape[0], int(z["heads"]),
                     False, str(z["query"]), 0)
    module.load_state_dict(sd)
    n2g = torch.from_numpy(z["n2g"])
    got = _twice(module.cuda().eval(), torch.from_numpy(z["x"]).to(torch.bfloat16), n2g, int(n2g.max()) + 1)
    ref_ac, ref32 = torch.from_numpy(z["out_autocast"]), torch.from_numpy(z["out_fp32_rounded_inputs"])
    scale = ref32.abs().clamp(min=1)
    err_ours, err_ref = (got - ref32).abs(), (ref_ac - ref32).abs()
    frac_ours, frac_ref = (err_ours <= 1e-2 * scale).float().mean().item(), (err_ref <= 1e-2 * scale).float().mean().item()
    rel_ac = ((got - ref_ac).norm() / ref_ac.norm()).item()
    msg = f"rel L2 vs autocast {rel_ac:.2e}; mean err ours {err_ours.mean():.2e} / ref {err_ref.mean():.2e}; within 1e-2 {frac_ours:.4f} / {frac_ref:.4f}"
    assert rel_ac <= 1e-2 and err_ours.mean().item() <= 1.1 * err_ref.mean().item() and frac_ours >= frac_ref - 0.002, msg


def test_module_errors():
    import ptgnn_b200 as P

    x, n2g = torch.randn(100, 64).cuda(), torch.zeros(100, dtype=torch.int64).cuda()
    bad_query = P.MultiheadSelfAttentionVarSizedElementReduce(64, 32, 16, 4, P.SimpleVarSizedElementReduce("max")).cuda()
    with torch.no_grad(), pytest.raises(ValueError, match="hidden_size"):
        _call(bad_query, x, n2g, 1)                              # the max query is 64 wide, the key layer 32
    odd = P.MultiheadSelfAttentionVarSizedElementReduce(48, 48, 16, 3, P.SimpleVarSizedElementReduce("max")).cuda()
    with torch.no_grad(), pytest.raises(NotImplementedError):
        _call(odd, torch.randn(100, 48).cuda(), n2g, 1)
    m = P.MultiheadSelfAttentionVarSizedElementReduce(64, 64, 16, 4, P.SimpleVarSizedElementReduce("max")).cuda()
    with pytest.raises(NotImplementedError):
        _call(m, x.to(torch.bfloat16).requires_grad_(True), n2g, 1)


def test_module_makes_no_host_synchronisation():
    gen = torch.Generator().manual_seed(5)
    n2g, G = _graphs(20_000, gen)
    x, n2g_d = (torch.randn(20_000, 256, generator=gen) * 0.5).cuda(), n2g.cuda()
    for query, value in (("max", False), ("weighted", True)):
        m = _module("multi", 256, 256, 128, 8, value, query, 1).cuda()
        xg = x.clone().requires_grad_(True)
        for grad in (False, True):
            with torch.set_grad_enabled(grad):
                _call(m, xg, n2g_d, G)                            # warm: plan cache
                torch.cuda.synchronize()
                torch.cuda.set_sync_debug_mode("error")
                try:
                    _call(m, xg, n2g_d, G)
                finally:
                    torch.cuda.set_sync_debug_mode("default")


def test_module_peak_memory_at_graph2seq_shape():
    """80 x 2,560 nodes, D = 256, 8 heads: the call's peak-memory increase stays below one [N, D] fp32 tensor (the reference's
    [N, heads * D] product alone is 8 of them)."""
    n2g = torch.repeat_interleave(torch.arange(80), 2560).cuda()
    x = torch.randn(n2g.shape[0], 256, device="cuda") * 0.5
    m = _module("multi", 256, 256, 128, 8, False, "max", 2).cuda()
    with torch.no_grad():
        _call(m, x, n2g, 80)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        _call(m, x, n2g, 80)
        torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    assert rise < x.numel() * 4, f"peak rise {rise / 2**20:.1f} MiB >= one [N, D] fp32 tensor ({x.numel() * 4 / 2**20:.1f} MiB)"


# ---- training -------------------------------------------------------------------------------------------------------------
def _grads_close(a, b, what):
    """The bar of test_gpu_backward.py: max error over max(1, max |ref|), and rel. L2, both <= 1e-4."""
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    scaled = (a - b).abs().max().item() / max(1.0, b.abs().max().item())
    rel = ((a - b).norm() / b.norm().clamp(min=1e-30)).item()
    assert scaled <= 1e-4 and rel <= 1e-4, f"{what}: scaled {scaled:.2e} rel L2 {rel:.2e}"


def _native_grads(module, x, n2g, G, grad_out):
    module.zero_grad()
    xd = x.cuda().requires_grad_(True)
    _call(module, xd, n2g.cuda(), G).backward(grad_out.cuda())
    return [xd.grad.clone()] + [p.grad.clone() for _, p in module.named_parameters()]


TRAIN_CASES = [("multi", 64, 64, 32, 4, True, "weighted"), ("multi", 128, 128, 64, 8, False, "max"), ("multi", 64, 64, 32, 1, False, "mean"),
               ("self", 64, 64, 32, 1, False, "weighted")]


@pytest.mark.parametrize("case", TRAIN_CASES, ids=lambda c: "-".join(map(str, c)))
def test_backward_against_autograd(case):
    kind, D, hidden, out, heads, value, query = case
    N = 3000
    gen = torch.Generator().manual_seed(41 + heads)
    n2g, G = _graphs(N, gen, 400)
    x = torch.randn(N, D, generator=gen) * 0.5
    module = _module(kind, D, hidden, out, heads, value, query, 42).cuda().train()
    grad_out = torch.randn(G, out, generator=gen)
    first = _native_grads(module, x, n2g, G, grad_out)
    again = _native_grads(module, x, n2g, G, grad_out)
    assert all(torch.equal(a, b) for a, b in zip(first, again)), "gradients are not run-to-run bit-identical"

    x64 = x.double().requires_grad_(True)
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in module.named_parameters()}
    _restated(module, x64, n2g, G, sd).backward(grad_out.double())
    _grads_close(first[0], x64.grad, f"{case} d x")
    for (name, _), g in zip(module.named_parameters(), first[1:]):
        _grads_close(g, sd[name].grad, f"{case} d {name}")


def test_graph2seq_encoder_two_sgd_steps_match_cpu():
    """graph2seq's summary (graph2seq.py:55-65, 116-122): gated layers at H = 128, the concatenation of the input and output node states,
    then the native 8-head reducer with a max query; two SGD steps against the same steps in float64 on the CPU."""
    import ptgnn_b200 as P

    N, H, T, G = 2000, 128, 2, 8
    gen = torch.Generator().manual_seed(51)
    adj = [(torch.randint(0, N, (c,), generator=gen), torch.randint(0, N, (c,), generator=gen)) for c in (2 * N, N)]
    n2g = torch.sort(torch.randint(0, G, (N,), generator=gen)).values
    h0 = torch.randn(N, H, generator=gen) * 0.5
    torch.manual_seed(52)
    layers = [P.GatedMessagePassingLayer(H, H, T, "sum").cuda(), P.GatedMessagePassingLayer(H, H, T, "sum").cuda()]
    reducer = _module("multi", 2 * H, 2 * H, H, 8, False, "max", 53).cuda()
    modules = layers + [reducer]
    params = [p for m in modules for p in m.parameters()]
    ref_params = [p.detach().cpu().double().clone().requires_grad_(True) for p in params]
    target = torch.randn(G, H, generator=torch.Generator().manual_seed(54))
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    opt = torch.optim.SGD(params, lr=0.05)
    for _ in range(2):
        opt.zero_grad()
        h = h0.cuda()
        for layer in layers:
            h = layer(h, adj_d)
        out = _call(reducer, torch.cat((h0.cuda(), h), dim=-1), n2g.cuda(), G)
        ((out - target.cuda()) ** 2).mean().backward()
        opt.step()

    def run_cpu():
        it = iter(ref_params)
        h = h0.double()
        for layer in layers:
            names = {n: next(it) for n, _ in layer.named_parameters()}
            h = O.gated_layer_forward(h, adj, [torch.empty(s.shape[0], 0, dtype=torch.float64) for s, _ in adj], aggregation_fn="sum",
                                      **gated_oracle_args(names))
        names = {n: next(it) for n, _ in reducer.named_parameters()}
        return _restated(reducer, torch.cat((h0.double(), h), dim=-1), n2g, G, names)

    ref_opt = torch.optim.SGD(ref_params, lr=0.05)
    for _ in range(2):
        ref_opt.zero_grad()
        ((run_cpu() - target.double()) ** 2).mean().backward()
        ref_opt.step()
    for p, r in zip(params, ref_params):
        _grads_close(p, r, "parameters after two SGD steps")


def test_global_gru_update_with_native_multihead_reducer_trains():
    import ptgnn_b200 as P

    N, H = 3000, 64
    gen = torch.Generator().manual_seed(61)
    n2g, G = _graphs(N, gen, 400)
    h = torch.randn(N, H, generator=gen) * 0.5
    torch.manual_seed(62)
    reducer = P.MultiheadSelfAttentionVarSizedElementReduce(H, H, H, 4, P.SimpleVarSizedElementReduce("mean"), use_value_layer=True)
    layer = P.GruGlobalStateUpdate(reducer, H, H).cuda().train()
    hd = h.cuda().requires_grad_(True)
    grad_out = torch.randn(N, H, generator=gen)
    layer(hd, [], n2g.cuda(), {}, {}, []).backward(grad_out.cuda())

    h64 = h.double().requires_grad_(True)
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in layer.named_parameters()}
    pr = "_AbstractGlobalGraphExchange__global_graph_representation_module."
    g = _restated(reducer, h64, n2g, G, {k[len(pr):]: v for k, v in sd.items() if k.startswith(pr)})
    ref = O.gru_cell(g[n2g], h64, *(sd["_GruGlobalStateUpdate__gru_cell." + k] for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")))
    ref.backward(grad_out.double())
    _grads_close(hd.grad, h64.grad, "d h")
    for name, param in layer.named_parameters():
        _grads_close(param.grad, sd[name].grad, f"d {name}")
