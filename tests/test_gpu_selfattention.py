"""MultiHeadSelfAttentionMessagePassing on the GPU: the chunked attention kernel against float64 element by element under the bound of
DESIGN.md §4 (selfattention_reference.bound), the layer against the float64 restatement and the reference's fixtures, bf16 against the
reference's autocast fixture, gradients against torch.autograd through the float64 restatement, run-to-run identity, no host
synchronisation with the graph count handed in, CUDA-graph capture inside a container, the unsupported cases, and the backward kernels
(native_selfatt_backward) against float64 element by element under selfattention_reference.backward_bound, with backward(2^k dO) = 2^k
backward(dO)."""
import os

import numpy as np
import pytest
import torch

import selfattention_reference as SR
from helpers import assert_close

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["selfatt_h1_d16", "selfatt_h3_d32", "selfatt_h8_d16", "selfatt_h4_dk64_dv32", "selfatt_h2_dk128_dv64"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    f = {k: int(z[k]) if z[k].ndim == 0 else torch.from_numpy(z[k]) for k in z.files}
    f["sd"] = {k[4:]: v for k, v in f.items() if k.startswith("sd::")}
    return f


def layer_of(f):
    import ptgnn_b200 as P

    m = P.MultiHeadSelfAttentionMessagePassing(f["in_dim"], f["dk"], f["dv"], f["out_dim"], f["inter"], f["heads"],
                                               max_num_nodes=f["max_num_nodes"])
    m.load_state_dict(f["sd"], strict=True)
    return m.cuda().eval()


def kernel(t, n2g, G, heads, dk, dv, L):
    from ptgnn_b200.reduceops import graph_plan
    from ptgnn_b200.selfattention import native_selfatt

    plan = graph_plan(n2g, G)
    runs = [native_selfatt(t, plan, heads, dk, dv, L) for _ in range(2)]
    plan.validate()
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]), "two runs differ"
    return runs[0]


def check_bound(t32, n2g, heads, dk, dv, L, what):
    G = int(n2g.max()) + 1
    o, lse = kernel(t32, n2g, G, heads, dk, dv, L)
    exact = SR.attention(t32.double(), n2g, heads, dk, L)
    bnd = SR.bound(t32, n2g, heads, dk, L)
    err = (o.double() - exact).abs()
    bad = int((err > bnd).sum())
    assert bad == 0, f"{what}: {bad} elements over the bound (worst ratio {float((err / bnd).max()):.2f})"
    return o, lse, exact


@pytest.mark.parametrize("name", NAMES)
def test_kernel_against_float64(name):
    f = load(name)
    n2g = f["n2g"].cuda()
    t = torch.nn.functional.linear(f["x"].double(), f["sd"][SR.PREFIX + "selfatt_head_transforms.weight"].double()).float().cuda()
    _, lse, _ = check_bound(t, n2g, f["heads"], f["dk"], f["dv"], f["max_num_nodes"], name)
    a, b, _ = SR.split_heads(t.double(), f["heads"], f["dk"])
    ref = []
    for s, e in SR.chunks(n2g, f["max_num_nodes"]):
        ref.append(torch.logsumexp(torch.einsum("khd,vhd->khv", a[s:e], b[s:e]) / f["dk"] ** 0.5, dim=-1))
    ref = torch.cat(ref)
    assert float(((lse.double() - ref).abs() / ref.abs().clamp(min=1)).max()) <= 1e-5


@pytest.mark.parametrize("dk,dv", [(16, 128), (128, 128), (32, 16), (64, 64)])
@pytest.mark.parametrize("L", [1, 63, 250])
def test_kernel_other_shapes(dk, dv, L):
    gen = torch.Generator().manual_seed(dk * 1000 + dv + L)
    heads = 3
    n2g = torch.repeat_interleave(torch.arange(5), torch.tensor([300, 1, 0, 129, 64]))
    t = torch.randn(n2g.numel(), heads * (2 * dk + dv), generator=gen)
    check_bound(t.cuda(), n2g.cuda(), heads, dk, dv, L, f"dk={dk} dv={dv} L={L}")


@pytest.mark.parametrize("case", ["max_in_last_block", "all_equal"])
def test_kernel_logit_extremes(case):
    heads, dk, dv, L = 2, 16, 16, 250
    n = 250 + 130                                   # one full chunk (four key blocks, the last partial) and a partial one
    gen = torch.Generator().manual_seed(7)
    t = torch.zeros(n, heads, 2 * dk + dv)
    t[:, :, 2 * dk:] = torch.randn(n, heads, dv, generator=gen)
    if case == "max_in_last_block":                 # s_ij = a_i0 b_j0 / 4 = +-80; the maximum sits in the chunk's last key block
        t[:, :, 0] = 4.0
        t[:, :, dk] = -80.0
        t[249, :, dk] = 80.0
        t[n - 1, :, dk] = 80.0
    t = t.reshape(n, -1).cuda()
    n2g = torch.zeros(n, dtype=torch.int64, device="cuda")
    o, lse, exact = check_bound(t, n2g, heads, dk, dv, L, case)
    if case == "all_equal":
        mean = torch.cat([t[s:e].double().reshape(e - s, heads, -1)[:, :, 2 * dk:].mean(0, keepdim=True).expand(e - s, -1, -1)
                          for s, e in ((0, 250), (250, n))]).reshape(n, -1)
        assert float((o.double() - mean).abs().max()) <= 1e-6
    else:
        assert float((lse.double() - 80.0).abs().max()) <= 1e-4


def test_kernel_more_ctas_than_one_wave():
    heads, dk, dv, L = 8, 16, 16, 250
    n2g = torch.repeat_interleave(torch.arange(80), 2560).cuda()       # 204,800 nodes: 880 chunks, 3,520 tiles per head
    gen = torch.Generator(device="cuda").manual_seed(11)
    t = torch.randn(n2g.numel(), heads * (2 * dk + dv), generator=gen, device="cuda")
    check_bound(t, n2g, heads, dk, dv, L, "204,800 nodes")


def test_kernel_bf16():
    f = load("selfatt_h8_d16")
    n2g = f["n2g"].cuda()
    t = torch.nn.functional.linear(f["x"], f["sd"][SR.PREFIX + "selfatt_head_transforms.weight"]).cuda()
    o, _ = kernel(t.to(torch.bfloat16), n2g, int(n2g.max()) + 1, f["heads"], f["dk"], f["dv"], f["max_num_nodes"])
    ref = SR.attention(t.to(torch.bfloat16).double(), n2g, f["heads"], f["dk"], f["max_num_nodes"])
    assert o.dtype == torch.bfloat16
    assert float((o.double() - ref).norm() / ref.norm()) <= 1e-2


def _twice(layer, x, n2g):
    with torch.no_grad():
        a = layer(x, [], n2g, {}, {}, [])
        b = layer(x, [], n2g, {}, {}, [])
    assert torch.equal(a, b), "two runs differ"
    return a


@pytest.mark.parametrize("name", NAMES)
def test_layer_fp32_against_float64_and_reference_golden(name):
    f = load(name)
    got = _twice(layer_of(f), f["x"].cuda(), f["n2g"].cuda())
    ref = SR.layer_forward(f["x"].double(), f["n2g"], {k: v.double() for k, v in f["sd"].items()}, f["heads"], f["dk"], f["max_num_nodes"])
    assert_close(got, ref, 1e-5, f"{name} vs float64")
    assert_close(got, f["out"], 1e-5, f"{name} vs reference")


def test_layer_bf16_vs_reference_autocast():
    """DESIGN §4 bf16 rule: rel. L2 <= 1e-2 against the reference's autocast output, and at least as close to the fp32 result as the
    reference's autocast path is.  The layer returns bf16 for bf16 states while the autocast LayerNorm returns fp32, so the autocast
    output is compared after the same final rounding to bf16."""
    f = load("selfatt_h8_d16_bf16ac")
    got = _twice(layer_of(f), f["x"].cuda().to(torch.bfloat16), f["n2g"].cuda())
    assert got.dtype == torch.bfloat16
    got = got.cpu().float()
    ref32, ref_ac = f["out_fp32_rounded_inputs"], f["out_autocast"].to(torch.bfloat16).float()
    scale = ref32.abs().clamp(min=1)
    err_ours, err_ref = (got - ref32).abs(), (ref_ac - ref32).abs()
    frac_ours, frac_ref = (err_ours <= 1e-2 * scale).float().mean().item(), (err_ref <= 1e-2 * scale).float().mean().item()
    rel_ac = ((got - f["out_autocast"]).norm() / f["out_autocast"].norm()).item()
    msg = f"rel L2 vs autocast {rel_ac:.2e}; mean err ours {err_ours.mean():.2e} / ref {err_ref.mean():.2e}; within 1e-2 {frac_ours:.4f} / {frac_ref:.4f}"
    assert rel_ac <= 1e-2 and err_ours.mean().item() <= 1.1 * err_ref.mean().item() and frac_ours >= frac_ref - 0.002, msg


@pytest.mark.parametrize("name", ["selfatt_h3_d32", "selfatt_h2_dk128_dv64"])
def test_backward_against_autograd(name):
    f = load(name)
    layer = layer_of(f).train()
    x = f["x"].cuda().requires_grad_(True)
    n2g = f["n2g"].cuda()
    gen = torch.Generator().manual_seed(3)
    g = torch.randn(x.shape[0], f["out_dim"], generator=gen)
    out = layer(x, [], n2g, {}, {}, [])
    out.backward(g.cuda())
    sd64 = {k: v.double().requires_grad_(True) for k, v in f["sd"].items()}
    x64 = f["x"].double().requires_grad_(True)
    SR.layer_forward(x64, f["n2g"], sd64, f["heads"], f["dk"], f["max_num_nodes"]).backward(g.double())
    pairs = [("d node_states", x.grad, x64.grad)] + [(n, p.grad, sd64[n].grad) for n, p in layer.named_parameters()]
    assert len(pairs) == 11
    for what, got, ref in pairs:
        got = got.cpu().double()
        scale = ref.abs().max().clamp(min=1e-30)
        assert float((got - ref).abs().max() / scale) <= 1e-4, f"{name} {what}: scaled max error"
        assert float((got - ref).norm() / ref.norm().clamp(min=1e-30)) <= 1e-4, f"{name} {what}: rel. L2 error"
    # a second backward is bit-identical
    grads = [p.grad.clone() for p in layer.parameters()] + [x.grad.clone()]
    layer.zero_grad()
    x.grad = None
    layer(x, [], n2g, {}, {}, []).backward(g.cuda())
    assert all(torch.equal(a, b) for a, b in zip(grads, [p.grad for p in layer.parameters()] + [x.grad]))


def test_layer_makes_no_host_synchronisation_with_the_count_handed_in():
    from ptgnn_b200.edgeplan import shared_num_graphs

    f = load("selfatt_h1_d16")
    layer = layer_of(f)
    x, n2g = f["x"].cuda(), f["n2g"].cuda()
    G = int(f["n2g"].max()) + 1
    with torch.no_grad():
        layer(x, [], n2g, {}, {}, [])
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            with shared_num_graphs(G):
                layer(x, [], n2g, {}, {}, [])
        finally:
            torch.cuda.set_sync_debug_mode("default")


def test_container_eager_equals_captured_replay():
    import ptgnn_b200 as P

    class _Embed(torch.nn.Module):
        def forward(self, x):
            return x

    H, N, T = 64, 3000, 2
    torch.manual_seed(4)
    layers = [P.GatedMessagePassingLayer(H, H, T, "sum"), P.MultiHeadSelfAttentionMessagePassing(H, 16, 16, H, 128, 4, max_num_nodes=100),
              P.GatedMessagePassingLayer(H, H, T, "sum")]
    gnn = P.GraphNeuralNetwork(layers, _Embed(), False, False).cuda().eval()
    gen = torch.Generator().manual_seed(5)
    adj = [(torch.randint(0, N, (c,), generator=gen).cuda(), torch.randint(0, N, (c,), generator=gen).cuda()) for c in (2 * N, N)]
    n2g = torch.sort(torch.randint(0, 12, (N,), generator=gen)).values.cuda()
    h = (torch.randn(N, H, generator=gen) * 0.5).cuda()
    G = int(n2g.max()) + 1
    with torch.no_grad():
        eager = gnn.gnn(h, adj, None, n2g, {}, {}, num_graphs=G)
    graphed = gnn.capture(h.clone(), adj, n2g, num_graphs=G)
    assert torch.equal(graphed.replay(), eager), "captured replay differs from the eager run"


def test_unsupported_cases_raise():
    import ptgnn_b200 as P

    x = torch.randn(10, 32, device="cuda")
    n2g = torch.zeros(10, dtype=torch.int64, device="cuda")
    with pytest.raises(NotImplementedError):
        P.MultiHeadSelfAttentionMessagePassing(32, 24, 16, 32, 64, 2).cuda().eval()(x, [], n2g, {}, {}, [])
    with pytest.raises(NotImplementedError):
        P.MultiHeadSelfAttentionMessagePassing(32, 16, 16, 32, 64, 2, target_reference="tok").cuda().eval()(x, [], n2g, {}, {}, [])
    with pytest.raises(NotImplementedError):
        P.MultiHeadSelfAttentionMessagePassing(32, 16, 16, 32, 64, 2, dropout_rate=0.1).cuda().train()(x, [], n2g, {}, {}, [])
    with pytest.raises(NotImplementedError):
        P.MultiHeadSelfAttentionMessagePassing(32, 16, 16, 32, 64, 2).cuda()(x.bfloat16().requires_grad_(True), [], n2g, {}, {}, [])
    with pytest.raises(NotImplementedError):
        P.MultiHeadSelfAttentionMessagePassing(32, 16, 16, 32, 64, 2).cuda().eval()(x, [], n2g, {}, {}, [], gather_states=x)
    with torch.no_grad():       # eval mode with p > 0 is the identity and runs
        P.MultiHeadSelfAttentionMessagePassing(32, 16, 16, 32, 64, 2, dropout_rate=0.1).cuda().eval()(x, [], n2g, {}, {}, [])


# ---- backward kernels, element by element ------------------------------------------------------------------------------------
SCALES = (-37, -27, -17, 17)        # the gradient magnitudes of test_gpu_backward_edges.py: backward(2^k dO) = 2^k backward(dO)
PAIRS = [(dk, dv) for dk in (16, 32, 64, 128) for dv in (16, 32, 64, 128)]
SIZES = [0, 1, 63, 64, 65, 250, 251, 1000]


def bwd_map(kind, seed):
    """(n2g, G): the sizes in graph order, or shuffled with an empty graph in between and two trailing empty graphs."""
    if kind == "sorted":
        return torch.repeat_interleave(torch.arange(len(SIZES)), torch.tensor(SIZES)), len(SIZES)
    counts = SIZES[1:4] + [0] + SIZES[4:] + [0, 0]
    n2g = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    return n2g[torch.randperm(n2g.numel(), generator=torch.Generator().manual_seed(seed))], len(counts)


def check_backward(t, n2g, G, heads, dk, dv, L, what, scales=SCALES):
    """native_selfatt_backward twice (bit-identical) on the forward kernel's o and lse, against backward_formula under backward_bound
    (float64 on the GPU), and backward(2^k dO) = 2^k backward(dO) bit for bit for k in ``scales``.  Returns the worst err / bound."""
    from ptgnn_b200.reduceops import graph_plan
    from ptgnn_b200.selfattention import native_selfatt, native_selfatt_backward

    t, n2g = t.cuda(), n2g.cuda()
    plan = graph_plan(n2g, G)
    o, lse = native_selfatt(t, plan, heads, dk, dv, L)
    gen = torch.Generator(device="cuda").manual_seed(t.shape[0] + dk + dv + L)
    d_o = torch.randn(t.shape[0], heads * dv, generator=gen, device="cuda")
    runs = [native_selfatt_backward(t, plan, heads, dk, dv, L, o, lse, d_o) for _ in range(2)]
    plan.validate()
    assert torch.equal(runs[0], runs[1]), f"{what}: two backward runs differ"
    got = runs[0]
    ref = SR.backward_formula(t, o, lse, d_o, n2g.cpu(), heads, dk, L)
    bnd = SR.backward_bound(t, o, lse, d_o, n2g.cpu(), heads, dk, L)
    err = (got.double() - ref).abs()
    bad = int((err > bnd).sum())
    ratio = float((err / bnd).max())
    assert bad == 0, f"{what}: {bad} elements over the bound (worst ratio {ratio:.2f})"
    for k in scales:
        assert torch.equal(native_selfatt_backward(t, plan, heads, dk, dv, L, o, lse, d_o * 2.0 ** k), got * 2.0 ** k), \
            f"{what}: backward(2^{k} dO) != 2^{k} backward(dO)"
    return ratio


@pytest.mark.parametrize("kind", ["sorted", "unsorted"])
@pytest.mark.parametrize("dk,dv", PAIRS)
def test_backward_kernels_every_instance(dk, dv, kind):
    n2g, G = bwd_map(kind, dk + dv)
    t = torch.randn(n2g.numel(), 3 * (2 * dk + dv), generator=torch.Generator().manual_seed(dk * 7 + dv))
    check_backward(t, n2g, G, 3, dk, dv, 250, f"dk={dk} dv={dv} {kind}")


@pytest.mark.parametrize("kind", ["sorted", "unsorted"])
@pytest.mark.parametrize("L", [1, 16, 63, 64, 65, 1000])
def test_backward_kernels_chunk_lengths(L, kind):
    """L = 1000 holds the largest graph in one chunk; 250 runs in test_backward_kernels_every_instance."""
    n2g, G = bwd_map(kind, L)
    t = torch.randn(n2g.numel(), 3 * (2 * 64 + 32), generator=torch.Generator().manual_seed(L))
    check_backward(t, n2g, G, 3, 64, 32, L, f"L={L} {kind}")


@pytest.mark.parametrize("L", [2, 250])
def test_backward_kernels_more_graphs_than_one_scan_block(L):
    """3,000 graphs of 0 to 5 rows: the tile scan (pergraph::item_ptr_kernel) carries its sum over three blocks of 1,024 graphs."""
    gen = torch.Generator().manual_seed(L)
    counts = torch.randint(0, 6, (3000,), generator=gen)
    n2g = torch.repeat_interleave(torch.arange(3000), counts)
    t = torch.randn(n2g.numel(), 3 * (2 * 16 + 16), generator=gen)
    check_backward(t, n2g, 3000, 3, 16, 16, L, f"3,000 graphs L={L}")


def test_backward_kernels_graph2seq_shape():
    n2g = torch.repeat_interleave(torch.arange(80), 2560)        # 204,800 rows, 880 chunks of at most 250 rows, 8 heads
    t = torch.randn(n2g.numel(), 8 * (2 * 16 + 16), generator=torch.Generator().manual_seed(80))
    check_backward(t, n2g, 80, 8, 16, 16, 250, "80 x 2,560")


@pytest.mark.parametrize("case", ["max_in_last_block", "all_equal"])
def test_backward_kernels_logit_extremes(case):
    """The forward test's logits: +-80 with the maximum in the chunk's last key block (p down to e^-160, below float32's range, so the
    bound alone: scaled products can be subnormal), and all-equal logits."""
    heads, dk, dv, L = 2, 16, 16, 250
    n = 250 + 130
    gen = torch.Generator().manual_seed(8)
    t = torch.zeros(n, heads, 2 * dk + dv)
    t[:, :, 2 * dk:] = torch.randn(n, heads, dv, generator=gen)
    if case == "max_in_last_block":
        t[:, :, 0] = 4.0
        t[:, :, dk] = -80.0
        t[249, :, dk] = 80.0
        t[n - 1, :, dk] = 80.0
    check_backward(t.reshape(n, -1), torch.zeros(n, dtype=torch.int64), 1, heads, dk, dv, L, case,
                   scales=() if case == "max_in_last_block" else SCALES)


def test_backward_parametrisation_reaches_every_instance():
    assert len(set(PAIRS)) == 16, "selfatt_bwd_kv_kernel / selfatt_bwd_q_kernel<DK, DV>: 16 instances each"
