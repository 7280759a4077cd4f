"""GraphNorm on the GPU: the kernels against the float32 emulation of their order bit for bit and against float64 element by element
under the bound of DESIGN.md §4 (graphnorm_reference.bound), the layer against the reference's fixtures, bf16 under the bf16 rule,
gradients against torch.autograd through the float64 restatement, run-to-run identity, no host synchronisation with the graph count
handed in, CUDA-graph capture inside a container, the unsupported cases, and the backward kernels (native_graph_norm_backward) against
emulate_backward bit for bit and against float64 under graphnorm_reference.backward_bound, with backward(2^k dy) = 2^k backward(dy)."""
import os

import numpy as np
import pytest
import torch

import graphnorm_reference as GR
from helpers import TOL, assert_close

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["graphnorm_d32", "graphnorm_d64", "graphnorm_d128", "graphnorm_d256"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    f = {k: torch.from_numpy(z[k]) for k in z.files}
    f["sd"] = {k[4:]: v for k, v in f.items() if k.startswith("sd::")}
    return f


def layer_of(f):
    import ptgnn_b200 as P

    m = P.GraphNorm(f["x"].shape[1])
    m.load_state_dict(f["sd"], strict=True)
    return m.cuda()


def params(D, seed):
    gen = torch.Generator().manual_seed(seed)
    return 1.0 + 0.5 * torch.randn(1, D, generator=gen), torch.rand(1, D, generator=gen) * 1.5, 0.3 * torch.randn(1, D, generator=gen)


def kernel(x, n2g, G, gamma, alpha, bias):
    """Two NaN-prefilled runs of the forward kernels, which must agree bit for bit: (y, mean, rstd) on the CPU."""
    from ptgnn_b200.graphnorm import native_graph_norm
    from ptgnn_b200.reduceops import graph_plan

    plan = graph_plan(n2g, G)
    runs = []
    for _ in range(2):
        out = torch.full_like(x, float("nan"))
        runs.append(native_graph_norm(x, plan, gamma.cuda(), alpha.cuda(), bias.cuda(), 1e-10, out=out))
    plan.validate()
    assert all(torch.equal(a, b) for a, b in zip(*runs)), "two runs differ"
    assert not bool(runs[0][0].isnan().any()), "unwritten output elements"
    return [t.cpu() for t in runs[0]]


# (counts per graph id, D, shuffle): the issue's shapes plus edges of the chunking (1 row, 31 / 32 / 33 rows, a graph id without nodes)
SHAPES = {
    "80x2560_d128": ([2560] * 80, 128, False),
    "40x2000_d64": ([2000] * 40, 64, True),
    "one_graph_204800_d128": ([204800], 128, False),
    "10000x20_d32": ([20] * 10000, 32, True),
    "edges_d96": ([1, 31, 32, 33, 0, 1, 64, 65, 1000], 96, True),
    "edges_d256": ([3, 0, 1, 97, 32], 256, True),
    "edges_d160": ([129, 1, 2, 0, 0, 40], 160, True),
}


def graph_map(counts, shuffle, seed):
    gen = torch.Generator().manual_seed(seed)
    n2g = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    return n2g[torch.randperm(n2g.numel(), generator=gen)] if shuffle else n2g


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_kernel_against_emulation_and_float64(shape, dtype):
    counts, D, shuffle = SHAPES[shape]
    n2g = graph_map(counts, shuffle, D + len(counts))
    G = len(counts)
    gen = torch.Generator().manual_seed(len(counts) * 7 + D)
    x = torch.randn(n2g.numel(), D, generator=gen) * 2.0 + torch.randn(G, D, generator=gen)[n2g] * 3.0
    if dtype == "bf16":
        x = x.to(torch.bfloat16)
    gamma, alpha, bias = params(D, D)
    y, mean, rstd = kernel(x.cuda(), n2g.cuda(), G, gamma, alpha, bias)
    ey, emean, erstd = GR.emulate_forward(x, n2g, gamma, alpha, bias, G=G)
    assert y.dtype == x.dtype
    assert torch.equal(mean, emean) and torch.equal(rstd, erstd), f"{shape}: statistics differ from the emulated kernel order"
    assert torch.equal(y, ey), f"{shape}: output differs from the emulated kernel order"
    if dtype == "fp32":
        exact = GR.layer_forward(x.double(), n2g, gamma.double(), alpha.double(), bias.double(), G=G)
        bnd = GR.bound(x, n2g, gamma, alpha, bias, G=G)
        err = (y.double() - exact).abs()
        bad = int((err > bnd).sum())
        assert bad == 0, f"{shape}: {bad} elements over the bound (worst ratio {float((err / bnd).max()):.2f})"


def test_one_node_graphs_with_alpha_one_give_bias_exactly():
    D = 64
    n2g = graph_map([1, 5, 1, 0, 40, 1], True, 3)
    gen = torch.Generator().manual_seed(4)
    x = torch.randn(n2g.numel(), D, generator=gen) * 100.0
    gamma, bias = torch.randn(1, D, generator=gen), torch.randn(1, D, generator=gen)
    for dt in (torch.float32, torch.bfloat16):
        y, _, _ = kernel(x.to(dt).cuda(), n2g.cuda(), 6, gamma, torch.ones(1, D), bias)
        for g in (0, 2, 5):
            rows = (n2g == g).nonzero()[:, 0]
            assert torch.equal(y[rows], bias.to(dt).expand(rows.numel(), -1)), f"graph {g} ({dt})"


def _twice(layer, x, n2g):
    with torch.no_grad():
        a = layer(x, [], n2g, {}, {}, [])
        b = layer(x, [], n2g, {}, {}, [])
    assert torch.equal(a, b), "two runs differ"
    return a


@pytest.mark.parametrize("name", NAMES)
def test_layer_against_reference_golden_and_float64(name):
    f = load(name)
    got = _twice(layer_of(f).eval(), f["x"].cuda(), f["n2g"].cuda())
    sd = f["sd"]
    ref = GR.layer_forward(f["x"].double(), f["n2g"], sd["gamma"].double(), sd["alpha"].double(), sd["bias"].double())
    assert_close(got, f["out"], TOL, f"{name} vs reference")
    assert_close(got, ref, TOL, f"{name} vs float64")


def test_layer_bf16_vs_reference():
    """DESIGN §4 bf16 rule: rel. L2 <= 1e-2 against the reference fed the same bf16 states, and at least as close to the fp32 result
    on those states as the reference's bf16 path is.  The layer returns bf16 while the reference returns fp32, so the reference's
    output is compared after the same final rounding to bf16."""
    f = load("graphnorm_d128_bf16")
    got = _twice(layer_of(f).eval(), f["x"].cuda().to(torch.bfloat16), f["n2g"].cuda())
    assert got.dtype == torch.bfloat16
    got = got.cpu().float()
    ref32, ref_b = f["out_fp32_rounded_inputs"], f["out_bf16"].to(torch.bfloat16).float()
    scale = ref32.abs().clamp(min=1)
    err_ours, err_ref = (got - ref32).abs(), (ref_b - ref32).abs()
    frac_ours, frac_ref = (err_ours <= 1e-2 * scale).float().mean().item(), (err_ref <= 1e-2 * scale).float().mean().item()
    rel = ((got - f["out_bf16"]).norm() / f["out_bf16"].norm()).item()
    msg = f"rel L2 vs reference {rel:.2e}; mean err ours {err_ours.mean():.2e} / ref {err_ref.mean():.2e}; within 1e-2 {frac_ours:.4f} / {frac_ref:.4f}"
    assert rel <= 1e-2 and err_ours.mean().item() <= 1.1 * err_ref.mean().item() and frac_ours >= frac_ref - 0.002, msg


def _grads_against_autograd(layer, x_cpu, n2g_cpu, dy, what):
    x = x_cpu.cuda().requires_grad_(True)
    n2g = n2g_cpu.cuda()
    layer(x, [], n2g, {}, {}, []).backward(dy.cuda())
    p64 = {n: p.detach().cpu().double().requires_grad_(True) for n, p in layer.named_parameters()}
    x64 = x_cpu.double().requires_grad_(True)
    GR.layer_forward(x64, n2g_cpu, p64["gamma"], p64["alpha"], p64["bias"]).backward(dy.double())
    pairs = [("d node_states", x.grad, x64.grad)] + [(n, p.grad, p64[n].grad) for n, p in layer.named_parameters()]
    assert len(pairs) == 4
    for name, got, ref in pairs:
        got = got.cpu().double()
        scale = ref.abs().max().clamp(min=1e-30)
        assert float((got - ref).abs().max() / scale) <= 1e-4, f"{what} {name}: scaled max error"
        assert float((got - ref).norm() / ref.norm().clamp(min=1e-30)) <= 1e-4, f"{what} {name}: rel. L2 error"
    grads = [p.grad.clone() for p in layer.parameters()] + [x.grad.clone()]
    layer.zero_grad()
    x.grad = None
    layer(x, [], n2g, {}, {}, []).backward(dy.cuda())
    assert all(torch.equal(a, b) for a, b in zip(grads, [p.grad for p in layer.parameters()] + [x.grad])), f"{what}: second backward differs"


@pytest.mark.parametrize("name", NAMES)
def test_backward_against_autograd(name):
    f = load(name)
    _grads_against_autograd(layer_of(f).train(), f["x"], f["n2g"], f["dy"], name)


def test_backward_against_autograd_many_chunks_and_graphs():
    import ptgnn_b200 as P

    D = 64
    n2g = graph_map([3000, 1, 0, 20] + [7] * 500, True, 9)
    gen = torch.Generator().manual_seed(10)
    x = torch.randn(n2g.numel(), D, generator=gen) + torch.randn(504, D, generator=gen)[n2g]
    layer = P.GraphNorm(D)
    with torch.no_grad():
        for p, v in zip((layer.gamma, layer.alpha, layer.bias), params(D, 11)):
            p.copy_(v)
    _grads_against_autograd(layer.cuda().train(), x, n2g, torch.randn(n2g.numel(), D, generator=gen), "3,000-row graph")


def test_layer_makes_no_host_synchronisation_with_the_count_handed_in():
    from ptgnn_b200.edgeplan import shared_num_graphs

    f = load("graphnorm_d64")
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
    norm = P.GraphNorm(H)
    with torch.no_grad():
        for p, v in zip((norm.gamma, norm.alpha, norm.bias), params(H, 12)):
            p.copy_(v)
    layers = [P.GatedMessagePassingLayer(H, H, T, "sum"), norm, P.GatedMessagePassingLayer(H, H, T, "sum")]
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
        P.GraphNorm(32).cuda()(x.bfloat16().requires_grad_(True), [], n2g, {}, {}, [])
    with pytest.raises(NotImplementedError):
        P.GraphNorm(32).cuda().eval()(x, [], n2g, {}, {}, [], gather_states=x)
    for D in (48, 288, 16):
        with pytest.raises(NotImplementedError):
            with torch.no_grad():
                P.GraphNorm(D).cuda()(torch.randn(10, D, device="cuda"), [], n2g, {}, {}, [])
    with torch.no_grad():       # bf16 without gradients runs
        assert P.GraphNorm(32).cuda()(x.bfloat16(), [], n2g, {}, {}, []).dtype == torch.bfloat16


# ---- backward kernels, element by element ------------------------------------------------------------------------------------
SCALES = (-37, -27, -17, 17)        # the gradient magnitudes of test_gpu_backward_edges.py: backward(2^k dy) = 2^k backward(dy)
EDGE_COUNTS = [1, 31, 32, 33, 0, 64, 65, 1000, 1]      # the forward's edge sizes; graphs 2 and 6 get all-equal rows
BWD_SHAPES = {f"edges_d{D}_a{a}": (EDGE_COUNTS, D, True, a) for D in range(32, 257, 32) for a in (0.0, 0.5, 1.0, 1.7)}
BWD_SHAPES.update({name: (counts, D, shuffle, None) for name, (counts, D, shuffle) in SHAPES.items()})


def backward_kernel(x, dy, n2g, G, gamma, alpha, mean, rstd):
    """Two runs of native_graph_norm_backward, which must agree bit for bit: (dx, d gamma, d alpha, d beta) on the CPU."""
    from ptgnn_b200.graphnorm import native_graph_norm_backward
    from ptgnn_b200.reduceops import graph_plan

    plan = graph_plan(n2g, G)
    runs = [native_graph_norm_backward(x, plan, gamma.cuda(), alpha.cuda(), 1e-10, mean, rstd, dy) for _ in range(2)]
    plan.validate()
    assert all(torch.equal(a, b) for a, b in zip(*runs)), "two backward runs differ"
    return [t.cpu() for t in runs[0]]


@pytest.mark.parametrize("shape", list(BWD_SHAPES))
def test_backward_kernels_against_emulation_and_float64(shape):
    """The backward kernels equal emulate_backward bit for bit and backward_formula within backward_bound, on the forward kernels'
    mean and rstd; backward(2^k dy) = 2^k backward(dy) bit for bit."""
    counts, D, shuffle, a = BWD_SHAPES[shape]
    n2g = graph_map(counts, shuffle, D + len(counts) + 1)
    G = len(counts)
    gen = torch.Generator().manual_seed(len(counts) * 11 + D)
    x = torch.randn(n2g.numel(), D, generator=gen) * 2.0 + torch.randn(G, D, generator=gen)[n2g] * 3.0
    if counts is EDGE_COUNTS:
        for g in (2, 6):
            x[n2g == g] = torch.randn(D, generator=gen) * 3.0
    dy = torch.randn(n2g.numel(), D, generator=gen)
    gamma, alpha, bias = params(D, D + 1)
    if a is not None:
        alpha = torch.full((1, D), a)
    xd, dyd, n2gd = x.cuda(), dy.cuda(), n2g.cuda()
    _, mean, rstd = GR.emulate_forward(x, n2g, gamma, alpha, bias, G=G)
    _, kmean, krstd = kernel(xd, n2gd, G, gamma, alpha, bias)
    assert torch.equal(kmean, mean) and torch.equal(krstd, rstd)
    got = backward_kernel(xd, dyd, n2gd, G, gamma, alpha, kmean.cuda(), krstd.cuda())
    emu = GR.emulate_backward(x, dy, n2g, mean, rstd, gamma, alpha, G=G)
    names = ("dx", "d gamma", "d alpha", "d beta")
    for name, g, e in zip(names, got, emu):
        assert torch.equal(g, e), f"{shape} {name}: differs from the emulated kernel order ({int((g != e).sum())} elements)"
    ref = GR.backward_formula(x, dy, n2g, mean, rstd, gamma, alpha, G=G)
    bnd = GR.backward_bound(x, dy, n2g, mean, rstd, gamma, alpha, G=G)
    for name, g, r, b in zip(names, got, ref, bnd):
        bad = int(((g.double() - r).abs() > b).sum())
        assert bad == 0, f"{shape} {name}: {bad} elements over the bound (worst ratio {float(((g.double() - r).abs() / b).max()):.2f})"
    for k in SCALES:
        scaled = backward_kernel(xd, dyd * 2.0 ** k, n2gd, G, gamma, alpha, kmean.cuda(), krstd.cuda())
        for name, g, s in zip(names, got, scaled):
            assert torch.equal(s, g * 2.0 ** k), f"{shape} {name}: backward(2^{k} dy) != 2^{k} backward(dy)"


def test_backward_shapes_reach_every_vpl_instance():
    assert sorted({D // 32 for _, D, _, _ in BWD_SHAPES.values()}) == list(range(1, 9)), "graphnorm_bwd_chunk_kernel<VPL>: 8 instances"
