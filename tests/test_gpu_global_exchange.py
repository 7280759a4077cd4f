"""GruGlobalStateUpdate on the GPU: the per-graph readout kernel against float64 with per-element bounds, the layer (table GRU)
against the float64 oracle, bf16 against the reference's autocast fixture, a VarMisuse-style stack in a container (chain, capture,
no host synchronisation), and training against torch.autograd through the oracle.  Every case runs twice and must be bit-identical.

Readout bound (DESIGN.md §3.5 gives the summation order).  With u = 2^-24 and gamma_k = k u / (1 - k u): a chunk's gate dot product is
a per-lane fmaf chain over H / 32 features, then a five-level butterfly: |dz| <= gamma_{H/32+5} sum_f |x_f w_f|.  s = 1 / (1 + expf(-z)):
expf <= 2 ulp, the add and the division 1/2 ulp each, so |ds| <= s (1 - s) |dz| + 4 u s.  A chunk of at most CHUNK = 32 rows accumulates
fmaf(s, x, acc) in node order, then the graph's k chunks are added in chunk order from 0: |d g| <= gamma_{32 + k} sum_n s_n |x_n| +
sum_n |x_n| |ds_n|; mean adds u |g|.  The float64 s is used in place of the computed one: the 1 % slack on the bound covers that."""
import os

import numpy as np
import pytest
import torch

from helpers import assert_close, gated_oracle_args
import global_exchange_reference as GX
from oracle import ptgnn_oracle as O

pytestmark = pytest.mark.gpu

CHUNK = 32
U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gamma(k):
    return k * U / (1 - k * U)


def _n2g_layout(name, gen):
    """(node_to_graph_idx [N] int64, num_graphs)."""
    if name == "sizes":            # graphs of 1, CHUNK - 1, CHUNK, CHUNK + 1 and 3 CHUNK + 5 nodes, in node order
        sizes = [1, CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 5]
        return torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes)), len(sizes)
    if name == "one_big":          # 40,000 nodes in one graph
        return torch.zeros(40_000, dtype=torch.int64), 1
    if name == "config2":          # 80 x 2,560
        return torch.repeat_interleave(torch.arange(80), 2560), 80
    if name == "unsorted_gaps":    # shuffled ids, graphs 2 and 7 empty, two trailing empty graphs (num_graphs > max + 1)
        ids = torch.tensor([0, 1, 3, 4, 5, 6, 8])[torch.randint(0, 7, (3000,), generator=gen)]
        ids[:2] = torch.tensor([0, 8])
        return ids, 11
    raise ValueError(name)


def _readout_ref(x64, n2g, G, kind, w64):
    """float64 readout and its per-element bound."""
    H = x64.shape[1]
    ax = x64.abs()
    if kind == "weighted":
        z = x64 @ w64.reshape(-1)
        s = torch.sigmoid(z)
        dz = gamma(H // 32 + 5) * (ax @ w64.abs().reshape(-1))
        ds = s * (1 - s) * dz + 4 * U * s
    else:
        s = torch.ones(x64.shape[0], dtype=torch.float64)
        ds = torch.zeros_like(s)
    idx = n2g.reshape(-1, 1).expand(-1, H)
    g = torch.zeros(G, H, dtype=torch.float64).scatter_add_(0, idx, x64 * s[:, None])
    mass = torch.zeros(G, H, dtype=torch.float64).scatter_add_(0, idx, ax * s[:, None])
    prop = torch.zeros(G, H, dtype=torch.float64).scatter_add_(0, idx, ax * ds[:, None])
    count = torch.bincount(n2g, minlength=G).to(torch.float64)
    chunks = torch.ceil(count / CHUNK)
    bound = ((CHUNK + chunks) * U / (1 - (CHUNK + chunks) * U))[:, None] * mass + prop
    if kind == "mean":
        c = count.clamp(min=1)[:, None]
        g, bound = g / c, bound / c + U * (g / c).abs()
    return g, bound * 1.01, s


def _native_readout(x, n2g, G, kind, w):
    from ptgnn_b200 import _native as N
    from ptgnn_b200.reduceops import graph_plan, native_readout

    mode = {"weighted": N.READOUT_WEIGHTED_SUM, "sum": N.READOUT_SUM, "mean": N.READOUT_MEAN}[kind]
    n2g_d = n2g.cuda()
    plan = graph_plan(n2g_d, G)
    a = native_readout(x.cuda(), plan, mode, None if w is None else w.cuda())[0]
    b = native_readout(x.cuda(), plan, mode, None if w is None else w.cuda())[0]
    plan.validate()
    assert torch.equal(a, b), "readout is not run-to-run bit-identical"
    return a.cpu().double()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("H", [64, 128, 256])
@pytest.mark.parametrize("layout", ["sizes", "one_big", "config2", "unsorted_gaps"])
def test_readout_against_float64(layout, H, dtype):
    if layout in ("one_big", "config2") and H == 256:
        pytest.skip("H = 256 is covered on the smaller layouts (the float64 reference of 204,800 x 256 takes gigabytes)")
    gen = torch.Generator().manual_seed(len(layout) * 1000 + H)
    n2g, G = _n2g_layout(layout, gen)
    x = (torch.randn(n2g.shape[0], H, generator=gen) * 0.5).to(dtype)
    w = torch.randn(1, H, generator=gen) * (1.0 / H ** 0.5)
    x64 = x.double()
    for kind in ("weighted", "sum", "mean"):
        ref, bound, _ = _readout_ref(x64, n2g, G, kind, w.double() if kind == "weighted" else None)
        got = _native_readout(x, n2g, G, kind, w if kind == "weighted" else None)
        err = (got - ref).abs()
        ratio = float((err / bound.clamp(min=1e-300)).max())
        assert bool((err <= bound).all()), f"{layout} H={H} {dtype} {kind}: error / bound {ratio:.3f}"
        empty = torch.bincount(n2g, minlength=G) == 0
        assert bool((got[empty] == 0).all()), "graphs without nodes must be exactly 0"
        # the bound is tight enough to reject a kernel that drops a graph's last partial chunk
        count = torch.bincount(n2g, minlength=G)
        last = [b for b in range(G) if count[b] % CHUNK != 0]
        if last:
            mutant = ref.clone()
            for b in last:
                nodes = (n2g == b).nonzero().reshape(-1)
                tail = nodes[(count[b] // CHUNK) * CHUNK:]
                s = torch.sigmoid(x64[tail] @ w.double().reshape(-1)) if kind == "weighted" else torch.ones(len(tail), dtype=torch.float64)
                part = (x64[tail] * s[:, None]).sum(0)
                mutant[b] -= part / (count[b] if kind == "mean" else 1)
            assert not bool(((mutant - ref).abs() <= bound).all()), "the bound does not reject a dropped last chunk"


def _layer(kind, H, seed, S=None, dropout=0.0):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    reducer = P.WeightedSumVarSizedElementReduce(H) if kind == "weighted" else P.SimpleVarSizedElementReduce(kind)
    return P.GruGlobalStateUpdate(reducer, H, H if S is None else S, dropout_rate=dropout).cuda().eval()


def _params64(layer):
    sd = {k: v.detach().cpu().double() for k, v in layer.state_dict().items()}
    p = "_GruGlobalStateUpdate__gru_cell."
    w = sd.get("_AbstractGlobalGraphExchange__global_graph_representation_module._WeightedSumVarSizedElementReduce__weights_layer.weight")
    return w, [sd[p + k] for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]


def _graphs(N, gen, per_graph=500):
    G = max(1, (N + per_graph - 1) // per_graph)
    n2g = torch.randint(0, G, (N,), generator=gen)
    return n2g, int(n2g.max()) + 1


def _twice(layer, h, n2g):
    with torch.no_grad():
        a = layer(h.cuda(), [], n2g.cuda(), {}, {}, [])
        b = layer(h.cuda(), [], n2g.cuda(), {}, {}, [])
    assert torch.equal(a, b), "layer output is not run-to-run bit-identical"
    return a.float().cpu()


def _oracle64(layer, h, n2g, kind):
    w, p = _params64(layer)
    return GX.global_gru_update_forward(h.double(), n2g, kind, w, *p)


@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("N", [1, 63, 64, 65, 127, 129, 1000, 64 * (33 * 3 + 5) + 17, 40_000])
def test_layer_fp32_against_float64(N, H):
    gen = torch.Generator().manual_seed(N + H)
    n2g, _ = _graphs(N, gen)
    h = torch.randn(N, H, generator=gen) * 0.5
    layer = _layer("weighted", H, N + H)
    assert_close(_twice(layer, h, n2g), _oracle64(layer, h, n2g, "weighted"), what=f"fp32 global layer N={N} H={H}")


@pytest.mark.parametrize("kind", ["weighted", "sum", "mean", "max", "min"])
def test_layer_fp32_every_reducer(kind):
    gen = torch.Generator().manual_seed(7)
    n2g, _ = _graphs(5000, gen)
    h = torch.randn(5000, 64, generator=gen) * 0.5
    layer = _layer(kind, 64, 11)
    assert_close(_twice(layer, h, n2g), _oracle64(layer, h, n2g, kind), what=f"fp32 global layer, {kind}")


def test_layer_fp32_custom_reducer_and_composed_fallback():
    import ptgnn_b200 as P

    class HalfMean(P.AbstractVarSizedElementReduce):      # a user module: called as is, its output feeds the table GRU
        def forward(self, inputs):
            return 0.5 * P.scatter_mean(inputs.element_embeddings, inputs.element_to_sample_map, dim=0, dim_size=inputs.num_samples)

    gen = torch.Generator().manual_seed(3)
    n2g, G = _graphs(3000, gen)
    for H in (64, 32):                                    # 32: no state-only GRU instance -> gathered summaries + native GRUCell
        h = torch.randn(3000, H, generator=gen) * 0.5
        torch.manual_seed(H)
        layer = P.GruGlobalStateUpdate(HalfMean(), H, H).cuda().eval()
        _, p = _params64(layer)
        g = 0.5 * O.scatter(h.double(), n2g, G, "mean")
        assert_close(_twice(layer, h, n2g), O.gru_cell(g[n2g], h.double(), *p), what=f"custom reducer H={H}")
        layer = _layer("weighted", H, H + 1)
        assert_close(_twice(layer, h, n2g), _oracle64(layer, h, n2g, "weighted"), what=f"weighted H={H}")


@pytest.mark.parametrize("H", [64, 128, 256])
@pytest.mark.parametrize("N", [1, 65, 1000, 40_000])
def test_layer_bf16(N, H):
    gen = torch.Generator().manual_seed(N * 3 + H)
    n2g, _ = _graphs(N, gen)
    h = (torch.randn(N, H, generator=gen) * 0.5).to(torch.bfloat16)
    layer = _layer("weighted", H, N + H + 1)
    got = _twice(layer, h, n2g)
    ref = _oracle64(layer, h.float(), n2g, "weighted").float()
    rel = ((got - ref).norm() / ref.norm()).item()
    frac = ((got - ref).abs() <= 1e-2 * ref.abs().clamp(min=1)).float().mean().item()
    assert rel <= 1e-2 and frac >= 0.999, f"bf16 N={N} H={H}: rel L2 {rel:.2e}, within 1e-2: {frac:.4f}"


def test_layer_bf16_vs_reference_autocast():
    """DESIGN §4 bf16 rule: rel. L2 <= 1e-2 against the reference's autocast output, and at least as close to the fp32 result as the
    reference's autocast path is."""
    import ptgnn_b200 as P

    z = np.load(os.path.join(GOLDEN, "global_weighted_bf16ac.npz"))
    H = z["h"].shape[1]
    layer = P.GruGlobalStateUpdate(P.WeightedSumVarSizedElementReduce(H), H, H)
    layer.load_state_dict({k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")})
    layer = layer.cuda().eval()
    got = _twice(layer, torch.from_numpy(z["h"]).to(torch.bfloat16), torch.from_numpy(z["n2g"]))
    ref_ac, ref32 = torch.from_numpy(z["out_autocast"]), torch.from_numpy(z["out_fp32_rounded_inputs"])
    scale = ref32.abs().clamp(min=1)
    err_ours, err_ref = (got - ref32).abs(), (ref_ac - ref32).abs()
    frac_ours, frac_ref = (err_ours <= 1e-2 * scale).float().mean().item(), (err_ref <= 1e-2 * scale).float().mean().item()
    rel_ac = ((got - ref_ac).norm() / ref_ac.norm()).item()
    msg = f"rel L2 vs autocast {rel_ac:.2e}; mean err ours {err_ours.mean():.2e} / ref {err_ref.mean():.2e}; within 1e-2 {frac_ours:.4f} / {frac_ref:.4f}"
    assert rel_ac <= 1e-2 and err_ours.mean().item() <= 1.1 * err_ref.mean().item() and frac_ours >= frac_ref - 0.002, msg


@pytest.mark.parametrize("name", ["global_weighted", "global_sum", "global_mean", "global_max"])
def test_layer_fp32_vs_reference_golden(name):
    import ptgnn_b200 as P

    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    H, kind = z["h"].shape[1], str(z["kind"])
    reducer = P.WeightedSumVarSizedElementReduce(H) if kind == "weighted" else P.SimpleVarSizedElementReduce(kind)
    layer = P.GruGlobalStateUpdate(reducer, H, H)
    layer.load_state_dict({k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")})
    got = _twice(layer.cuda().eval(), torch.from_numpy(z["h"]), torch.from_numpy(z["n2g"]))
    assert_close(got, torch.from_numpy(z["out"]), what=name)


# ---- VarMisuse GGNN stack (varmisuse/train.py:76-107): taps, shared gated x3, global, gated, join, gated x3, global, gated, join ----
def _varmisuse_stack(H, T, seed):
    import ptgnn_b200 as P

    class _Embed(torch.nn.Module):
        def forward(self, x):
            return x

    torch.manual_seed(seed)
    shared = P.GatedMessagePassingLayer(H, H, T, "sum")
    j1, j2 = P.MeanResidualLayer(H), P.MeanResidualLayer(H)
    glob1 = P.GruGlobalStateUpdate(P.WeightedSumVarSizedElementReduce(H), H, H)
    glob2 = P.GruGlobalStateUpdate(P.WeightedSumVarSizedElementReduce(H), H, H)
    g1, g2 = P.GatedMessagePassingLayer(H, H, T, "sum"), P.GatedMessagePassingLayer(H, H, T, "sum")
    layers = [j1.pass_through_dummy_layer(), shared, shared, shared, glob1, g1, j1,
              j2.pass_through_dummy_layer(), shared, shared, shared, glob2, g2, j2]
    return P.GraphNeuralNetwork(layers, _Embed(), False, False).cuda().eval(), layers


def _stack_oracle(layers, h, adj, n2g):
    import ptgnn_b200 as P

    x = h.double()
    taps = {}
    for layer in layers:
        if isinstance(layer, P.MeanResidualLayer):
            x = (taps.pop(id(layer)) + x) / 2
        elif isinstance(layer, P.GatedMessagePassingLayer):
            a = gated_oracle_args({k: v.cpu().double() for k, v in layer.state_dict().items()})
            x = O.gated_layer_forward(x, adj, [torch.empty(s.shape[0], 0, dtype=torch.float64) for s, _ in adj], aggregation_fn="sum", **a)
        elif isinstance(layer, P.GruGlobalStateUpdate):
            w, p = _params64(layer)
            x = GX.global_gru_update_forward(x, n2g, "weighted", w, *p)
        else:   # a tap: remembers the states for its join
            taps[id(layer._ResidualOriginLayer__target_layer)] = x
    return x


def _stack_inputs(N, H, T, seed):
    gen = torch.Generator().manual_seed(seed)
    adj = [(torch.randint(0, N, (c,), generator=gen), torch.randint(0, N, (c,), generator=gen)) for c in (2 * N, N, N // 2)][:T]
    n2g = torch.sort(torch.randint(0, 40, (N,), generator=gen)).values
    h = torch.randn(N, H, generator=gen) * 0.5
    return h, adj, n2g


def test_varmisuse_stack_chain_capture_and_sync_free(monkeypatch):
    N, H, T = 8000, 64, 3
    h, adj, n2g = _stack_inputs(N, H, T, 5)
    gnn, layers = _varmisuse_stack(H, T, 6)
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    hd, n2g_d = h.cuda(), n2g.cuda()
    G = int(n2g.max()) + 1
    with torch.no_grad():
        chained = gnn.gnn(hd, adj_d, None, n2g_d, {}, {}, num_graphs=G)
        again = gnn.gnn(hd, adj_d, None, n2g_d, {}, {})                 # count read from the device instead
        monkeypatch.setenv("PTGNN_B200_CHAIN", "0")
        plain = gnn.gnn(hd, adj_d, None, n2g_d, {}, {}, num_graphs=G)
        monkeypatch.delenv("PTGNN_B200_CHAIN")
    assert torch.equal(chained, again) and torch.equal(chained, plain), "chained / unchained / handed-over count runs differ"
    ref = _stack_oracle(layers, h, adj, n2g)
    err = ((chained.cpu().double() - ref).abs() / ref.abs().clamp(min=1)).max().item()
    assert err <= 5e-5, f"free-running stack error {err:.2e}"
    # trailing empty graphs change nothing
    with torch.no_grad():
        more = gnn.gnn(hd, adj_d, None, n2g_d, {}, {}, num_graphs=G + 3)
    assert torch.equal(more, chained)
    # capture: replay equals eager bit for bit
    graphed = gnn.capture(hd.clone(), adj_d, n2g_d)
    assert torch.equal(graphed.replay(), chained), "captured replay differs from the eager run"
    # with the count handed in, a global layer call makes no host synchronisation
    glob = layers[4]
    from ptgnn_b200.edgeplan import shared_num_graphs

    with torch.no_grad():
        glob(hd, adj_d, n2g_d, {}, {}, [])               # warm: plan cache, weight cache
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            with shared_num_graphs(G):
                glob(hd, adj_d, n2g_d, {}, {}, [])
        finally:
            torch.cuda.set_sync_debug_mode("default")


def test_graph_id_out_of_range_raises_at_next_poll():
    from ptgnn_b200.edgeplan import shared_num_graphs

    layer = _layer("weighted", 64, 1)
    n2g = torch.zeros(500, dtype=torch.int64)
    n2g[17] = 9
    n2g_d, h = n2g.cuda(), torch.randn(500, 64).cuda()
    with torch.no_grad(), shared_num_graphs(4):
        layer(h, [], n2g_d, {}, {}, [])
        torch.cuda.synchronize()
        with pytest.raises(IndexError):
            layer(h, [], n2g_d, {}, {}, [])


# ---- training -------------------------------------------------------------------------------------------------------------
class _FixedMask(torch.nn.Module):
    def __init__(self, mask):
        super().__init__()
        self.mask = mask

    def forward(self, x):
        return x * self.mask.to(x.device)


def _grads_close(a, b, what):
    """The bar of test_gpu_backward.py: max error over max(1, max |ref|), and rel. L2, both <= 1e-4."""
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    scaled = (a - b).abs().max().item() / max(1.0, b.abs().max().item())
    rel = ((a - b).norm() / b.norm().clamp(min=1e-30)).item()
    assert scaled <= 1e-4 and rel <= 1e-4, f"{what}: scaled {scaled:.2e} rel L2 {rel:.2e}"


@pytest.mark.parametrize("kind,dropout", [("weighted", False), ("weighted", True), ("sum", False), ("mean", False), ("max", False)])
def test_backward_against_autograd(kind, dropout):
    N, H = 3000, 64
    gen = torch.Generator().manual_seed(21)
    n2g, G = _graphs(N, gen, 400)
    h = torch.randn(N, H, generator=gen) * 0.5
    layer = _layer(kind, H, 22).train()
    mask = (torch.rand(G, H, generator=gen) > 0.3).float() / 0.7
    if dropout:
        layer._AbstractGlobalGraphExchange__dropout = _FixedMask(mask)
    hd = h.cuda().requires_grad_(True)
    out = layer(hd, [], n2g.cuda(), {}, {}, [])
    grad_out = torch.randn(N, H, generator=gen)
    out.backward(grad_out.cuda())

    h64 = h.double().requires_grad_(True)
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in layer.named_parameters()}
    wk = "_AbstractGlobalGraphExchange__global_graph_representation_module._WeightedSumVarSizedElementReduce__weights_layer.weight"
    p = [sd["_GruGlobalStateUpdate__gru_cell." + k] for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    g = GX.graph_readout(h64, n2g, G, kind, sd.get(wk))
    if dropout:
        g = g * mask.double()
    ref = O.gru_cell(g[n2g], h64, *p)
    ref.backward(grad_out.double())
    _grads_close(hd.grad, h64.grad, f"{kind} d h")
    for name, param in layer.named_parameters():
        _grads_close(param.grad, sd[name].grad, f"{kind} d {name}")


def test_two_sgd_steps_through_container_match_cpu():
    import ptgnn_b200 as P

    N, H, T = 2000, 64, 2
    h, adj, n2g = _stack_inputs(N, H, T, 31)
    gnn, layers = _varmisuse_stack(H, T, 32)
    gnn.train()
    params = [p for p in gnn.parameters()]
    ref_params = [p.detach().cpu().double().clone().requires_grad_(True) for p in params]
    index = {id(p): i for i, p in enumerate(params)}
    target = torch.randn(N, H, generator=torch.Generator().manual_seed(33))
    opt = torch.optim.SGD(params, lr=0.05)
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    for _ in range(2):
        opt.zero_grad()
        out = gnn.gnn(h.cuda(), adj_d, None, n2g.cuda(), {}, {}, num_graphs=int(n2g.max()) + 1)
        ((out - target.cuda()) ** 2).mean().backward()
        opt.step()
    # the same two steps on the CPU in float64, through the oracle with the reference's parameter layout
    def run_cpu(x):
        taps = {}
        for layer in layers:
            names = {n: ref_params[index[id(p)]] for n, p in layer.named_parameters()}
            if isinstance(layer, P.MeanResidualLayer):
                x = (taps.pop(id(layer)) + x) / 2
            elif isinstance(layer, P.GatedMessagePassingLayer):
                a = gated_oracle_args(names)
                x = O.gated_layer_forward(x, adj, [torch.empty(s.shape[0], 0, dtype=torch.float64) for s, _ in adj], aggregation_fn="sum", **a)
            elif isinstance(layer, P.GruGlobalStateUpdate):
                w = names["_AbstractGlobalGraphExchange__global_graph_representation_module._WeightedSumVarSizedElementReduce__weights_layer.weight"]
                x = GX.global_gru_update_forward(x, n2g, "weighted", w, *(names["_GruGlobalStateUpdate__gru_cell." + k]
                                                                          for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")))
            else:
                taps[id(layer._ResidualOriginLayer__target_layer)] = x
        return x

    ref_opt = torch.optim.SGD(ref_params, lr=0.05)
    for _ in range(2):
        ref_opt.zero_grad()
        ((run_cpu(h.double()) - target.double()) ** 2).mean().backward()
        ref_opt.step()
    for p, r in zip(params, ref_params):
        _grads_close(p, r, "parameters after two SGD steps")
