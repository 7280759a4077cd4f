"""EGCMessagePassingLayer on the fused aggregation kernel's EGC write-out (DESIGN.md §3.14), against the float64 restatement of
tests/egc_reference.py: element by element within a derived bound (fp32), the bf16 emulation and the reference's autocast
fixtures (bf16), float64 autograd and the reference's gradients (backward), and the paths, caches and container around it."""
import functools

import pytest
import torch

import egc_reference as E
import fused_reference as R
from helpers import golden_adjacency, golden_state_dict, load_golden

pytestmark = pytest.mark.gpu

AGGS = ("sum", "mean", "max", "min")
SHAPES = [(64, 64, 8, 4), (128, 128, 8, 4), (128, 256, 8, 4), (64, 128, 4, 8), (128, 128, 2, 1), (128, 64, 8, 2)]
B, T, BLOCKS = 24, 3, 400          # 24: half a block is not a multiple of 8; the structured graph's empty type is type 1


@functools.lru_cache(maxsize=1)
def _graph():
    adj, n = R.structured_graph(B, T, BLOCKS, num_edges=20_000)
    return adj, [(s.cuda(), t.cuda()) for s, t in adj], n


def _layer(H, out, heads, bases, agg, seed=0, T_=T):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    layer = P.EGCMessagePassingLayer(H, out, T_, agg, num_bases=bases, num_heads=heads).cuda().eval()
    W, cw, cb = E.params_of({k: v.detach().cpu() for k, v in layer.state_dict().items()}, T_)
    return layer, W, cw, cb


def _run(layer, h, adj_d, n, block_targets=B):
    """The layer's output on an explicit block size, twice: the first output after checking the second is bit-identical."""
    import ptgnn_b200 as P

    outs = []
    for _ in range(2):
        plan = P.EdgePlan(adj_d, n, block_targets=block_targets)
        with torch.no_grad(), P.edgeplan.shared_plan(plan):
            outs.append(layer(h.cuda(), adj_d))
        plan.validate()
    assert torch.equal(outs[0], outs[1]), "EGC forward is not run-to-run bit-identical"
    return outs[0].float().cpu()


def _uses_fused(H, out, heads, bases, bf16=False):
    import ptgnn_b200 as P

    return P.egc.use_fused(P._native.lib(), bf16, H, out, heads, bases)


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("H,out,heads,bases", SHAPES)
def test_fp32_forward_within_the_float64_bound(H, out, heads, bases, agg):
    assert _uses_fused(H, out, heads, bases)
    adj, adj_d, n = _graph()
    layer, W, cw, cb = _layer(H, out, heads, bases, agg)
    h = torch.randn(n, H, generator=torch.Generator().manual_seed(3))
    got = _run(layer, h, adj_d, n)
    ref, bnd = E.forward64(h, adj, W, cw, cb, agg, heads, bases)
    R.check_bound(got, ref, bnd, f"EGC {agg} H={H} out={out} heads={heads} bases={bases}")
    empty = torch.ones(n, dtype=torch.bool)
    empty[torch.cat([t for _, t in adj])] = False
    assert int(empty.sum()) > 0 and bool((got[empty] == 0).all()), "targets without in-edges must give exactly 0"


@pytest.mark.parametrize("agg", AGGS)
def test_no_edges_gives_zeros(agg):
    layer, *_ = _layer(64, 64, 8, 4, agg)
    empty = [(torch.zeros(0, dtype=torch.int64, device="cuda"),) * 2 for _ in range(T)]
    out = _run(layer, torch.randn(100, 64), empty, 100)
    assert bool((out == 0).all())


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("H,out,heads,bases", [(64, 64, 8, 4), (128, 256, 8, 4), (64, 128, 4, 8), (128, 128, 2, 1)])
def test_bf16_forward_against_the_emulation(H, out, heads, bases, agg):
    assert _uses_fused(H, out, heads, bases, bf16=True)
    adj, adj_d, n = _graph()
    layer, W, cw, cb = _layer(H, out, heads, bases, agg)
    h = torch.randn(n, H, generator=torch.Generator().manual_seed(4)).to(torch.bfloat16)
    got = _run(layer, h, adj_d, n)
    with torch.no_grad():
        assert layer(h.cuda(), adj_d).dtype == torch.bfloat16
    # per element: exact wherever no fp32 accumulation lands near a bf16 midpoint (test_egc_native_cpu.py shows that kernels which
    # drop the rounding of A, of the products or of the coefficients fail this)
    ref, bnd = E.bf16_kernel_reference(h.float(), adj, W, cw, cb, agg, heads, bases)
    R.check_bound(got, ref, bnd, f"EGC bf16 {agg} H={H} out={out} heads={heads} bases={bases}")
    exact, _ = E.forward64(h.float(), adj, W, cw, cb, agg, heads, bases)
    assert E.rel_l2(got, exact) <= 1e-2


@pytest.mark.parametrize("agg", ["sum", "max"])
def test_bf16_forward_against_the_reference_under_autocast(agg):
    import ptgnn_b200 as P

    g = load_golden(f"egc_{agg}_bf16ac")
    adj = [(s.cuda(), t.cuda()) for s, t in golden_adjacency(g)]
    layer = P.EGCMessagePassingLayer(64, 64, len(adj), agg, num_bases=4, num_heads=8)
    layer.load_state_dict(golden_state_dict(g), strict=True)
    layer = layer.cuda().eval()
    with torch.no_grad():
        out = layer(torch.from_numpy(g["h"]).cuda().to(torch.bfloat16), adj)
    bars = E.n2_bars(out.float(), torch.from_numpy(g["out_autocast"]), torch.from_numpy(g["out_fp32_rounded_inputs"]))
    assert bars == {"rel_l2": True, "mean": True, "within": True}, bars


def test_no_edge_sized_message_tensor(monkeypatch):
    import ptgnn_b200 as P

    n, E_ = 50_000, 400_000
    gen = torch.Generator().manual_seed(6)
    adj = [(torch.randint(0, n, (E_ // 2,), generator=gen).cuda(), torch.randint(0, n, (E_ // 2,), generator=gen).cuda()) for _ in range(2)]
    layer, *_ = _layer(128, 128, 8, 4, "sum", T_=2)
    h = torch.randn(n, 128, device="cuda")
    msg_bytes = E_ * 512 * 4

    def peak(fused: bool):
        monkeypatch.setenv("PTGNN_B200_FP32_MODE", "" if fused else "tf32")
        plan = P.EdgePlan(adj, n)
        with torch.no_grad(), P.edgeplan.shared_plan(plan):
            layer(h, adj)                       # warm: the weight cache and the plan's arrays
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out = layer(h, adj)
            torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, out

    fused_peak, a = peak(True)
    composed_peak, b = peak(False)
    assert fused_peak < msg_bytes / 4, f"fused peak {fused_peak / 2**20:.1f} MiB"
    assert composed_peak > msg_bytes, f"composed peak {composed_peak / 2**20:.1f} MiB"
    assert E.rel_l2(a, b) <= 2e-6


def test_paths(monkeypatch):
    import ptgnn_b200 as P

    adj, adj_d, n = _graph()
    # a shape outside the supported set (out = 96 is not a multiple of 128 / 2) stays composed, and still matches the restatement
    assert not _uses_fused(64, 96, 4, 2)
    layer, W, cw, cb = _layer(64, 96, 4, 2, "min")
    h = torch.randn(n, 64, generator=torch.Generator().manual_seed(7))
    ref, _ = E.forward64(h, adj, W, cw, cb, "min", 4, 2)
    assert E.rel_l2(_run(layer, h, adj_d, n), ref) <= 1e-6
    with pytest.raises(NotImplementedError):
        with torch.no_grad():
            layer(h.cuda().to(torch.bfloat16), adj_d)
    # PTGNN_B200_FP32_MODE=tf32 on a supported shape: the composed path, within 2e-5 of the fused result
    layer, *_ = _layer(128, 128, 8, 4, "mean")
    h = torch.randn(n, 128, generator=torch.Generator().manual_seed(8))
    fused = _run(layer, h, adj_d, n)
    monkeypatch.setenv("PTGNN_B200_FP32_MODE", "tf32")
    assert not _uses_fused(128, 128, 8, 4)
    composed = _run(layer, h, adj_d, n)
    scale = composed.abs().max()
    assert float((fused - composed).abs().max() / scale) <= 2e-5


def test_eval_weight_cache_is_reused_and_refreshed_after_an_in_place_edit():
    adj, adj_d, n = _graph()
    layer, W, cw, cb = _layer(64, 64, 8, 4, "sum")
    h = torch.randn(n, 64, generator=torch.Generator().manual_seed(9))
    first = _run(layer, h, adj_d, n)
    (entry,) = layer._derived_weights.values()
    key, buf = entry["key"], entry["buf"].data_ptr()
    _run(layer, h, adj_d, n)
    assert entry["key"] == key and entry["buf"].data_ptr() == buf
    bases0 = layer._EGCMessagePassingLayer__bases[0].weight
    with torch.no_grad():
        bases0.mul_(-2.0)
    got = _run(layer, h, adj_d, n)
    assert entry["key"] != key
    ref, bnd = E.forward64(h, adj, [bases0.detach().cpu()] + W[1:], cw, cb, "sum", 8, 4)
    R.check_bound(got, ref, bnd, "after an in-place edit")
    assert not torch.equal(got, first)


def _grad_check(layer, h, adj, adj_d, agg, heads, bases, g_out, tol=1e-4):
    """Native gradients against float64 autograd of the restatement (relative L2 per tensor)."""
    W, cw, cb = E.params_of({k: v.detach().cpu() for k, v in layer.state_dict().items()}, len(adj))
    layer.zero_grad()
    x = h.cuda().requires_grad_(True)
    out = layer(x, adj_d)
    out.backward(g_out.cuda())
    p64 = [w.double().requires_grad_(True) for w in W] + [cw.double().requires_grad_(True), cb.double().requires_grad_(True)]
    h64 = h.double().requires_grad_(True)
    ref = E.forward_torch(h64, adj, p64[:-2], p64[-2], p64[-1], agg, heads, bases)
    ref_grads = torch.autograd.grad(ref, [h64] + p64, g_out.double())
    coeff = layer._EGCMessagePassingLayer__weight_coeffs
    native = [x.grad] + [b.weight.grad for b in layer._EGCMessagePassingLayer__bases] + [coeff.weight.grad, coeff.bias.grad]
    for name, a, b in zip(["h"] + [f"bases{t}" for t in range(len(W))] + ["coeff.weight", "coeff.bias"], native, ref_grads):
        if bool((b != 0).any()):
            assert E.rel_l2(a, b) <= tol, f"{agg} d {name}: {E.rel_l2(a, b):.2e}"
        else:
            assert bool((a == 0).all()), f"{agg} d {name} should be 0"
    return out


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("H,out,heads,bases", [(64, 64, 8, 4), (128, 128, 8, 4), (64, 128, 4, 8)])
def test_gradients_against_float64_autograd(H, out, heads, bases, agg):
    import ptgnn_b200 as P

    adj, _, n = _graph()
    # tie-free max / min: the structured graph with its repeated (source, target) edges of one type removed, random states
    adj = [tuple(torch.unique(s * n + t).div(n, rounding_mode="floor") if i == 0 else torch.unique(s * n + t) % n for i in range(2))
           for s, t in adj]
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    layer, *_ = _layer(H, out, heads, bases, agg, seed=1)
    layer.train()
    gen = torch.Generator().manual_seed(10)
    h = torch.randn(n, H, generator=gen)
    g_out = torch.randn(n, out, generator=gen)
    with P.edgeplan.shared_plan(P.EdgePlan(adj_d, n, block_targets=B)):
        _grad_check(layer, h, adj, adj_d, agg, heads, bases, g_out)


@pytest.mark.parametrize("agg", AGGS)
def test_gradients_against_the_reference_fixture(agg):
    import ptgnn_b200 as P

    g = load_golden(f"egc_grad_{agg}")
    adj = golden_adjacency(g)
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    layer = P.EGCMessagePassingLayer(64, 64, len(adj), agg, num_bases=int(g["bases"]), num_heads=int(g["heads"]))
    layer.load_state_dict(golden_state_dict(g), strict=True)
    layer = layer.cuda()
    out = _grad_check(layer, torch.from_numpy(g["h"]), adj, adj_d, agg, int(g["heads"]), int(g["bases"]), torch.from_numpy(g["d_out"]))
    assert E.rel_l2(out, torch.from_numpy(g["out"])) <= 1e-6
    names = dict(layer.named_parameters())
    for k in names:
        ref = torch.from_numpy(g["grad::" + k])
        assert E.rel_l2(names[k].grad, ref) <= 1e-4 if bool(ref.any()) else bool((names[k].grad == 0).all()), k


def _container(H=64):
    import ptgnn_b200 as P

    torch.manual_seed(12)
    r = P.ConcatResidualLayer(H)
    e1 = P.EGCMessagePassingLayer(H, H, T, "sum")
    e2 = P.EGCMessagePassingLayer(2 * H, H, T, "max")

    class Embed(torch.nn.Module):
        def forward(self, x):
            return x

    return P.GraphNeuralNetwork([r.pass_through_dummy_layer(), e1, r, e2], Embed(), introduce_backwards_edges=False,
                                add_self_edges=False).cuda(), (e1, e2)


def test_container_training_steps_match_the_float64_restatement():
    gen = torch.Generator().manual_seed(13)
    n, H = 600, 64
    adj = [(torch.randint(0, n, (c,), generator=gen), torch.randint(0, n - 20, (c,), generator=gen)) for c in (2500, 0, 1200)]
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    h = torch.randn(n, H, generator=gen)
    target = torch.randn(n, H, generator=gen)
    gnn, (e1, e2) = _container(H)
    gnn.train()
    ref_params = [[p.detach().cpu().double().clone() for p in E.params_of({k: v for k, v in e.state_dict().items()}, T)[0]] +
                  [p.detach().cpu().double().clone() for p in E.params_of({k: v for k, v in e.state_dict().items()}, T)[1:]] for e in (e1, e2)]
    opt = torch.optim.SGD(gnn.parameters(), lr=0.05)
    lr = 0.05
    for step in range(3):
        opt.zero_grad()
        out = gnn.gnn(h.cuda(), adj_d, None, None, {}, {})
        loss = ((out - target.cuda()) ** 2).mean()
        loss.backward()
        opt.step()
        # the same step in float64 on the restatement
        ps = [[p.requires_grad_(True) for p in ps_] for ps_ in ref_params]
        x1 = E.forward_torch(h.double(), adj, ps[0][:T], ps[0][T], ps[0][T + 1], "sum", 8, 4)
        x2 = E.forward_torch(torch.cat([h.double(), x1], -1), adj, ps[1][:T], ps[1][T], ps[1][T + 1], "max", 8, 4)
        ref_loss = ((x2 - target.double()) ** 2).mean()
        grads = torch.autograd.grad(ref_loss, [p for ps_ in ps for p in ps_])
        assert abs(float(loss.detach()) - float(ref_loss.detach())) <= 1e-5 * max(1.0, float(ref_loss))
        it = iter(grads)
        ref_params = [[(p - lr * next(it)).detach() for p in ps_] for ps_ in ps]
    for e, ps_ in zip((e1, e2), ref_params):
        W, cw, cb = E.params_of({k: v.detach().cpu() for k, v in e.state_dict().items()}, T)
        for a, b in zip(W + [cw, cb], ps_):
            assert E.rel_l2(a, b) <= 1e-5


def test_container_capture_replays_bit_identically():
    gen = torch.Generator().manual_seed(14)
    n, H = 3000, 64
    adj_d = [(torch.randint(0, n, (c,), generator=gen).cuda(), torch.randint(0, n, (c,), generator=gen).cuda()) for c in (9000, 0, 4000)]
    h = torch.randn(n, H, generator=gen).cuda()
    gnn, _ = _container(H)
    gnn.eval()
    with torch.no_grad():
        eager = gnn.gnn(h, adj_d, None, None, {}, {})
        graphed = gnn.capture(h, adj_d)
        first = graphed.replay().clone()
        h.copy_(torch.randn(n, H, generator=gen).cuda())
        second = graphed.replay().clone()
        eager2 = gnn.gnn(h, adj_d, None, None, {}, {})
    assert torch.equal(first, eager) and torch.equal(second, eager2)


def test_refusals():
    import ptgnn_b200 as P

    n = 2000
    gen = torch.Generator().manual_seed(15)
    # an adjacency of its own: the fp16-range flag stays set on its cached plan
    adj_d = [(torch.randint(0, n, (c,), generator=gen).cuda(), torch.randint(0, n, (c,), generator=gen).cuda()) for c in (5000, 0, 3000)]
    layer, *_ = _layer(64, 64, 8, 4, "sum")
    h = torch.randn(n, 64, device="cuda")
    h[5, 3] = 70000.0
    with torch.no_grad():
        layer(h, adj_d)
        torch.cuda.synchronize()
        with pytest.raises(FloatingPointError):
            layer(h, adj_d)
    layer.train()
    with pytest.raises(NotImplementedError):
        layer(torch.randn(n, 64, device="cuda").to(torch.bfloat16), adj_d)
    dropping = P.EGCMessagePassingLayer(64, 64, T, "sum", dropout_rate=0.2).cuda().train()
    with pytest.raises(NotImplementedError):
        dropping(torch.randn(n, 64, device="cuda"), adj_d)
