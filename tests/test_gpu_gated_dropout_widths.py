"""GatedMessagePassingLayer in training mode with per-edge dropout at the widths the fused kernel does not take: the masked messages
of the three-kernel path element by element against float64, the layer's forward and gradients against the float64 restatement of
test_gpu_gated_dropout.py with the same mask, reproducibility, the stacks of the reference's Typilus and VarMisuse training scripts
without an edge-sized tensor saved for the backward, path selection, and a forward without host synchronisation."""
import math
from unittest import mock

import numpy as np
import pytest
import torch

import edge_dropout_reference as R
import unfused_reference as U
from test_gpu_gated_dropout import KEY, _fixed_key, _graph, _key, _reference

pytestmark = pytest.mark.gpu


def _layer(H, D, T, agg, p, seed, **kw):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    return P.GatedMessagePassingLayer(H, D, T, agg, dropout_rate=p, **kw).cuda().train()


def _edge_graph(gen, n):
    """types with 0, 127, 128 and 129 edges, and a target (node 5) with 300 in-edges of type 2"""
    counts = [0, 127, 128, 129]
    adj = [(torch.randint(0, n, (c,), generator=gen), torch.randint(0, n, (c,), generator=gen)) for c in counts]
    s, t = adj[2]
    adj[2] = (torch.cat([s, torch.randint(0, n, (300,), generator=gen)]), torch.cat([t, torch.full((300,), 5, dtype=torch.int64)]))
    return adj


@pytest.mark.parametrize("H,D", [(32, 32), (64, 64), (128, 64), (64, 256), (256, 256), (64, 16)])
def test_masked_messages_vs_float64(H, D):
    from ptgnn_b200 import autograd as A
    from ptgnn_b200.edgeplan import EdgePlan

    gen = torch.Generator().manual_seed(21)
    n, p = 700, 0.3
    adj = _edge_graph(gen, n)
    E = sum(int(s.shape[0]) for s, _ in adj)
    h = torch.randn(n, H, generator=gen)
    W = [torch.randn(D, H, generator=gen) / math.sqrt(H) for _ in adj]
    plan = EdgePlan([(s.cuda(), t.cuda()) for s, t in adj], n)
    got = A.edge_messages_dropout(plan, h.cuda(), [w.cuda() for w in W], _key(), p).double().cpu()

    # the kernel multiplies W_t (mask * h[src]) by 1 / (1 - p) after the products: the GEMM bound of the scaled rows, plus the
    # rounding of that multiply
    rows = torch.cat([h[s] for s, _ in adj]).double() * torch.from_numpy(R.keep_mask(KEY, E, H, p)).double() * R.scale(p)
    off = np.cumsum([0] + [int(s.shape[0]) for s, _ in adj])
    ident = [(torch.arange(off[t], off[t + 1]), tg) for t, (_, tg) in enumerate(adj)]
    _, ref, err = U.fp32_messages(rows, ident, W, False, mode="tc")
    bound = err + U.U * (ref.abs() + err)
    assert got.shape == ref.shape
    bad = (got - ref).abs() > bound
    assert not bool(bad.any()), f"{int(bad.sum())} elements outside the bound, max error {float((got - ref).abs().max()):.3e}"


@pytest.mark.parametrize("agg", ["sum", "mean", "max", "min"])
@pytest.mark.parametrize("H,D", [(64, 64), (128, 64)])
def test_forward_vs_float64(agg, H, D):
    gen = torch.Generator().manual_seed(23)
    n, counts, p = 900, [2500, 0, 1200, 40], 0.1
    adj = _graph(gen, n, counts)
    layer = _layer(H, D, len(counts), agg, p, 24)
    h = torch.randn(n, H, generator=gen)
    E = sum(int(s.shape[0]) for s, _ in adj)
    with _fixed_key(), torch.no_grad(), mock.patch("ptgnn_b200.autograd.gated_forward_composed", side_effect=AssertionError("composed")):
        got = layer(h.cuda(), [(s.cuda(), t.cuda()) for s, t in adj]).double().cpu()
    ref, _, _ = _reference(layer, h, adj, agg, p, R.keep_mask(KEY, E, H, p))
    ref = ref.detach()
    # 3xTF32 messages (fp32-exact up to ~2^-21 of the message magnitude), fp32 reduce and the fp32 GRU: the bound of the fused-path test
    bound = 2e-5 + 2e-6 * ref.abs()
    err = (got - ref).abs()
    assert bool((err <= bound).all()), f"max error {float(err.max()):.3e}"


@pytest.mark.parametrize("agg,H,D", [("sum", 64, 64), ("mean", 64, 64), ("max", 64, 64), ("min", 64, 64), ("max", 32, 32),
                                     ("sum", 256, 256), ("min", 64, 256), ("mean", 256, 32), ("max", 128, 64)])
def test_gradients_vs_float64_autograd(agg, H, D):
    gen = torch.Generator().manual_seed(25)
    n, counts, p = 300, [900, 0, 400, 20], 0.1
    adj = _graph(gen, n, counts)
    layer = _layer(H, D, len(counts), agg, p, 26)
    h = torch.randn(n, H, generator=gen)
    g = torch.randn(n, H, generator=gen)
    E = sum(int(s.shape[0]) for s, _ in adj)
    hd = h.cuda().requires_grad_(True)
    with _fixed_key(), mock.patch("ptgnn_b200.autograd.gated_forward_composed", side_effect=AssertionError("composed")):
        out = layer(hd, [(s.cuda(), t.cuda()) for s, t in adj])
        (out * g.cuda()).sum().backward()
    ref, x, params = _reference(layer, h, adj, agg, p, R.keep_mask(KEY, E, H, p))
    (ref * g.double()).sum().backward()

    def close(got, want, what, tol=1e-4):
        got, want = got.detach().cpu().double(), want.detach().cpu().double()
        scale = max(1.0, float(want.abs().max()))
        err = float((got - want).abs().max()) / scale
        assert err <= tol, f"{what}: max error {err:.3e} (scaled)"

    close(out, ref, "output")
    close(hd.grad, x.grad, "d h")
    named = dict(layer.named_parameters())
    for k, v in params.items():
        close(named["_GatedMessagePassingLayer__" + k].grad, v.grad, k)


def test_reproducible_and_fresh_masks_and_p_one():
    gen = torch.Generator().manual_seed(27)
    n, counts, H = 400, [1500, 600], 64
    adj = [(s.cuda(), t.cuda()) for s, t in _graph(gen, n, counts)]
    h = torch.randn(n, H, generator=gen).cuda()
    layer = _layer(H, H, 2, "sum", 0.1, 28)

    def run():
        hd = h.clone().requires_grad_(True)
        out = layer(hd, adj)
        out.square().sum().backward()
        grads = [hd.grad.clone()] + [q.grad.clone() for q in layer.parameters()]
        layer.zero_grad()
        return out.detach(), grads

    torch.manual_seed(11)
    a, ga = run()
    b, _ = run()
    torch.manual_seed(11)
    c, gc = run()
    assert torch.equal(a, c) and all(torch.equal(x, y) for x, y in zip(ga, gc))
    assert not torch.equal(a, b)

    drop_all = _layer(H, H, 2, "max", 1.0, 28)
    with torch.no_grad():
        got = drop_all(h, adj)
        gru = drop_all._GatedMessagePassingLayer__state_update
        want = gru(torch.zeros(n, H, device="cuda"), h)
    assert torch.allclose(got, want, atol=1e-5, rtol=0)


def _typilus_stack(T):
    import ptgnn_b200 as P

    torch.manual_seed(31)
    mp = P.GatedMessagePassingLayer(64, 64, T, "max", dropout_rate=0.1)
    r = P.ConcatResidualLayer(64)
    return [r.pass_through_dummy_layer()] + [mp] * 7 + [r, P.GatedMessagePassingLayer(128, 64, T, "max", dropout_rate=0.1)]


def _varmisuse_stack(T):
    import ptgnn_b200 as P

    torch.manual_seed(32)
    mp = P.GatedMessagePassingLayer(64, 64, T, "sum", dropout_rate=0.01)
    glob = P.GruGlobalStateUpdate(P.WeightedSumVarSizedElementReduce(64), 64, 64, dropout_rate=0.1)
    return [mp, mp, glob, mp]


class _Identity(torch.nn.Module):
    def forward(self, x):
        return x


@pytest.mark.parametrize("stack", [_typilus_stack, _varmisuse_stack])
def test_stacks_train_without_saving_edge_sized_tensors(stack):
    import ptgnn_b200 as P
    from ptgnn_b200.edgeplan import EdgePlan

    gen = torch.Generator().manual_seed(33)
    n, counts, graphs = 3000, [7000, 2500, 400], 30
    adj = [(s.cuda(), t.cuda()) for s, t in _graph(gen, n, counts)]
    E = sum(int(s.shape[0]) for s, _ in adj)
    gnn = P.GraphNeuralNetwork(stack(len(counts)), _Identity(), False, False).cuda().train()
    h0 = torch.randn(n, 64, generator=gen).cuda()
    n2g = torch.sort(torch.randint(0, graphs, (n,), generator=gen)).values.cuda()
    saved, edge_ids = [], []
    block_plan = EdgePlan.block_plan

    def spy(self, *args, **kwargs):
        edge_ids.append(bool(kwargs.get("edge_ids", args[0] if args else False)))
        return block_plan(self, *args, **kwargs)

    def pack(t):
        saved.append(tuple(t.shape))
        return t

    with mock.patch("ptgnn_b200.autograd.gated_forward_composed", side_effect=AssertionError("composed")), \
            mock.patch.object(EdgePlan, "block_plan", spy), torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        out = gnn.gnn(h0, adj, None, n2g, {}, {})
        target = torch.randn(out.shape, generator=gen).cuda()
        loss = ((out - target) ** 2).mean()
    loss.backward()
    assert math.isfinite(float(loss.detach())) and float(loss.detach()) > 0
    grads = [q.grad for q in gnn.parameters()]
    assert all(gr is not None and bool(torch.isfinite(gr).all()) for gr in grads)
    assert saved and not any(len(s) >= 1 and s[0] == E for s in saved), saved
    assert not any(edge_ids), "no layer of these stacks reads the block plan's edge ids"


def test_path_selection():
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(35)
    n, counts = 500, [1500, 300]
    adj = [(s.cuda(), t.cuda()) for s, t in _graph(gen, n, counts)]
    h = torch.randn(n, 64, generator=gen).cuda().requires_grad_(True)
    layer = _layer(64, 64, 2, "sum", 0.2, 36)
    assert not layer.edge_dropout_active
    with mock.patch("ptgnn_b200.autograd.gated_forward_composed", side_effect=AssertionError("composed")):
        layer(h, adj).sum().backward()
    assert torch.isfinite(h.grad).all() and h.grad.abs().sum() > 0
    assert _layer(64, 128, 2, "sum", 0.2, 36).edge_dropout_active

    from ptgnn_b200 import autograd as A

    feats = [torch.randn(int(s.shape[0]), 8, generator=gen).cuda() for s, _ in adj]
    with_features = _layer(64, 64, 2, "sum", 0.2, 37, edge_feature_dimension=8)
    with mock.patch("ptgnn_b200.autograd.gated_forward_composed", wraps=A.gated_forward_composed) as composed:
        with_features(h, adj, edge_features=feats).sum().backward()
    assert composed.call_count == 1


def test_forward_does_not_synchronise():
    gen = torch.Generator().manual_seed(39)
    n, counts, H = 800, [3000, 900], 64
    adj = [(s.cuda(), t.cuda()) for s, t in _graph(gen, n, counts)]
    h = torch.randn(n, H, generator=gen).cuda().requires_grad_(True)
    layer = _layer(H, H, 2, "max", 0.1, 40)
    layer(h, adj)                               # the plan and the weight cache
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = layer(h, adj)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(out).all()
