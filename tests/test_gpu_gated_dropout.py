"""GatedMessagePassingLayer in training mode with per-edge dropout on the fused kernel (ptgnn_b200/csrc/edge_dropout.cuh): the mask
bits against the numpy restatement, the block plan's edge ids, the forward and the gradients against a float64 restatement of
gatedmessagepassing.py:46-69 with the same mask, reproducibility, and a training step through the container."""
import math
from unittest import mock

import numpy as np
import pytest
import torch

import edge_dropout_reference as R
from helpers import random_adjacency

pytestmark = pytest.mark.gpu

KEY = (0x2545F491, 0x6C8E9CF5)


def _key():
    return torch.tensor(np.array(KEY, dtype=np.uint32).view(np.int32), device="cuda")


def _fixed_key():
    return mock.patch("ptgnn_b200.autograd.draw_dropout_key", lambda device: _key())


def _graph(gen, n, counts):
    """random edges, plus targets without edges (the last 7 nodes) and one target with 150 edges of type 0 (groups longer than 64)"""
    adj = random_adjacency(gen, n - 7, counts)
    if counts[0] > 0:
        s, t = adj[0]
        hub = torch.randint(0, n, (150,), generator=gen)
        adj[0] = (torch.cat([s, hub]), torch.cat([t, torch.full((150,), 3, dtype=torch.int64)]))
    return adj


def _reference(layer, h, adj, agg, p, mask):
    """float64 gatedmessagepassing.py:46-69 with the dropout mask `mask` [E, H] (cat(types) order)"""
    sd = {k.split("__", 1)[1]: v.detach().double().cpu() for k, v in layer.state_dict().items()}
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    x = h.detach().double().cpu().clone().requires_grad_(True)
    n = x.shape[0]
    msgs, tgts, off = [], [], 0
    for t, (s, tg) in enumerate(adj):
        m = torch.from_numpy(mask[off:off + s.shape[0]]).double() * R.scale(p)
        off += s.shape[0]
        msgs.append((x[s.cpu()] * m) @ params[f"edge_message_transformation_layers.{t}.weight"].t())
        tgts.append(tg.cpu())
    msg, tgt = torch.cat(msgs), torch.cat(tgts)
    D = msg.shape[1]
    if agg in ("sum", "mean"):
        a = torch.zeros(n, D, dtype=torch.float64).index_add(0, tgt, msg)
        if agg == "mean":
            a = a / torch.bincount(tgt, minlength=n).clamp(min=1)[:, None]
    else:
        fill = -math.inf if agg == "max" else math.inf
        a = torch.full((n, D), fill, dtype=torch.float64).scatter_reduce(0, tgt[:, None].expand(-1, D), msg, "amax" if agg == "max" else "amin")
        a = torch.where(torch.isinf(a), torch.zeros_like(a), a)
    out = torch.gru_cell(a, x, params["state_update.weight_ih"], params["state_update.weight_hh"],
                                       params["state_update.bias_ih"], params["state_update.bias_hh"])
    return out, x, params


def _layer(H, T, agg, p, seed):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    return P.GatedMessagePassingLayer(H, 128, T, agg, dropout_rate=p).cuda().train()


@pytest.mark.parametrize("K", [64, 128])
def test_mask_bits_match_the_restatement_in_both_orders(K):
    from ptgnn_b200 import autograd as A
    from ptgnn_b200.edgeplan import EdgePlan

    gen = torch.Generator().manual_seed(1)
    adj = [(s.cuda(), t.cuda()) for s, t in _graph(gen, 500, [1300, 0, 700])]
    plan = EdgePlan(adj, 500)
    E = plan.num_edges
    for p in (0.1, 0.5, 1.0):
        want = R.keep_bits(R.keep_mask(KEY, E, K, p))
        got = A.edge_dropout_bits(_key(), E, K, p).cpu().numpy()
        assert np.array_equal(got, want), p
        eid = plan.block_edge_ids
        got = A.edge_dropout_bits(_key(), E, K, p, eid[:E]).cpu().numpy()
        assert np.array_equal(got, want[eid[:E].cpu().numpy()]), p


def test_block_plan_edge_ids():
    from ptgnn_b200.edgeplan import EdgePlan

    gen = torch.Generator().manual_seed(2)
    adj = [(s.cuda(), t.cuda()) for s, t in _graph(gen, 3000, [9000, 0, 4000, 30])]
    plain, with_ids = EdgePlan(adj, 3000, large_blocks=True), EdgePlan(adj, 3000, large_blocks=True)
    plain.block_plan()
    with_ids.block_plan(edge_ids=True)
    E = plain.num_edges
    for i in (1, 2, 3):
        assert torch.equal(plain._block[i][:E] if i > 1 else plain._block[i], with_ids._block[i][:E] if i > 1 else with_ids._block[i])
    eid = with_ids.block_edge_ids[:E].long()
    assert torch.equal(torch.sort(eid).values, torch.arange(E, device="cuda"))
    assert torch.equal(with_ids._block[2][:E], with_ids.src32[eid])


@pytest.mark.parametrize("agg", ["sum", "mean", "max", "min"])
@pytest.mark.parametrize("H", [64, 128])
def test_forward_vs_float64(agg, H):
    gen = torch.Generator().manual_seed(3)
    n, counts, p = 900, [2500, 0, 1200, 40], 0.1
    adj = _graph(gen, n, counts)
    layer = _layer(H, len(counts), agg, p, 4)
    h = torch.randn(n, H, generator=gen)
    E = sum(int(s.shape[0]) for s, _ in adj)
    mask = R.keep_mask(KEY, E, H, p)
    with _fixed_key(), torch.no_grad():
        got = layer(h.cuda(), [(s.cuda(), t.cuda()) for s, t in adj]).double().cpu()
    ref, _, _ = _reference(layer, h, adj, agg, p, mask)
    ref = ref.detach()
    # per element: the 3xFP16 products and fp32 sums of the fused kernel (|error| ~ 2^-21 of the message magnitude summed into a
    # target, plus 2^-24 |W s| from folding 1 / (1 - p) into the weights), then the fp32 GRU, which is 1-Lipschitz in its input
    # up to the gate weights
    bound = 2e-5 + 2e-6 * ref.abs()
    err = (got - ref).abs()
    assert bool((err <= bound).all()), f"max error {float(err.max()):.3e}"


@pytest.mark.parametrize("agg", ["sum", "mean", "max", "min"])
def test_gradients_vs_float64_autograd(agg):
    gen = torch.Generator().manual_seed(5)
    n, counts, H, p = 300, [900, 0, 400, 20], 128, 0.1
    adj = _graph(gen, n, counts)
    layer = _layer(H, len(counts), agg, p, 6)
    h = torch.randn(n, H, generator=gen)
    g = torch.randn(n, H, generator=gen)
    E = sum(int(s.shape[0]) for s, _ in adj)
    mask = R.keep_mask(KEY, E, H, p)
    hd = h.cuda().requires_grad_(True)
    with _fixed_key():
        out = layer(hd, [(s.cuda(), t.cuda()) for s, t in adj])
    (out * g.cuda()).sum().backward()
    ref, x, params = _reference(layer, h, adj, agg, p, mask)
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
    gen = torch.Generator().manual_seed(7)
    n, counts, H = 400, [1500, 600], 128
    adj = [(s.cuda(), t.cuda()) for s, t in _graph(gen, n, counts)]
    h = torch.randn(n, H, generator=gen).cuda()
    layer = _layer(H, 2, "sum", 0.1, 8)

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

    drop_all = _layer(H, 2, "max", 1.0, 8)
    with torch.no_grad():
        got = drop_all(h, adj)
        gru = drop_all._GatedMessagePassingLayer__state_update
        want = gru(torch.zeros(n, 128, device="cuda"), h)
    assert torch.allclose(got, want, atol=1e-5, rtol=0)


def test_container_trains_without_saving_edge_sized_tensors():
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(12)
    n, counts, H = 2000, [6000, 2000, 100], 128
    adj = [(s.cuda(), t.cuda()) for s, t in _graph(gen, n, counts)]
    E = sum(int(s.shape[0]) for s, _ in adj)
    torch.manual_seed(12)
    layers = [P.GatedMessagePassingLayer(H, H, len(counts), agg, dropout_rate=0.1) for agg in ("sum", "mean", "max", "min")]
    gnn = P.GraphNeuralNetwork(layers * 2, torch.nn.Identity(), False, False).cuda().train()
    h0 = torch.randn(n, H, generator=gen).cuda()
    target = torch.randn(n, H, generator=gen).cuda()
    saved = []

    def pack(t):
        saved.append(tuple(t.shape))
        return t

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        out = gnn.gnn(h0, adj, None, None, {}, {})
        loss = ((out - target) ** 2).mean()
    loss.backward()
    assert math.isfinite(float(loss.detach())) and float(loss.detach()) > 0
    grads = [q.grad for q in gnn.parameters()]
    assert all(gr is not None and bool(torch.isfinite(gr).all()) for gr in grads)
    assert any(float(gr.abs().max()) > 0 for gr in grads)
    assert saved and not any(len(s) >= 1 and s[0] == E for s in saved), saved
