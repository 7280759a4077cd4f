"""The fused aggregation kernel at target blocks larger than 176 (``EdgePlan(large_blocks=True)``, the plan the layers build through
``plan_for``): B = 240, the kernel's largest block, and B = 208, against the float64 reference of tests/fused_reference.py with its
per-element bounds.  Four-tile instances (fp32 K = 128, bf16 K = 256) run on a two-slot ring there, the others on three slots.

The graph is ``fused_reference.structured_graph`` at that B plus one block whose only edges are self-loops: target row B - 1 receives
edges, the last block is partial, groups hold more than 64 edges (one MMA's columns), a type is empty in non-empty blocks, and the graph is one
graph of N > B nodes whose sources come from every block.  Every case runs twice and must be bit-identical."""
import functools

import pytest
import torch

import egc_reference as E
import fused_reference as R
import unfused_reference as UR

pytestmark = pytest.mark.gpu

AGGS = ("sum", "mean", "max", "min")
T = 6
BLOCKS = 140


@functools.lru_cache(maxsize=2)
def _graph(B):
    adj, N = R.structured_graph(B, T, BLOCKS, num_edges=60_000)
    tgt = torch.cat([t for _, t in adj])
    used = torch.zeros((N + B - 1) // B, dtype=torch.bool)
    used[tgt // B] = True
    b = int(torch.nonzero(~used[:-1])[0])                       # an empty full block -> self-loops on every row, nothing else
    loops = torch.arange(b * B, (b + 1) * B)
    s0, t0 = adj[0]
    adj[0] = (torch.cat([s0, loops]), torch.cat([t0, loops]))
    facts = R.structure_facts(adj, N, B)
    assert B - 1 in facts["rows"] and facts["partial_last_block"] and facts["empty_type_in_nonempty_block"]
    assert max(facts["group_sizes"]) > 64 and N > B
    return adj, [(s.cuda(), t.cuda()) for s, t in adj], N


def _mlp(K, agg, ut, act=None, ln=False, seed=0):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    layer = P.MlpMessagePassingLayer(K, 128, 128, T, agg, message_activation=torch.nn.GELU() if act == "gelu" else None,
                                     use_layer_norm=ln, use_dense_layer=False, use_target_state_as_message_input=ut).cuda().eval()
    p = "_MlpMessagePassingLayer__"
    sd = layer.state_dict()
    return layer, [sd[f"{p}edge_message_transformation_layers.{t}._MLP__mlp_modules.1.weight"].cpu() for t in range(T)]


def _run(layer, h, adj_d, N, B):
    import ptgnn_b200 as P

    outs = []
    for _ in range(2):
        plan = P.EdgePlan(adj_d, N, block_targets=B, large_blocks=True)
        with torch.no_grad(), P.edgeplan.shared_plan(plan):
            outs.append(layer(h.cuda(), adj_d))
        plan.validate()
        assert plan.block_targets == B
    assert torch.equal(outs[0], outs[1]), "fused aggregate is not run-to-run bit-identical"
    return outs[0].float().cpu()


def _states(N, K, bf16, seed):
    h = torch.randn(N, K, generator=torch.Generator().manual_seed(seed))
    return h.to(torch.bfloat16) if bf16 else h


CASES = [(B, bf16, agg) for B in (240, 208) for bf16 in (False, True) for agg in AGGS]


@pytest.mark.parametrize("B,bf16,agg", CASES, ids=[f"B{B}-{'bf16' if b else 'fp32'}-{a}" for B, b, a in CASES])
def test_large_block_aggregate(B, bf16, agg):
    K = 256 if bf16 and B == 240 else 128          # fp32 K = 128 and bf16 K = 256: four tiles per slot, two slots
    ut = agg in ("mean", "min")
    adj, adj_d, N = _graph(B)
    h = _states(N, K, bf16, B + K)
    layer, w = _mlp(K, agg, ut, seed=B)
    got = _run(layer, h, adj_d, N, B)
    ref, bound, _ = R.aggregate(*R.messages(h, adj, w, ut, bf16), N, agg, bf16)
    R.check_bound(got, ref, bound, f"B={B} {'bf16' if bf16 else 'fp32'} K={K} use_target={ut} {agg}")


@pytest.mark.parametrize("bf16", [False, True])
def test_large_block_layernorm_epilogue(bf16):
    """Whole-row LayerNorm write-out after a GELU at B = 240: the aggregate's bound carried through GELU and LayerNorm
    (unfused_reference.layer_norm), then the bf16 rounding."""
    B = 240
    adj, adj_d, N = _graph(B)
    h = _states(N, 128, bf16, 51)
    layer, w = _mlp(128, "sum", True, act="gelu", ln=True, seed=51)
    with torch.no_grad():
        for p in layer.parameters():
            if p.dim() == 1:
                p.uniform_(0.5, 1.5, generator=torch.Generator(device="cuda").manual_seed(p.numel()))
    sd = {k: v.double().cpu() for k, v in layer.state_dict().items()}
    ln_w, ln_b = sd["_MlpMessagePassingLayer__state_update.0.weight"], sd["_MlpMessagePassingLayer__state_update.0.bias"]
    got = _run(layer, h, adj_d, N, B)
    y, by, _ = R.aggregate(*R.messages(h, adj, w, True, bf16), N, "sum", bf16, act="gelu", round_bf16=False)
    ref, bound = UR.layer_norm(y, by, ln_w, ln_b, 1e-5)
    if bf16:
        ref, bound = UR.round_bf16(ref, bound)
    R.check_bound(got, ref, bound, f"{'bf16' if bf16 else 'fp32'} LayerNorm at B={B}")


@pytest.mark.parametrize("agg", ["sum", "max"])
def test_large_block_egc_write_out(agg):
    """EGC bases-combining write-out (fp32, 128 -> 128, 8 heads, 4 bases) at B = 240 within the float64 bound of egc_reference."""
    import ptgnn_b200 as P

    B = 240
    adj, adj_d, N = _graph(B)
    torch.manual_seed(5)
    layer = P.EGCMessagePassingLayer(128, 128, T, agg, num_bases=4, num_heads=8).cuda().eval()
    assert P.egc.use_fused(P._native.lib(), False, 128, 128, 8, 4)
    W, cw, cb = E.params_of({k: v.detach().cpu() for k, v in layer.state_dict().items()}, T)
    h = _states(N, 128, False, 5)
    got = _run(layer, h, adj_d, N, B)
    ref, bnd = E.forward64(h, adj, W, cw, cb, agg, 8, 4)
    R.check_bound(got, ref, bnd, f"EGC {agg} B={B}")


def test_layer_plan_uses_the_large_recommendation():
    """plan_for builds with ptgnn_b200_block_plan_large_block_targets (whole waves of 132 CTAs, B <= 240); EdgePlan's default and
    ptgnn_b200_block_plan_block_targets keep B <= 176."""
    import ptgnn_b200 as P

    lib = P._native.lib()
    assert int(lib.ptgnn_b200_block_plan_large_block_targets(10**8)) == 240
    assert int(lib.ptgnn_b200_block_plan_large_block_targets(132 * 240)) == 240
    assert int(lib.ptgnn_b200_block_plan_large_block_targets(204_800)) == 224      # 915 blocks: seven waves
    assert int(lib.ptgnn_b200_block_plan_block_targets(204_800)) == 176
    adj, adj_d, N = _graph(240)
    P.edgeplan.clear_plan_cache()
    plan = P.plan_for(adj_d, N)
    assert plan.block_targets == int(lib.ptgnn_b200_block_plan_large_block_targets(N))
    assert P.EdgePlan(adj_d, N).block_targets <= 176
    for bad in (248, 256, 236):
        with pytest.raises(ValueError):
            P.EdgePlan(adj_d, N, block_targets=bad, large_blocks=True)
    with pytest.raises(ValueError):
        P.EdgePlan(adj_d, N, block_targets=240)
