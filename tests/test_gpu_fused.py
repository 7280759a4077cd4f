"""The fused gather -> per-type Linear -> segmented-reduce kernel (csrc/fused_mp.cu): block plan bit-exact against the oracle,
layers through the fused path against the oracle (fp32: 1e-5; bf16: the bars of test_gpu_bf16.py), fused == unfused."""
import os

import numpy as np
import pytest
import torch

from helpers import assert_close, gated_oracle_args, random_adjacency
from oracle import ptgnn_oracle as O

pytestmark = pytest.mark.gpu


def _dev(adj):
    return [(s.cuda(), t.cuda()) for s, t in adj]


def _mlp_ref(layer, h, adj, agg, use_target=True):
    sd = {k: v.clone().cpu() for k, v in layer.state_dict().items()}
    p = "_MlpMessagePassingLayer__"
    T = len(adj)
    return O.mlp_layer_forward(
        h, adj, [torch.empty(a[0].shape[0], 0) for a in adj],
        [[sd[f"{p}edge_message_transformation_layers.{t}._MLP__mlp_modules.1.weight"]] for t in range(T)], agg,
        use_target_state_as_message_input=use_target,
        ln_weight=sd[p + "state_update.0.weight"], ln_bias=sd[p + "state_update.0.bias"],
        dense_weight=sd[p + "state_update.1.weight"], dense_bias=sd[p + "state_update.1.bias"])


@pytest.mark.parametrize("n,counts", [(1000, [3000, 0, 1500, 700]), (5000, [20000, 1, 130]), (17, [5]), (240, [900, 900])])
def test_block_plan_bit_exact(n, counts):
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(n)
    adj = random_adjacency(gen, n, counts)
    plan = P.EdgePlan(_dev(adj), n)
    bp = plan.block_plan()
    B = plan.block_targets
    ref = O.block_plan(adj, n, B)
    _, group_off, src_f, tl_f, _ = plan._block
    E = sum(counts)
    assert np.array_equal(group_off.cpu().numpy(), ref["group_off"])
    assert np.array_equal(src_f.cpu().numpy()[:E], ref["src_f"])
    assert np.array_equal(tl_f.cpu().numpy()[:E], ref["tl_f"])
    assert bp.block_targets == B and 8 <= B <= 176       # fused_mp.cuh kMaxBlockTargets: agg_s must fit H100 shared memory
    assert int(P._native.lib().ptgnn_b200_block_plan_block_targets(10**8)) == 176   # large graphs get the largest block


@pytest.mark.parametrize("block_targets", [8, 24, 88, 176])
@pytest.mark.parametrize("n,counts", [(1000, [3000, 0, 1500, 700]), (5000, [20000, 1, 130]), (17, [5]), (240, [900, 900])])
def test_block_plan_bit_exact_explicit_block_targets(n, counts, block_targets):
    """EdgePlan(block_targets=B) builds its block plan at B (n = 1000, 5000, 17 are not multiples of any of these B; 240 is one
    of 8 and 24 but not of 88 or 176)."""
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(n)
    adj = random_adjacency(gen, n, counts)
    plan = P.EdgePlan(_dev(adj), n, block_targets=block_targets)
    bp = plan.block_plan()
    assert plan.block_targets == block_targets and bp.block_targets == block_targets
    ref = O.block_plan(adj, n, block_targets)
    _, group_off, src_f, tl_f, _ = plan._block
    E = sum(counts)
    assert np.array_equal(group_off.cpu().numpy(), ref["group_off"])
    assert np.array_equal(src_f.cpu().numpy()[:E], ref["src_f"])
    assert np.array_equal(tl_f.cpu().numpy()[:E], ref["tl_f"])


@pytest.mark.parametrize("agg", ["sum", "mean", "max", "min"])
@pytest.mark.parametrize("n,H,counts", [
    (3001, 128, [9000, 9000, 5000, 1, 130, 0, 2000]),
    (1000, 64, [3000, 1500, 0, 700]),
    (300, 128, [40000]),                 # in-degree 133 for every target: groups split into several sub-groups
    (5, 128, [3, 0]),
])
def test_fused_gated_vs_oracle(agg, n, H, counts):
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(n + H)
    torch.manual_seed(n)
    adj = random_adjacency(gen, n, counts)
    h = torch.randn(n, H, generator=gen)
    layer = P.GatedMessagePassingLayer(H, 128, len(counts), agg).cuda().eval()
    assert P._native.lib().ptgnn_b200_fused_supported(0, H, 128) == 1
    ref = O.gated_layer_forward(h, adj, [torch.empty(c, 0) for c in counts], aggregation_fn=agg,
                                **gated_oracle_args({k: v.clone().cpu() for k, v in layer.state_dict().items()}))
    with torch.no_grad():
        got = layer(h.cuda(), _dev(adj))
    # 133-term sums with |agg| ~ 11: the fp32 rounding of the reference's own sequential sum is ~1e-5 there (sqrt(133) adds x
    # half an ulp of 11), so two correct fp32 implementations differ by more than 1e-5 on this one case -> 3e-5
    tol = 3e-5 if (counts == [40000] and agg in ("sum", "mean")) else 1e-5
    assert_close(got, ref, tol=tol, what=f"fused gated {agg} N={n} H={H}")


def test_fused_gated_hub_and_isolated_targets():
    """One hub target receiving 3000 edges of one type (many sub-groups, one segment), targets without any edge."""
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(11)
    torch.manual_seed(11)
    n, H = 1500, 128
    src = torch.randint(0, n, (3000,), generator=gen)
    adj = [(src, torch.full((3000,), 777, dtype=torch.int64)),
           (torch.randint(0, n, (500,), generator=gen), torch.randint(0, 300, (500,), generator=gen))]
    h = torch.randn(n, H, generator=gen)
    for agg in ("sum", "max"):
        layer = P.GatedMessagePassingLayer(H, 128, 2, agg).cuda().eval()
        ref = O.gated_layer_forward(h, adj, [torch.empty(3000, 0), torch.empty(500, 0)], aggregation_fn=agg,
                                    **gated_oracle_args({k: v.clone().cpu() for k, v in layer.state_dict().items()}))
        with torch.no_grad():
            got = layer(h.cuda(), _dev(adj))
        # a 3000-term fp32 sum (|partial sums| ~ 50): the reference's own sequential summation carries ~sqrt(3000) x 2^-24 x 50 =
        # 1.6e-4 of rounding noise, so agreement to 5e-5 on the hub row is already inside what fp32 defines; max is exact-ish
        assert_close(got, ref, tol=5e-5 if agg == "sum" else 1e-5, what=f"hub {agg}")


@pytest.mark.parametrize("agg", ["sum", "max", "mean"])
@pytest.mark.parametrize("use_target", [True, False])
@pytest.mark.parametrize("n,Hin,Hout,counts", [(2500, 128, 128, [9000, 9000, 5000, 1]), (900, 64, 64, [4000, 300])])
def test_fused_mlp_vs_oracle(agg, use_target, n, Hin, Hout, counts):
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(n + Hin)
    torch.manual_seed(n + 1)
    adj = random_adjacency(gen, n, counts)
    h = torch.randn(n, Hin, generator=gen)
    layer = P.MlpMessagePassingLayer(Hin, Hout, 128, len(counts), agg, use_target_state_as_message_input=use_target).cuda().eval()
    ref = _mlp_ref(layer, h, adj, agg, use_target)
    with torch.no_grad():
        got = layer(h.cuda(), _dev(adj))
    assert_close(got, ref, what=f"fused mlp {agg} target={use_target}")


def test_fused_equals_unfused_and_is_deterministic(monkeypatch):
    """Same layer through the fused kernel and through the round-1 three-kernel path: both within tolerance of each other;
    max is bit-identical (order-independent); the fused result is run-to-run bit-reproducible."""
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(5)
    torch.manual_seed(5)
    n, H = 4000, 128
    adj = random_adjacency(gen, n, [12000, 8000, 3000])
    h = torch.randn(n, H, generator=gen).cuda()
    for agg in ("sum", "max"):
        layer = P.GatedMessagePassingLayer(H, 128, 3, agg).cuda().eval()
        with torch.no_grad():
            a = layer(h, _dev(adj))
            b = layer(h, _dev(adj))
            monkeypatch.setenv("PTGNN_B200_FP32_MODE", "tf32")
            c = layer(h, _dev(adj))
            monkeypatch.delenv("PTGNN_B200_FP32_MODE")
        assert torch.equal(a, b)
        assert_close(a, c, what=f"fused vs unfused {agg}")


@pytest.mark.parametrize("agg", ["sum", "max"])
@pytest.mark.parametrize("H", [64, 128, 256])
def test_fused_gated_bf16(agg, H):
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(H)
    torch.manual_seed(H)
    n, counts = 2000, [6000, 4000, 0, 900]
    adj = random_adjacency(gen, n, counts)
    h = torch.randn(n, H, generator=gen).to(torch.bfloat16)
    layer = P.GatedMessagePassingLayer(H, 128, len(counts), agg).cuda().eval()
    assert P._native.lib().ptgnn_b200_fused_supported(1, H, 128) == 1
    ref = O.gated_layer_forward(h.float(), adj, [torch.empty(c, 0) for c in counts], aggregation_fn=agg,
                                **gated_oracle_args({k: v.clone().cpu() for k, v in layer.state_dict().items()}))
    with torch.no_grad():
        got = layer(h.cuda(), _dev(adj)).float().cpu()
    rel = ((got - ref).norm() / ref.norm()).item()
    frac = ((got - ref).abs() <= 1e-2 * ref.abs().clamp(min=1)).float().mean().item()
    assert rel <= 1e-2 and frac >= 0.999, f"bf16 fused gated {agg} H={H}: rel L2 {rel:.2e}, within 1e-2: {frac:.4f}"


def test_fused_mlp_bf16():
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(9)
    torch.manual_seed(9)
    n, H, counts = 2000, 128, [6000, 4000, 900]
    adj = random_adjacency(gen, n, counts)
    h = torch.randn(n, H, generator=gen).to(torch.bfloat16)
    layer = P.MlpMessagePassingLayer(H, H, 128, len(counts), "max").cuda().eval()
    ref = _mlp_ref(layer, h.float(), adj, "max")
    with torch.no_grad():
        got = layer(h.cuda(), _dev(adj)).float().cpu()
    rel = ((got - ref).norm() / ref.norm()).item()
    assert rel <= 1e-2, f"bf16 fused mlp: rel L2 {rel:.2e}"


def test_fused_fp16_range_overflow_is_reported():
    """|x| >= 65504 cannot go through the 3xFP16 split: the kernels flag it, the host raises at the next poll."""
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(2)
    n, H = 500, 128
    adj = random_adjacency(gen, n, [2000])
    h = torch.randn(n, H, generator=gen)
    h[3, 5] = 1.0e6
    layer = P.GatedMessagePassingLayer(H, 128, 1, "sum").cuda().eval()
    adj_d = _dev(adj)
    plan = P.EdgePlan(adj_d, n)
    with torch.no_grad(), P.edgeplan.shared_plan(plan):
        layer(h.cuda(), adj_d)
    with pytest.raises(FloatingPointError):
        plan.validate()
    os.environ["PTGNN_B200_FP32_MODE"] = "tf32"      # the 3xTF32 kernels take the same input
    try:
        plan2 = P.EdgePlan(adj_d, n)
        with torch.no_grad(), P.edgeplan.shared_plan(plan2):
            out = layer(h.cuda(), adj_d)
        plan2.validate()
        assert torch.isfinite(out).all()
    finally:
        del os.environ["PTGNN_B200_FP32_MODE"]


def test_out_of_range_index_is_reported():
    import ptgnn_b200 as P

    n = 100
    adj = [(torch.tensor([1, 2, 3]), torch.tensor([4, 5, 100]))]
    plan = P.EdgePlan(_dev(adj), n)
    with pytest.raises(IndexError):
        plan.validate()
