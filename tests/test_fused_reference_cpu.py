"""CPU checks of the fused-kernel test infrastructure: the structured graphs really contain every case they are built for
(recomputed through ``oracle.block_plan``), the float64 reference's bounds are tight enough to reject a kernel that runs
hi*hi alone, and ``EdgePlan(block_targets=...)`` rejects block sizes the fused kernel cannot take."""
import pytest
import torch

import fused_reference as R


@pytest.mark.parametrize("B,T,num_blocks", [(8, 6, 2500), (24, 5, 800), (88, 6, 400), (176, 4, 265), (8, 128, 400)])
def test_structured_graph_covers_the_kernel_branches(B, T, num_blocks):
    adj, N = R.structured_graph(B, T, num_blocks)
    f = R.structure_facts(adj, N, B)
    half = B // 2
    assert f["num_blocks"] == num_blocks
    assert set(R.GROUP_SIZES) <= f["group_sizes"], set(R.GROUP_SIZES) - f["group_sizes"]
    assert f["nb"] == {1, 2, 3, 4}
    assert set(R.SPLITS) <= f["splits"] and f["split_is_n"], set(R.SPLITS) - f["splits"]
    assert f["rows"] == {0, half - 1, half, B - 1}
    assert {15, 31, 47} <= f["batch_cross"] and f["upper_batch_cross"], f["batch_cross"]
    assert f["max_subgroups_per_segment"] >= 3                  # the hub; 63 -> 64 crossings give 2
    assert f["multi_type_targets"] > 0 and R.EMPTY_TYPE in f["empty_types"] and f["empty_type_in_nonempty_block"]
    assert f["empty_block_between"] and f["max_empty_run"] >= 2
    assert f["partial_last_block"] and f["last_row_target"]
    assert f["self_loops"] > 0 and f["duplicates"] > 0 and f["sources_0_and_last"]
    E = sum(int(a[0].shape[0]) for a in adj)
    assert 45_000 <= E <= 55_000


def test_fp32_bound_rejects_dropped_correction_terms():
    """The per-element bound at C_S <= 2^-18 of the mass must fail a kernel that computes hi*hi only (fp16 operands)."""
    gen = torch.Generator().manual_seed(3)
    K, N, T = 128, 600, 3
    adj = [(torch.randint(0, N, (1500,), generator=gen), torch.randint(0, N, (1500,), generator=gen)) for _ in range(T)]
    h = torch.randn(N, K, generator=gen) * 2.0 ** -12
    w = [torch.randn(128, 2 * K, generator=gen) / 16 for _ in range(T)]
    tgt, m, err = R.messages(h, adj, w, True, False)
    assert float(err.max()) > 0
    ref, bound, _ = R.aggregate(tgt, m, err, N, "sum", False)
    hh = h.half().double()
    _, m_hi, _ = R.messages(hh, adj, [x.half().double() for x in w], True, False)
    got = torch.zeros(N, 128, dtype=torch.float64).index_add_(0, tgt, m_hi)
    with pytest.raises(AssertionError):
        R.check_bound(got, ref, bound, "hi*hi only")
    # the exact aggregate itself passes, and so does one perturbed by a quarter of each message's bound
    R.check_bound(ref, ref, bound, "exact")
    R.check_bound(torch.zeros(N, 128, dtype=torch.float64).index_add_(0, tgt, m + 0.25 * err), ref, bound, "perturbed")
    assert R.fp32_message_constant(128, 2) <= 2.0 ** -18


def test_bf16_reference_is_exact_except_near_midpoints():
    gen = torch.Generator().manual_seed(4)
    K, N = 64, 300
    adj = [(torch.randint(0, N, (2000,), generator=gen), torch.randint(0, N, (2000,), generator=gen))]
    h = torch.randn(N, K, generator=gen).to(torch.bfloat16)
    w = [torch.randn(128, K, generator=gen) / 8]
    tgt, m, err = R.messages(h, adj, w, False, True)
    assert torch.equal(m, m.to(torch.bfloat16).double())          # nominal messages are bf16 values
    amb = (err > 0).double().mean().item()
    assert 0 < amb < 0.1, amb                                     # most messages must be matched exactly
    ref, bound, _ = R.aggregate(tgt, m, err, N, "sum", True)
    # the output may be 1 bf16 ulp off where no message is ambiguous: 3 ulps everywhere must fail
    with pytest.raises(AssertionError):
        R.check_bound(ref * (1 + 3 * 2.0 ** -7), ref, bound, "3 ulp off")
    R.check_bound(ref, ref, bound, "exact")


@pytest.mark.parametrize("bad", [0, 4, 12, 100, 184, 256, -8, 8.5])
def test_edge_plan_rejects_block_targets(bad):
    import ptgnn_b200 as P

    adj = [(torch.tensor([0, 1]), torch.tensor([1, 0]))]
    with pytest.raises(ValueError):
        P.EdgePlan(adj, 2, block_targets=bad)

