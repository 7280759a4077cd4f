"""The backward reference's bounds on the CPU: the transposed aggregation's bound rejects the fused kernel's unscaled 3xFP16 split of a
small gradient and accepts the scaled one, and the bit-exact split emulation behaves as the kernels' representation."""
import pytest
import torch

import backward_reference as BR
import fused_reference as FR


def _case(gen, n=500, D=128, H=128, T=3, edges=2000):
    adj = [(torch.randint(0, n, (edges,), generator=gen), torch.randint(0, n, (edges,), generator=gen)) for _ in range(T)]
    W = [torch.randn(D, H, generator=gen) / 11.3 for _ in range(T)]
    return adj, W


def test_transposed_bound_rejects_the_unscaled_split_of_small_gradients():
    gen = torch.Generator().manual_seed(5)
    n = 500
    adj, W = _case(gen, n)
    d_agg = torch.randn(n, 128, generator=gen) * 2.0 ** -27
    ref, bound = BR.transposed_aggregate(d_agg, adj, W, n, fused=True)
    unscaled = BR.emulate_transposed_aggregate(d_agg, adj, W, n, 1.0)
    with pytest.raises(AssertionError):
        FR.check_bound(unscaled, ref, bound, "unscaled split at 2^-27")
    scaled = BR.emulate_transposed_aggregate(d_agg, adj, W, n, BR.pow2_scale(d_agg))
    assert FR.check_bound(scaled, ref, bound, "scaled split at 2^-27") <= 1.0
    # at O(1) gradients both splits are within the bound
    big = d_agg * 2.0 ** 27
    ref, bound = BR.transposed_aggregate(big, adj, W, n, fused=True)
    FR.check_bound(BR.emulate_transposed_aggregate(big, adj, W, n, 1.0), ref, bound, "unscaled split at 1")


def test_split_emulation_represents_its_operand():
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(64, 40, generator=gen) * torch.logspace(-30, 4, 40)
    x[0, :4] = torch.tensor([0.0, -0.0, 6e4, -6e4])
    s = BR.pow2_scale(x)
    assert 512 <= float(x.abs().max()) * s < 1024
    v = BR.split_value(x, s)
    # 22 significant bits of the scaled operand, plus 2^-36 absolute in scaled units
    assert bool(((v - x.double()).abs() <= 4 * FR.U * x.double().abs() + FR.ABS_F16 / s).all())
    hi, lo = BR.gather_split(x, torch.tensor([3, 3, 0], dtype=torch.int32), None)
    assert hi.shape == (3, 40) and torch.equal(hi[0], hi[1]) and torch.equal(hi[2], x[0].half())
    assert bool(torch.isinf(BR.gather_split(x[:1] * 2.0, None, None)[0][0, 2]))      # 1.2e5: beyond fp16 without a scale


def test_gru_gate_bound_holds_for_an_fp32_evaluation():
    """The kernel's formulas in fp32 torch ops (libm functions, no fma) fall within the bound; a 1-ulp perturbation of each output
    stays within it too, a 2^-12 relative one does not."""
    gen = torch.Generator().manual_seed(7)
    N, H = 300, 32
    gi = torch.randn(N, 3 * H, generator=gen) * 8
    gh = torch.randn(N, 3 * H, generator=gen) * 8
    h = torch.randn(N, H, generator=gen)
    g = torch.randn(N, H, generator=gen) * 2.0 ** -30
    r = 1 / (1 + torch.exp(-(gi[:, :H] + gh[:, :H])))
    z = 1 / (1 + torch.exp(-(gi[:, H:2 * H] + gh[:, H:2 * H])))
    n_ = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
    dn = g * (1 - z) * (1 - n_ * n_)
    dz = g * (h - n_) * z * (1 - z)
    dr = dn * gh[:, 2 * H:] * r * (1 - r)
    ref = BR.gru_gate_grads(gi, gh, h, g)
    FR.check_bound(torch.cat([dr, dz, dn], 1), *ref["d_gi"], "d_gi")
    FR.check_bound(torch.cat([dr, dz, dn * r], 1), *ref["d_gh"], "d_gh")
    FR.check_bound(g * z, *ref["d_h"], "d_h")
    with pytest.raises(AssertionError):
        FR.check_bound(ref["d_gi"][0] * (1 + 2.0 ** -12), *ref["d_gi"], "perturbed d_gi")
