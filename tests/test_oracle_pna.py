"""CPU: the float32 restatement of the PNA kernel (tests/pna_reference.py) against the fixtures of the unmodified reference
(tests/golden/pna_*.npz), the forward mutants it must reject, and the backward formula against torch.autograd."""
import glob
import os

import numpy as np
import pytest
import torch

import pna_reference as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FORWARD = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "pna_*.npz")))


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    m = torch.from_numpy(z["messages"])
    if bool(z["bf16"]):
        m = m.to(torch.bfloat16)
    return dict(messages=m, targets=torch.from_numpy(z["targets"]), n=int(z["num_nodes"]), delta=float(z["delta"]),
                out=torch.from_numpy(z["out"]), z=z)


def mismatch(got, ref, D, bf16=False):
    """(sum, mean, max and min columns equal bit for bit, NaN included, and the std within one rounding of the message dtype: torch's
    float32 CPU sqrt is not always correctly rounded, the restatement's (and the kernel's) is; scaled columns within the bound)."""
    s_equal = torch.equal(torch.isnan(got[:, :5 * D]), torch.isnan(ref[:, :5 * D])) and torch.equal(
        torch.nan_to_num(got[:, :4 * D], nan=0.0), torch.nan_to_num(ref[:, :4 * D], nan=0.0))
    std_err = (torch.nan_to_num(got[:, 4 * D:5 * D]).double() - torch.nan_to_num(ref[:, 4 * D:5 * D]).double()).abs()
    s_equal = s_equal and bool((std_err <= (2.0 ** -8 if bf16 else 2 * R.U) * torch.nan_to_num(ref[:, 4 * D:5 * D]).double()).all())
    finite = ~torch.isnan(ref)
    err = (got.double() - ref.double()).abs()
    within = bool(((err <= R.scaled_bound(torch.nan_to_num(ref), D)) | ~finite | (err == 0))[:, 5 * D:].all())
    return s_equal, within


def test_fixtures_cover_the_cases():
    assert len(FORWARD) == 10
    f = load("pna_d64_delta2.3")
    counts = torch.bincount(f["targets"], minlength=f["n"])
    assert (counts == 0).sum() >= 4 and (counts == 1).sum() >= 3 and counts.max() >= 300
    assert torch.isnan(f["messages"]).sum() == 1
    assert torch.isnan(f["out"]).any()
    assert abs(f["delta"] - 2.3) < 1e-12 and float(np.float32(2.3)) != 2.3


@pytest.mark.parametrize("name", FORWARD)
def test_restatement_reproduces_the_reference(name):
    f = load(name)
    got, _, _ = R.emulate_forward(f["messages"], f["targets"], f["n"], f["delta"])
    D = f["messages"].shape[1]
    s_equal, within = mismatch(got, f["out"], D, name.endswith("bf16"))
    assert s_equal, f"{name}: S columns differ from the reference"
    assert within, f"{name}: scaled columns outside the bound"
    if name.endswith("bf16"):      # S is bf16-representable, the scaled blocks are not rounded
        S = got[:, :5 * D]
        assert torch.equal(torch.nan_to_num(S.to(torch.bfloat16).float()), torch.nan_to_num(S))


def same_args(f, amx, amn):
    """The winning edge ids equal torch_scatter's (recorded with the fixture; the gradient fixture has none)."""
    z = f["z"]
    return "arg_max" not in z or (torch.equal(amx, torch.from_numpy(z["arg_max"]).long())
                                  and torch.equal(amn, torch.from_numpy(z["arg_min"]).long()))


@pytest.mark.parametrize("name", FORWARD)
def test_restatement_picks_the_reference_winners(name):
    f = load(name)
    _, amx, amn = R.emulate_forward(f["messages"], f["targets"], f["n"], f["delta"])
    assert same_args(f, amx, amn)


@pytest.mark.parametrize("mutant", R.MUTANTS)
def test_forward_mutants_fail(mutant):
    """Each mutant changes the output (the mean and relu mutants) or the winning edge ids (last-occurrence ties: the values are the
    same, the gradient's routing is not) on the forward fixtures."""
    failed = 0
    for name in FORWARD:
        f = load(name)
        got, amx, amn = R.emulate_forward(f["messages"], f["targets"], f["n"], f["delta"], mutant=mutant)
        failed += not (all(mismatch(got, f["out"], f["messages"].shape[1], name.endswith("bf16"))) and same_args(f, amx, amn))
    expected = {"clamped_count": 10, "fmaxf_relu": 9, "last_tie": 9}[mutant]     # NaN and ties: every fixture but the gradient one
    assert failed >= expected, f"mutant {mutant} passed {len(FORWARD) - failed} of {len(FORWARD)} fixtures"


def test_argmax_ties_pick_the_first_edge():
    f = load("pna_d8_delta1")
    targets = f["targets"]
    _, amx, amn = R.emulate_forward(f["messages"], targets, f["n"], f["delta"])
    tied = (targets == 7).nonzero().flatten()
    # rows 1, 3 and 5 of target 7 are equal: where one of them wins, the first of them does
    for arg in (amx, amn):
        assert not bool(torch.isin(arg[7], tied[3:6:2]).any())
    counts = torch.bincount(targets, minlength=f["n"])
    assert bool((amx[counts == 0] == targets.numel()).all())


def test_layer_forward_gradient_matches_the_reference():
    f = load("pna_grad_d8")
    z = f["z"]
    x = f["messages"].clone().requires_grad_(True)
    out = R.layer_forward(x, f["targets"], f["n"], f["delta"])
    assert torch.equal(out.detach(), f["out"])      # the reference's own operations, its sqrt included
    out.backward(torch.from_numpy(z["d_out"]))
    ref = torch.from_numpy(z["d_messages"])
    assert ((x.grad - ref).abs().max() / ref.abs().max()).item() <= 1e-6


def _backward_case(seed, D=16):
    gen = torch.Generator().manual_seed(seed)
    counts = [0, 1, 2, 300, 0, 17, 1, 33] + torch.randint(0, 12, (60,), generator=gen).tolist()
    t = torch.cat([torch.full((c,), v, dtype=torch.int64) for v, c in enumerate(counts)])
    t = t[torch.randperm(t.numel(), generator=gen)]
    m = torch.randn(t.numel(), D, generator=gen) + 0.5
    return m, t, len(counts), torch.randn(len(counts), 15 * D, generator=gen)


@pytest.mark.parametrize("seed", [1, 2])
def test_backward_formula_matches_autograd(seed):
    m, t, n, d_out = _backward_case(seed)
    delta = 2.3
    x = m.clone().requires_grad_(True)
    R.layer_forward(x, t, n, delta).backward(d_out)
    out, amx, amn = R.emulate_forward(m, t, n, delta)
    got = R.emulate_backward(m, t, n, delta, out, amx, amn, d_out)
    scale = x.grad.abs().max()
    assert ((got - x.grad).abs().max() / scale).item() <= 1e-5
    dropped = R.emulate_backward(m, t, n, delta, out, amx, amn, d_out, drop_mean_term=True)
    assert ((dropped - x.grad).abs().max() / scale).item() > 1e-3, "the mean term of the std gradient is not visible"


def test_backward_formula_matches_the_reference_gradient():
    f = load("pna_grad_d8")
    z = f["z"]
    out, amx, amn = R.emulate_forward(f["messages"], f["targets"], f["n"], f["delta"])
    got = R.emulate_backward(f["messages"], f["targets"], f["n"], f["delta"], out, amx, amn, torch.from_numpy(z["d_out"]))
    ref = torch.from_numpy(z["d_messages"])
    assert ((got - ref).abs().max() / ref.abs().max()).item() <= 1e-5
