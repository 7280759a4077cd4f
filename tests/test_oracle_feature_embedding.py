"""CPU: the float64 restatement of LinearFeatureEmbedder (tests/feature_embedding_reference.py) against the reference's fixtures, and the
teeth of the kernel's per-element error bound."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import feature_embedding_reference as R  # noqa: E402
from helpers import load_golden  # noqa: E402

FEATURES = (1, 50, 121)
DIMS = (8, 64, 256)


@pytest.mark.parametrize("act", R.ACTIVATIONS)
@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("F", FEATURES)
def test_restatement_reproduces_the_reference_forward(F, D, act):
    g = load_golden(f"feature_embed_f{F}")
    x, w = torch.from_numpy(g["x"]), torch.from_numpy(g[f"w_d{D}"])
    assert tuple(w.shape) == (D, F)
    ref = torch.from_numpy(g[f"out_d{D}_{act}"]).double()
    exact = R.forward(x, w, act)
    # the reference's own fp32 arithmetic is inside the kernel's bound too
    assert bool(((ref - exact).abs() <= R.bound(x, w, act)).all())
    assert torch.allclose(exact, ref, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("act", R.ACTIVATIONS)
@pytest.mark.parametrize("F", FEATURES)
def test_restatement_reproduces_the_reference_gradients(F, act):
    g = load_golden(f"feature_embed_f{F}")
    x, w = torch.from_numpy(g["x"]), torch.from_numpy(g["w_d64"])
    d_w, d_x = R.gradients(x, w, act, torch.from_numpy(g[f"grad_out_{act}"]))
    for got, key in ((d_w, f"grad_w_{act}"), (d_x, f"grad_x_{act}")):
        ref = torch.from_numpy(g[key]).double()
        assert float((got - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max())), key


@pytest.mark.parametrize("act", R.ACTIVATIONS)
def test_bf16_fixture_within_the_bf16_bound(act):
    g = load_golden("feature_embed_bf16ac")
    x, w = torch.from_numpy(g["x"]), torch.from_numpy(g["w"])
    ref = torch.from_numpy(g[f"out_{act}"]).double()
    assert bool(((ref - R.forward(x, w, act, bf16=True)).abs() <= R.bound(x, w, act, bf16=True)).all())
    # ... and the fp32 bound is far too tight for it: the bf16 bar is not vacuous
    assert not bool(((ref - R.forward(x, w, act)).abs() <= R.bound(x, w, act)).all())


@pytest.mark.parametrize("act", R.ACTIVATIONS)
@pytest.mark.parametrize("F,D", [(1, 8), (50, 64), (121, 256), (512, 64)])
def test_split_emulation_within_bound_and_mutant_outside(F, D, act):
    gen = torch.Generator().manual_seed(F * 1000 + D)
    x, w = torch.randn(300, F, generator=gen) * 3, torch.randn(D, F, generator=gen) / F ** 0.5
    exact, b = R.forward(x, w, act), R.bound(x, w, act)
    assert bool(((R.emulate_split(x, w, act) - exact).abs() <= b).all())
    if act != "relu" or F > 1:          # F = 1, relu: half the products are clamped away, the rest still fail below
        assert not bool(((R.emulate_split(x, w, act, correction=False) - exact).abs() <= b).all())
    assert not bool(((R.forward(x, w * (1 + 2.0 ** -9), act) - exact).abs() <= b).all()), "a 2^-9 weight error must not pass"
