"""graph2seq decoder on the CPU: the float64 restatement (decoder_reference.py) against the reference's own outputs and autograd
gradients (tests/golden/decoder_*.npz, written by tests/golden/generate_decoder_golden.py), the native class's constructor, parameter
order and state_dict against the reference's, the refusals that need no GPU, and the overlay's opt-in binding of the reference's
decoder."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import decoder_reference as DR
from oracle.refimport import reference_available

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["decoder_h32_l1", "decoder_h32_l4", "decoder_h128_l4", "decoder_h128_l7"]
INPUTS = ("memories", "origin", "initial_states", "target_token_ids", "copyable_elements_idxs", "copyable_elements_sample_idxs",
          "target_lengths")


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: torch.from_numpy(z[k]) if z[k].ndim else z[k].item() for k in z.files}


def params64(f):
    return {k[4:]: v.double().requires_grad_(True) for k, v in f.items() if k.startswith("sd::")}


def scaled(a, b):
    return ((a.double() - b.double()).abs() / b.double().abs().clamp(min=1)).max().item()


def grads_close(a, b, what):
    """The bar of test_gpu_backward.py: max error over max(1, max |ref|), and rel. L2, both <= 1e-4."""
    a, b = a.double(), b.double()
    s = (a - b).abs().max().item() / max(1.0, b.abs().max().item())
    rel = ((a - b).norm() / b.norm().clamp(min=1e-30)).item()
    assert s <= 1e-4 and rel <= 1e-4, f"{what}: scaled {s:.2e} rel L2 {rel:.2e}"


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_reference_decoder(name):
    f = load(name)
    sd = params64(f)
    mem, origin, h0, tokens, ce, ces, lengths = (f[k] for k in INPUTS)
    with torch.no_grad():
        copy_lp, target_lp, state = DR.compute_logprobs(sd, h0.double(), mem.double(), origin, tokens[:, :-1])
    for got, key in ((copy_lp, "copy_logprobs"), (target_lp, "target_logprobs"), (state, "gru_state")):
        err = scaled(got, f[key])
        assert err <= 1e-5, f"{name} {key}: float64 restatement vs fp32 reference {err:.2e}"
    m64, h64 = mem.double().requires_grad_(True), h0.double().requires_grad_(True)
    loss = DR.loss(sd, f["unk_id"], m64, origin, h64, tokens, ce, ces, lengths)
    assert abs(loss.item() - float(f["loss"])) <= 1e-5 * max(1.0, abs(float(f["loss"]))), f"{name}: loss"
    loss.backward()
    grads_close(m64.grad, f["grad::memories"], f"{name} d memories")
    grads_close(h64.grad, f["grad::initial_states"], f"{name} d initial_states")
    for k, v in sd.items():
        grads_close(v.grad, f["grad::" + k], f"{name} d {k}")


def test_fixtures_have_the_intended_structure():
    for name in NAMES:
        f = load(name)
        origin, tokens, ces, lengths = f["origin"], f["target_token_ids"], f["copyable_elements_sample_idxs"], f["target_lengths"]
        G, L = tokens.shape[0], tokens.shape[1] - 1
        counts = torch.bincount(origin, minlength=G)
        assert 0 in counts[:-1].tolist() and counts[-1] > 0, f"{name}: a sample without memories, not the last"
        assert {1, 31, 33} <= set(counts.tolist()) and counts.max() > 64 or name == "decoder_h128_l4", name
        assert not bool((origin[1:] >= origin[:-1]).all()), f"{name}: unsorted origin"
        with_copy = torch.zeros(G * L, dtype=torch.bool)
        with_copy[ces] = True
        unk = (tokens[:, 1:] == f["unk_id"]).flatten()
        assert bool((unk & with_copy).any()) and bool((unk & ~with_copy).any()), f"{name}: UNK with and without a valid copy"
        assert bool((~with_copy).any()), f"{name}: a step without a copyable element"
        assert bool((lengths < L + 1).any()), f"{name}: lengths shorter than the batch maximum"
    assert set(torch.bincount(load("decoder_h128_l4")["origin"]).tolist()) >= {0, 1, 31, 33, 65}


def test_restatement_reproduces_reference_fp32_on_bf16_rounded_memories():
    f = load("decoder_h128_l7_bf16ac")
    with torch.no_grad():
        copy_lp, target_lp, _ = DR.compute_logprobs(params64(f), f["initial_states"].double(), f["memories"].double(), f["origin"],
                                                    f["target_token_ids"][:, :-1])
    assert scaled(copy_lp, f["copy_fp32_rounded_inputs"]) <= 1e-5 and scaled(target_lp, f["target_fp32_rounded_inputs"]) <= 1e-5
    gap = (f["copy_autocast"] - f["copy_fp32_rounded_inputs"]).abs().max().item()
    assert gap > 1e-3, "the autocast fixture must differ from the fp32 one (the reference's bf16 path ran)"


def test_native_class_matches_reference_parameters_and_refuses_without_a_gpu():
    import ptgnn_b200 as P

    torch.manual_seed(0)
    m = P.GruCopyingDecoder(50, 16, 32, 24, unk_id=0, dropout_rate=0.2)
    assert sorted(m.state_dict()) == sorted(DR.P + k for k in DR.PARAMS)
    with pytest.raises(NotImplementedError, match="at most 8 steps"):
        m._compute_logprobs(torch.zeros(2, 32), torch.zeros(3, 24), torch.zeros(3, dtype=torch.int64), torch.zeros(2, 9, dtype=torch.int64))
    with pytest.raises(NotImplementedError, match="fp32 memories only"):
        m._compute_logprobs(torch.zeros(2, 32), torch.zeros(3, 24, dtype=torch.bfloat16), torch.zeros(3, dtype=torch.int64),
                            torch.zeros(2, 7, dtype=torch.int64))


@pytest.mark.skipif(not reference_available(), reason="the reference tree is not available")
def test_native_class_matches_reference_constructor_seeded_values_and_state_dict():
    code = f"""
import inspect, sys, torch
sys.path.insert(0, {ROOT!r})
from oracle.refimport import import_reference
import_reference()
from ptgnn.neuralmodels.sequence.grucopydecoder import GruCopyingDecoder as Ref
import ptgnn_b200 as P
params = lambda cls: [(p.name, p.kind, p.default) for p in inspect.signature(cls).parameters.values()]
assert params(Ref) == params(P.GruCopyingDecoder), (params(Ref), params(P.GruCopyingDecoder))
assert params(Ref._compute_logprobs) == params(P.GruCopyingDecoder._compute_logprobs)
assert params(Ref.forward) == params(P.GruCopyingDecoder.forward)
torch.manual_seed(3)
ref = Ref(300, 48, 128, 64, 0, 0.2)
torch.manual_seed(3)
nat = P.GruCopyingDecoder(300, 48, 128, 64, 0, 0.2)
assert list(ref.state_dict()) == list(nat.state_dict()), (list(ref.state_dict()), list(nat.state_dict()))
assert all(torch.equal(ref.state_dict()[k], v) for k, v in nat.state_dict().items()), "one seed, the same parameters"
torch.manual_seed(4)
other = Ref(300, 48, 128, 64, 0, 0.2)
nat.load_state_dict(other.state_dict())
assert all(torch.equal(other.state_dict()[k], v) for k, v in nat.state_dict().items())
print("ok")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.skipif(not reference_available(), reason="the reference tree is not available")
def test_overlay_binds_the_decoder_only_when_asked():
    code = f"""
import sys
sys.path.insert(0, {ROOT!r})
from oracle.refimport import import_reference
import_reference()
import ptgnn.neuralmodels.sequence.grucopydecoder as D
Ref = D.GruCopyingDecoder
import ptgnn.implementations.graph2seq.graph2seq as g2s          # imported before the overlay
import ptgnn_b200 as P
import ptgnn_b200.overlay as ov
r = ov.install(force_torch_scatter=True)
assert r["decoder"] is False and D.GruCopyingDecoder is Ref
ov.uninstall()
r = ov.install(force_torch_scatter=True, native_decoder=True)
assert r["decoder"] is True
assert sys.modules["ptgnn.neuralmodels.sequence.grucopydecoder"] is D, "the reference's module stays in place"
assert D.GruCopyingDecoder is P.GruCopyingDecoder
assert g2s.GruCopyingDecoderModel is D.GruCopyingDecoderModel and g2s.DecoderData is D.DecoderData
from dpu_utils.mlutils import Vocabulary
model = D.GruCopyingDecoderModel(hidden_size=32, embedding_size=16, memories_hidden_dim=24)
model._GruCopyingDecoderModel__output_vocabulary = Vocabulary.create_vocabulary(["a", "b"], max_size=10, count_threshold=0)
assert type(model.build_neural_module()) is P.GruCopyingDecoder
ov.uninstall()
assert D.GruCopyingDecoder is Ref and type(model.build_neural_module()) is Ref
print("ok")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr
