"""CPU checks of the char-embedder restatement (tests/char_embedding_reference.py) against the reference's fixtures, and of the native
``CharUnitEmbedder``'s interface and overlay binding (DESIGN.md §3.13)."""
import inspect
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import char_embedding_reference as R  # noqa: E402
from helpers import load_golden  # noqa: E402
from oracle.refimport import import_reference, reference_available  # noqa: E402

import ptgnn_b200  # noqa: E402
from ptgnn_b200 import overlay  # noqa: E402

needs_reference = pytest.mark.skipif(not reference_available(), reason="the reference tree is not present")
EMBEDDER_MODULE = "ptgnn.neuralmodels.embeddings.strelementrepresentationmodel"
KEYS = ["conv_l1.weight", "conv_l1.bias", "conv_l2.weight", "conv_l2.bias", "conv_l3.weight"]

# (fixture, output key, D, characters per token)
OUTPUTS = [("char_default", "out_d63", 63, None), ("char_default", "out_d127", 127, None), ("char_default", "out_d128", 128, None),
           ("char_default", "out_minl", 128, 7), ("char_cfg_a", "out", None, None), ("char_cfg_b", "out", None, None)]


def inputs(g, D, L):
    chars = torch.from_numpy(g["chars"])
    return (chars if L is None else chars[:, :L].contiguous()), R.params_of(g, D)


def test_fixture_set():
    g = load_golden("char_default")
    assert [int(x) for x in g["cnn"]] == [256, 3, 128, 3, 3] and int(g["num_chars"]) == 101 and g["chars"].shape[1] == 15
    assert {str(k) for k in g.keys()} >= {"out_d63", "out_d127", "out_d128", "out_minl", "out_bf16ac_d127"}
    cb = load_golden("char_cfg_b")
    assert all("grad::" + R.PRE + k in cb for k in KEYS)


@pytest.mark.parametrize("name,key,D,L", OUTPUTS)
def test_restatement_reproduces_reference_within_bound(name, key, D, L):
    g = load_golden(name)
    chars, ps = inputs(g, D, L)
    ref = torch.from_numpy(g[key]).double()
    assert torch.allclose(R.forward(chars, *ps, dtype=torch.float32).double(), ref, rtol=1e-5, atol=1e-6)
    exact = R.forward(chars, *ps)
    assert bool(((ref - exact).abs() <= R.bound(chars, *ps)).all())
    if L == 7:
        assert R.layers(chars, *ps)[2].shape[-1] == 1          # the minimal L: one output position


def test_bound_rejects_mutants():
    """A dropped tap, a dropped bias or an extra position pooled moves the output far outside the bound."""
    g = load_golden("char_default")
    chars, (w1, b1, w2, b2, w3) = inputs(g, 127, None)
    exact, b = R.forward(chars, w1, b1, w2, b2, w3), R.bound(chars, w1, b1, w2, b2, w3)

    def outside(out):
        return bool(((out - exact).abs() > b).any())

    assert outside(R.forward(chars, w1, torch.zeros_like(b1), w2, b2, w3))
    assert outside(R.forward(chars, w1, b1, w2, torch.zeros_like(b2), w3))
    for w in (w1, w2, w3):
        cut = w.clone()
        cut[..., -1] = 0
        args = [cut if x is w else x for x in (w1, b1, w2, b2, w3)]
        assert outside(R.forward(chars, *args))
    a1, a2, l3 = R.layers(chars, w1, b1, w2, b2, w3)
    padded = torch.nn.functional.conv1d(torch.nn.functional.pad(a2, (0, 1), value=1.0), w3.double())   # one more row pooled
    assert outside(padded.max(dim=-1).values)


@pytest.mark.parametrize("name,key,D,L", OUTPUTS)
def test_fp32_bar_separates_the_split_products_from_the_mutant_without_correction(name, key, D, L):
    g = load_golden(name)
    chars, ps = inputs(g, D, L)
    exact = R.forward(chars, *ps)
    assert R.rel_l2(R.emulate_split(chars, *ps), exact) <= R.FP32_REL_L2 / 10
    assert R.rel_l2(R.emulate_split(chars, *ps, correction=False), exact) > 10 * R.FP32_REL_L2


def test_bf16_emulation_meets_the_n2_bars_and_mutants_do_not():
    """The bf16 rounding emulation reproduces the reference's CPU autocast output; an all-zero output and the bias-dropped mutants fail
    every N2 bar and the emulation bar."""
    g = load_golden("char_default")
    chars, ps = inputs(g, 127, None)
    ac, f = torch.from_numpy(g["out_bf16ac_d127"]), torch.from_numpy(g["out_d127"])
    emu = R.emulate_bf16(chars, *ps)
    assert R.rel_l2(emu, ac) <= R.BF16_EMU_REL_L2 / 10 and all(R.n2_bars(emu, ac, f).values())
    for mutant in (torch.zeros_like(ac), R.emulate_bf16(chars, *ps, drop_bias=1), R.emulate_bf16(chars, *ps, drop_bias=2)):
        assert not any(R.n2_bars(mutant, ac, f).values())
        assert R.rel_l2(mutant, emu) > R.BF16_EMU_REL_L2 and R.rel_l2(mutant, R.forward(chars, *ps)) > 1e-2


def test_bf16_fixture_within_bound():
    g = load_golden("char_default")
    chars, ps = inputs(g, 127, None)
    ref = torch.from_numpy(g["out_bf16ac_d127"]).double()
    assert bool(((ref - R.forward(chars, *ps)).abs() <= R.bound(chars, *ps, bf16=True)).all())


def test_gradients_reproduce_fixture():
    g = load_golden("char_cfg_b")
    chars, ps = inputs(g, None, None)
    grads = R.gradients(chars, *ps, torch.from_numpy(g["grad_out"]))
    for k, gr in zip(KEYS, grads):
        ref = torch.from_numpy(g["grad::" + R.PRE + k]).double()
        assert float((gr - ref).abs().max()) <= 1e-4 * max(1.0, float(ref.abs().max()))


def test_constructor_signature_and_keys():
    cls = ptgnn_b200.CharUnitEmbedder
    assert list(inspect.signature(cls.__init__).parameters) == ["self", "num_chars", "embedding_size", "config", "dropout_rate"]
    assert inspect.signature(cls.__init__).parameters["dropout_rate"].default == 0.0
    assert list(inspect.signature(cls.forward).parameters) == ["self", "chars"]
    m = cls(30, 63, ptgnn_b200.embeddings.CnnConfig(64, 3, 64, 3, 3))
    assert list(m.state_dict()) == ["_CharUnitEmbedder__" + k for k in KEYS]


def test_scratch_is_not_pickled_or_deep_copied():
    import copy
    import pickle

    m = ptgnn_b200.CharUnitEmbedder(30, 63, ptgnn_b200.embeddings.CnnConfig(64, 3, 64, 3, 3))
    m._status, m._transformed = torch.zeros(2, dtype=torch.int32), ("key", torch.zeros(8, dtype=torch.uint8))
    for restored in (pickle.loads(pickle.dumps(m)), copy.deepcopy(m)):
        assert restored._status is None and restored._transformed is None
        assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), restored.state_dict().values()))


def test_cpu_tensors_raise():
    from ptgnn_b200._native import NativeLibraryError

    m = ptgnn_b200.CharUnitEmbedder(30, 63, ptgnn_b200.embeddings.CnnConfig(64, 3, 64, 3, 3))
    with pytest.raises(NativeLibraryError):
        m(torch.zeros(3, 15, dtype=torch.int64))


@needs_reference
def test_seeded_parameters_and_state_dicts_match_the_reference():
    import_reference()
    ref = __import__(EMBEDDER_MODULE, fromlist=["x"])
    for cfg, C, D in ((ref.CnnConfig(256, 3, 128, 3, 3), 101, 127), (ref.CnnConfig(64, 1, 256, 5, 2), 40, 63)):
        torch.manual_seed(5)
        r = ref.CharUnitEmbedder(C, D, cfg, 0.2)
        torch.manual_seed(5)
        n = ptgnn_b200.CharUnitEmbedder(C, D, cfg, 0.2)
        sig = lambda cls: [(q.name, q.default) for q in inspect.signature(cls.__init__).parameters.values()]
        assert sig(type(r)) == sig(type(n))
        assert list(r.state_dict()) == list(n.state_dict())
        assert all(torch.equal(a, b) for a, b in zip(r.state_dict().values(), n.state_dict().values()))
        n.load_state_dict(r.state_dict(), strict=True)
        r.load_state_dict(n.state_dict(), strict=True)


@needs_reference
def test_overlay_binds_the_char_embedder_only_on_request():
    import_reference()
    ref = __import__(EMBEDDER_MODULE, fromlist=["x"])
    ref_char, ref_sub = ref.CharUnitEmbedder, ref.SubtokenUnitEmbedder

    def build():
        model = ref.StrElementRepresentationModel(token_splitting="char", embedding_size=16)
        model._StrElementRepresentationModel__vocabulary = types.SimpleNamespace(num_chars_in_vocabulary=lambda: 30)
        return model.build_neural_module()

    try:
        report = overlay.install()
        assert report["char_embedder"] is False and ref.CharUnitEmbedder is ref_char
        overlay.uninstall()
        report = overlay.install(native_embedders=True)
        assert report["char_embedder"] is False and ref.CharUnitEmbedder is ref_char and type(build()) is ref_char
        overlay.uninstall()
        report = overlay.install(native_char_embedder=True)
        assert report["char_embedder"] is True and report["embedders"] is False
        assert ref.CharUnitEmbedder is ptgnn_b200.CharUnitEmbedder and ref.SubtokenUnitEmbedder is ref_sub
        assert type(build()) is ptgnn_b200.CharUnitEmbedder
    finally:
        overlay.uninstall()
    assert ref.CharUnitEmbedder is ref_char and ref.SubtokenUnitEmbedder is ref_sub
