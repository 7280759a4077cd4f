"""CPU checks of the node-embedder restatement (tests/embedding_reference.py) against the reference's fixtures, of the emulated kernel
order against its bound, and of the native classes' interface and overlay binding (DESIGN.md §3.12)."""
import glob
import inspect
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import embedding_reference as R  # noqa: E402
from helpers import GOLDEN_DIR, load_golden  # noqa: E402
from oracle.refimport import import_reference, reference_available  # noqa: E402

import ptgnn_b200  # noqa: E402
from ptgnn_b200 import overlay  # noqa: E402

NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "embed_*.npz")) if not p.endswith("_bf16ac.npz"))
needs_reference = pytest.mark.skipif(not reference_available(), reason="the reference tree is not present")
EMBEDDER_MODULE = "ptgnn.neuralmodels.embeddings.strelementrepresentationmodel"


def fixture(name):
    g = load_golden(name)
    kind = str(g["kind"])
    token = kind == "token"
    pre = "sd::_TokenUnitEmbedder__" if token else "sd::_SubtokenUnitEmbedder__"
    table = torch.from_numpy(g[pre + "embeddings.weight"])
    weight = torch.from_numpy(g[pre + "out_layer.weight"]) if bool(g["dense"]) else None
    ids = torch.from_numpy(g["token_idxs"])
    lengths = None if token else torch.from_numpy(g["lengths"])
    return g, ("sum" if token else kind), table, weight, ids, lengths, pre.replace("sd::", "grad::")


def test_fixture_set():
    assert len(NAMES) == 11 and os.path.exists(os.path.join(GOLDEN_DIR, "embed_sub_mean_dense_d64_bf16ac.npz"))
    kinds = {(str(load_golden(n)["kind"]), bool(load_golden(n)["dense"])) for n in NAMES}
    assert kinds >= {("token", False)} | {(k, d) for k in ("sum", "mean", "max") for d in (True, False)}
    assert {int(load_golden(n)["dim"]) for n in NAMES} == {63, 64, 128}


@pytest.mark.parametrize("name", NAMES)
def test_fixture_structure(name):
    g, kind, table, weight, ids, lengths, _ = fixture(name)
    V = table.shape[0]
    counts = torch.bincount(R.occurrences(ids, lengths, V)[2], minlength=V)
    assert int(counts.max()) > 2 * R.CHUNK and int((counts == 0).sum()) > 0
    if lengths is not None:
        S = ids.shape[1]
        assert int(lengths[0]) == 1 and int((lengths == S).sum()) > 1 and int(lengths.min()) >= 1
        pad = torch.arange(S)[None, :] >= lengths[:, None]
        assert int(pad.sum()) > 0 and bool(((ids[pad] > 0) & (ids[pad] < V)).all())
        assert int(g["dim"]) % 4 == 0 or weight is None


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_reference(name):
    g, kind, table, weight, ids, lengths, gp = fixture(name)
    table.requires_grad_(True)
    if weight is not None:
        weight.requires_grad_(True)
    out = R.module_forward(table, ids, lengths, kind, weight)
    assert torch.equal(out, torch.from_numpy(g["out"]))
    (out * torch.from_numpy(g["grad_out"])).sum().backward()
    assert torch.equal(table.grad, torch.from_numpy(g[gp + "embeddings.weight"]))
    if weight is not None:
        assert torch.equal(weight.grad, torch.from_numpy(g[gp + "out_layer.weight"]))


@pytest.mark.parametrize("name", NAMES)
def test_emulated_order_inside_bound_and_mutants_outside(name):
    g, kind, table, weight, ids, lengths, _ = fixture(name)
    exact = R.module_forward(table.double(), ids, lengths, kind)
    b = R.bound(table, ids, lengths, kind)
    emu, arg = R.emulate_forward(table, ids, lengths, kind)
    assert bool(((emu.double() - exact).abs() <= b).all())
    if lengths is not None:
        mutant, _ = R.emulate_forward(table, ids, lengths, kind, ignore_lengths=True)
        assert not bool(((mutant.double() - exact).abs() <= b).all())
        if kind == "mean":
            mutant, _ = R.emulate_forward(table, ids, lengths, kind, mean_by_slots=True)
            assert not bool(((mutant.double() - exact).abs() <= b).all())
    # bf16 output: one more rounding
    emu16, _ = R.emulate_forward(table, ids, lengths, kind, out_dtype=torch.bfloat16)
    assert bool(((emu16.double() - exact).abs() <= R.bound(table, ids, lengths, kind, out_dtype=torch.bfloat16)).all())
    # backward
    d = torch.from_numpy(g["grad_out"])
    V = table.shape[0]
    t64 = table.double().requires_grad_(True)
    (R.module_forward(t64, ids, lengths, kind) * d.double()).sum().backward()
    got = R.emulate_backward(d, ids, lengths, kind, V, arg)
    assert bool(((got.double() - t64.grad).abs() <= R.backward_bound(d, ids, lengths, kind, V, arg)).all())
    absent = torch.bincount(R.occurrences(ids, lengths, V)[2], minlength=V) == 0
    assert bool((got[absent] == 0).all())


@pytest.mark.parametrize("name", [n for n in NAMES if "dense" in n])
def test_dense_paths_inside_bound(name):
    g, kind, table, weight, ids, lengths, _ = fixture(name)
    exact = R.module_forward(table.double(), ids, lengths, kind, weight.double())
    pooled, _ = R.emulate_forward(table, ids, lengths, kind)
    pool_first = (pooled.double() @ weight.double().T).float()
    assert bool(((pool_first.double() - exact).abs() <= R.bound(table, ids, lengths, kind, weight)).all())
    if kind != "max":       # the identity pool(table[ids]) W^T = pool((table W^T)[ids]) holds for the linear poolings only
        tt = (table.double() @ weight.double().T).float()
        table_first, _ = R.emulate_forward(tt, ids, lengths, kind)
        assert bool(((table_first.double() - exact).abs() <= R.bound(table, ids, lengths, kind, weight, table_first=True)).all())


def test_constructor_signatures_and_keys():
    tok, sub = ptgnn_b200.TokenUnitEmbedder, ptgnn_b200.SubtokenUnitEmbedder
    assert list(inspect.signature(tok.__init__).parameters) == ["self", "vocabulary_size", "embedding_size", "dropout_rate"]
    assert list(inspect.signature(sub.__init__).parameters) == ["self", "vocabulary_size", "embedding_size", "dropout_rate",
                                                                "subtoken_combination_kind", "use_dense_output"]
    assert inspect.signature(sub.__init__).parameters["use_dense_output"].default is True
    assert list(inspect.signature(sub.forward).parameters) == ["self", "token_idxs", "lengths"]
    assert list(tok(7, 8, 0.1).state_dict()) == ["_TokenUnitEmbedder__embeddings.weight"]
    assert list(sub(7, 8, 0.1, "mean").state_dict()) == ["_SubtokenUnitEmbedder__embeddings.weight", "_SubtokenUnitEmbedder__out_layer.weight"]
    assert list(sub(7, 8, 0.1, "max", use_dense_output=False).state_dict()) == ["_SubtokenUnitEmbedder__embeddings.weight"]
    m = sub(7, 8, 0.1, "sum")
    assert m.embedding_layer.weight.shape == (7, 8) and isinstance(m.embedding_layer, torch.nn.Embedding)
    with pytest.raises(AssertionError):
        sub(7, 8, 0.1, "median")


@pytest.mark.parametrize("make", [lambda: ptgnn_b200.TokenUnitEmbedder(7, 8, 0.1), lambda: ptgnn_b200.SubtokenUnitEmbedder(7, 8, 0.1, "mean")])
def test_scratch_is_not_pickled_or_deep_copied(make):
    """The reference saves a model by pickling the whole module: the status word and the kept table must not travel with it."""
    import copy
    import io
    import pickle

    m = make()
    m._status, m._transformed = torch.zeros(1, dtype=torch.int32), ("key", torch.zeros(7, 8))      # as after a forward
    buf = io.BytesIO()
    torch.save(m, buf)
    buf.seek(0)
    for restored in (pickle.loads(pickle.dumps(m)), copy.deepcopy(m), torch.load(buf, weights_only=False)):
        assert type(restored) is type(m) and restored._status is None and restored._transformed is None
        assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), restored.state_dict().values()))
    assert m._status is not None and m._transformed is not None


def test_cpu_tensors_raise():
    from ptgnn_b200._native import NativeLibraryError

    with pytest.raises(NativeLibraryError):
        ptgnn_b200.TokenUnitEmbedder(7, 8, 0.0)(torch.zeros(3, dtype=torch.int64))
    with pytest.raises(NativeLibraryError):
        ptgnn_b200.SubtokenUnitEmbedder(7, 8, 0.0, "sum")(torch.zeros(3, 2, dtype=torch.int64), torch.ones(3, dtype=torch.int64))


@needs_reference
def test_state_dicts_load_strictly_both_ways():
    import_reference()
    ref = __import__(EMBEDDER_MODULE, fromlist=["x"])
    pairs = [(ref.TokenUnitEmbedder(9, 8, 0.1), ptgnn_b200.TokenUnitEmbedder(9, 8, 0.1))]
    for dense in (True, False):
        pairs.append((ref.SubtokenUnitEmbedder(9, 8, 0.1, "mean", use_dense_output=dense),
                      ptgnn_b200.SubtokenUnitEmbedder(9, 8, 0.1, "mean", use_dense_output=dense)))
    for r, n in pairs:
        assert list(r.state_dict()) == list(n.state_dict())
        assert inspect.signature(type(r).__init__) == inspect.signature(type(n).__init__)
        n.load_state_dict(r.state_dict(), strict=True)
        assert all(torch.equal(a, b) for a, b in zip(r.state_dict().values(), n.state_dict().values()))
        r.load_state_dict(n.state_dict(), strict=True)


@needs_reference
def test_overlay_binds_the_embedders_only_on_request():
    import_reference()
    ref = __import__(EMBEDDER_MODULE, fromlist=["x"])
    ref_tok, ref_sub, ref_char = ref.TokenUnitEmbedder, ref.SubtokenUnitEmbedder, ref.CharUnitEmbedder
    try:
        report = overlay.install()
        assert report["embedders"] is False and ref.SubtokenUnitEmbedder is ref_sub and ref.TokenUnitEmbedder is ref_tok
        overlay.uninstall()
        report = overlay.install(native_embedders=True)
        assert report["embedders"] is True
        assert ref.SubtokenUnitEmbedder is ptgnn_b200.SubtokenUnitEmbedder and ref.TokenUnitEmbedder is ptgnn_b200.TokenUnitEmbedder
        assert ref.CharUnitEmbedder is ref_char and sys.modules[EMBEDDER_MODULE] is ref

        def build(splitting, **kw):
            model = ref.StrElementRepresentationModel(token_splitting=splitting, embedding_size=16, **kw)
            if splitting == "char":      # a stand-in character vocabulary: build_neural_module only asks it for its size
                model._StrElementRepresentationModel__vocabulary = types.SimpleNamespace(num_chars_in_vocabulary=lambda: 30)
                return model.build_neural_module()
            model.initialize_metadata()
            for w in ["fooBar", "bazQux", "foo"] * 6:
                model.update_metadata_from(w)
            model.finalize_metadata()
            return model.build_neural_module()

        sub = build("subtoken", subtoken_combination="mean")
        assert type(sub) is ptgnn_b200.SubtokenUnitEmbedder
        reference_module = ref_sub(sub.embedding_layer.num_embeddings, 16, 0.2, "mean")
        sub.load_state_dict(reference_module.state_dict(), strict=True)
        assert type(build("token")) is ptgnn_b200.TokenUnitEmbedder
        assert type(build("char")) is ref_char
    finally:
        overlay.uninstall()
    assert ref.SubtokenUnitEmbedder is ref_sub and ref.TokenUnitEmbedder is ref_tok and ref.CharUnitEmbedder is ref_char
