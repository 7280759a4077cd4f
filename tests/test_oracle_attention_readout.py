"""Attention reducers on the CPU: the float restatement (attention_readout_reference.py) against the reference's own outputs
(tests/golden/attn_*.npz, written by tests/golden/generate_attention_readout_golden.py), the native classes' signatures and state_dict
keys against the reference's, and the overlay's opt-in binding of the reference's attention reducers."""
import inspect
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import attention_readout_reference as AR
import global_exchange_reference as GX
from oracle.refimport import reference_available

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["attn_mh1", "attn_mh1_value", "attn_mh4", "attn_mh4_value", "attn_mh8", "attn_mh8_value", "attn_self_weighted"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: z[k].item() if z[k].dtype.kind in "Ub" and z[k].ndim == 0 else
            (int(z[k]) if z[k].dtype.kind == "i" and z[k].ndim == 0 else torch.from_numpy(z[k])) for k in z.files}


def restated(f, x=None):
    """The restatement's output for fixture ``f`` (on ``x``, by default the fixture's states)."""
    cls = "" if f["cls"] == "self" else "Multihead"
    p = f"sd::_{cls}SelfAttentionVarSizedElementReduce__"
    x = f["x"] if x is None else x
    n2g = f["n2g"]
    G = int(n2g.max()) + 1
    w = f.get(p + "query_layer._WeightedSumVarSizedElementReduce__weights_layer.weight")
    queries = GX.graph_readout(x, n2g, G, f["query"], w)
    if f["cls"] == "self":
        return AR.self_attention_forward(x, n2g, G, queries, f[p + "key_layer.weight"], f[p + "output_layer.weight"])
    return AR.multihead_self_attention_forward(x, n2g, G, queries, f[p + "key_layer.weight"], f["heads"], f[p + "output_layer.weight"],
                                               f.get(p + "value_layer.weight"))


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_reference_attention_readout(name):
    f = load(name)
    assert torch.equal(restated(f), f["out"]), f"{name}: restatement differs from the reference's output"


def test_restatement_reproduces_reference_autocast():
    f = load("attn_mh8_bf16ac")
    with torch.autocast("cpu", dtype=torch.bfloat16):
        out = restated(f)
    assert torch.equal(out.float(), f["out_autocast"])
    assert torch.equal(restated(f), f["out_fp32_rounded_inputs"])


def test_restatement_in_float64_is_close_to_fp32_fixtures():
    for name in NAMES:
        f = load(name)
        f64 = {k: v.double() if isinstance(v, torch.Tensor) and v.is_floating_point() else v for k, v in f.items()}
        ref = restated(f64)
        err = ((ref - f["out"].double()).abs() / ref.abs().clamp(min=1)).max().item()
        assert err <= 1e-5, f"{name}: float64 restatement vs fp32 reference {err:.2e}"


def test_fixture_graph_map_has_the_intended_structure():
    f = load("attn_mh8")
    counts = torch.bincount(f["n2g"])
    assert counts[3] == 0 and counts[0] == 1 and counts[5] == 1, "a gap and two 1-node graphs"
    assert not bool((f["n2g"][1:] >= f["n2g"][:-1]).all()), "unsorted"
    assert bool((f["out"][3] == 0).all()), "the graph without nodes gives 0"


def test_native_classes_are_exported_with_reference_signatures():
    import ptgnn_b200 as P

    m = P.MultiheadSelfAttentionVarSizedElementReduce(256, 256, 128, 8, P.SimpleVarSizedElementReduce("max"))
    assert list(m.state_dict()) == ["_MultiheadSelfAttentionVarSizedElementReduce__key_layer.weight",
                                    "_MultiheadSelfAttentionVarSizedElementReduce__output_layer.weight"]
    assert tuple(m.state_dict()["_MultiheadSelfAttentionVarSizedElementReduce__output_layer.weight"].shape) == (128, 8 * 256)
    params = list(inspect.signature(P.MultiheadSelfAttentionVarSizedElementReduce).parameters)
    assert params == ["input_representation_size", "hidden_size", "output_representation_size", "num_heads",
                      "query_representation_summarizer", "use_value_layer"]


@pytest.mark.skipif(not reference_available(), reason="the reference tree is not available")
def test_native_classes_match_reference_signatures_and_state_dict_keys():
    code = f"""
import inspect, sys
sys.path.insert(0, {ROOT!r})
from oracle.refimport import import_reference
import_reference()
import ptgnn.neuralmodels.reduceops.varsizedsummary as R
import ptgnn_b200 as P
def params(cls):   # names, kinds and defaults (the annotations name each package's own reducer base class)
    return [(p.name, p.kind, p.default) for p in inspect.signature(cls).parameters.values()]
for name in ("SelfAttentionVarSizedElementReduce", "MultiheadSelfAttentionVarSizedElementReduce"):
    assert params(getattr(R, name)) == params(getattr(P, name)), (name, params(getattr(R, name)), params(getattr(P, name)))
def build(mod, name, value):
    q = mod.WeightedSumVarSizedElementReduce(64)
    if name == "SelfAttentionVarSizedElementReduce":
        return getattr(mod, name)(64, 32, 16, q)
    return getattr(mod, name)(64, 32, 16, 4, q, use_value_layer=value)
for name in ("SelfAttentionVarSizedElementReduce", "MultiheadSelfAttentionVarSizedElementReduce"):
    for value in (False, True):
        ref, nat = build(R, name, value), build(P, name, value)
        assert list(ref.state_dict()) == list(nat.state_dict()), (list(ref.state_dict()), list(nat.state_dict()))
        assert all(ref.state_dict()[k].shape == v.shape for k, v in nat.state_dict().items())
print("ok")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.skipif(not reference_available(), reason="the reference tree is not available")
def test_overlay_binds_attention_reducers_only_when_asked():
    code = f"""
import sys
sys.path.insert(0, {ROOT!r})
from oracle.refimport import import_reference
import_reference()
import ptgnn.neuralmodels.reduceops.varsizedsummary as R
RefMH, RefSA = R.MultiheadSelfAttentionVarSizedElementReduce, R.SelfAttentionVarSizedElementReduce
import ptgnn.implementations.graph2seq.graph2seq as g2s          # imported before the overlay: its binding must be re-bound
import ptgnn_b200 as P
import ptgnn_b200.overlay as ov
r = ov.install()
assert r["reducers"] is False
assert g2s.MultiheadSelfAttentionVarSizedElementReduce is RefMH and R.MultiheadSelfAttentionVarSizedElementReduce is RefMH
ov.uninstall()
r = ov.install(native_reducers=True)
assert r["reducers"] is True
import ptgnn.neuralmodels.reduceops as RO
for mod in (R, RO):
    assert mod.MultiheadSelfAttentionVarSizedElementReduce is P.MultiheadSelfAttentionVarSizedElementReduce
    assert mod.SelfAttentionVarSizedElementReduce is P.SelfAttentionVarSizedElementReduce
assert g2s.MultiheadSelfAttentionVarSizedElementReduce is P.MultiheadSelfAttentionVarSizedElementReduce
ov.uninstall()
assert g2s.MultiheadSelfAttentionVarSizedElementReduce is RefMH and R.MultiheadSelfAttentionVarSizedElementReduce is RefMH
assert R.SelfAttentionVarSizedElementReduce is RefSA
print("ok")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr
