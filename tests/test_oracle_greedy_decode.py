"""graph2seq greedy decoding on the CPU: the float64 restatement (greedy_decode_reference.py) against the reference's own
``greedy_decode`` (tests/golden/greedy_*.npz, written by tests/golden/generate_greedy_decode_golden.py), the copy-key and group
builder of ``ptgnn_b200.decoding`` on the same data, the refusals that need no GPU, and the overlay's opt-in binding of the method."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import greedy_decode_reference as GR
from oracle.refimport import reference_available

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["greedy_small", "greedy_rank", "greedy_end"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    f = {k: z[k] for k in z.files}
    f["sd"] = {k[4:]: torch.from_numpy(v) for k, v in f.items() if k.startswith("sd::")}
    f["vocab_obj"] = GR.TokenVocab([str(t) for t in f["vocab"]])
    f["value_list"] = [str(v) for v in f["values"]]
    ends = np.cumsum(f["out_lengths"])
    f["ref_tokens"] = [[str(t) for t in f["out_tokens"][e - n:e]] for e, n in zip(ends, f["out_lengths"])]
    return f


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_reference_greedy_decode(name):
    f = load(name)
    tokens, logprobs, _ = GR.greedy_decode(f["sd"], f["vocab_obj"], int(f["max_seq_len"]), f["value_list"], f["memories"], f["origin"],
                                           f["initial_states"])
    assert tokens == f["ref_tokens"], name
    ref = f["out_logprobs"].astype(np.float64)
    assert np.all(np.abs(logprobs - ref) <= 1e-5 * np.maximum(1.0, np.abs(ref))), (name, logprobs, ref)
    assert str(f["logprob_dtype"]) == "float32", "the reference sums log-probabilities in float32"


@pytest.mark.parametrize("name", NAMES)
def test_copy_groups_follow_the_reference_dictionary_order(name):
    from ptgnn_b200.decoding import CopyGroups

    f = load(name)
    vocab, values, origin = f["vocab_obj"], f["value_list"], f["origin"]
    G, V = f["initial_states"].shape[0], len(vocab)
    groups = CopyGroups(values, origin, G, vocab)
    keys = GR.row_keys(values, vocab)
    assert groups.keys.tolist() == keys
    for i, v in enumerate(values):
        assert groups.name(keys[i], vocab) == v
        assert (keys[i] < V) == (not vocab.is_unk(v))
    assert groups.oov == list(dict.fromkeys(v for v in values if vocab.is_unk(v)))
    for g in range(G):
        rows = np.flatnonzero(origin == g).tolist()
        expect = {}
        for i in rows:                       # the reference's dictionary: first occurrence fixes the order, rows in row order
            expect.setdefault(keys[i], []).append(i)
        j0, j1 = groups.group_ptr[g], groups.group_ptr[g + 1]
        got = {int(groups.group_key[j]): groups.member_rows[groups.member_ptr[j]:groups.member_ptr[j + 1]].tolist() for j in range(j0, j1)}
        assert list(got.items()) == list(expect.items()), (name, g)
    assert groups.member_ptr[-1] == len(values) and sorted(groups.member_rows.tolist()) == list(range(len(values)))


def test_fixtures_have_the_intended_structure():
    f = load("greedy_small")
    vocab, values = f["vocab_obj"], f["value_list"]
    assert len(vocab) < 100
    assert any(vocab.is_unk(v) for v in values) and any(not vocab.is_unk(v) for v in values)
    assert any(len(set(np.array(values)[f["origin"] == g])) < int((f["origin"] == g).sum()) for g in range(len(f["out_lengths"])))
    f = load("greedy_rank")
    vocab, sd = f["vocab_obj"], f["sd"]
    V = len(vocab)
    assert 250 <= V <= 350
    rank = np.argsort(np.argsort(-sd["_GruCopyingDecoder__vocab_bias"].numpy(), kind="stable"), kind="stable")
    copied = {int(rank[vocab.get_id_or_unk(v)]) for v in f["value_list"] if not vocab.is_unk(v)}
    assert {98, 99, 100, 101} <= copied, copied
    f = load("greedy_end")
    G = f["initial_states"].shape[0]
    assert 0 in np.bincount(f["origin"], minlength=G).tolist(), "a graph without memories"
    assert any(1 <= n < int(f["max_seq_len"]) for n in f["out_lengths"]), "an END after the first step"
    assert int(f["max_seq_len"]) in f["out_lengths"].tolist(), "a graph that never ends"


def test_unsupported_hidden_size_is_refused_before_any_launch():
    import ptgnn_b200 as P
    from ptgnn_b200 import decoding

    vocab = GR.TokenVocab([GR.UNK, GR.START, GR.END, "a"])
    module = P.GruCopyingDecoder(len(vocab), 8, 48, 16, unk_id=0, dropout_rate=0.0)
    with pytest.raises(NotImplementedError, match="hidden_size"):
        decoding.greedy_decode(GR.DecoderModelStub(vocab, 4), input_concrete_values=["a"], input_memories=torch.zeros(1, 16),
                               input_memories_origin_idx=torch.zeros(1, dtype=torch.int64), initial_states=torch.zeros(1, 48),
                               neural_model=module)


@pytest.mark.skipif(not reference_available(), reason="the reference tree is not available")
def test_overlay_binds_greedy_decode_only_when_asked():
    code = f"""
import sys
sys.path.insert(0, {ROOT!r})
from oracle.refimport import import_reference
import_reference()
import ptgnn.neuralmodels.sequence.grucopydecoder as D
original = D.GruCopyingDecoderModel.greedy_decode
import ptgnn_b200.overlay as ov
from ptgnn_b200 import decoding
r = ov.install(force_torch_scatter=True)
assert r["greedy_decode"] is False and D.GruCopyingDecoderModel.greedy_decode is original
ov.uninstall()
r = ov.install(force_torch_scatter=True, native_greedy_decode=True)
assert r["greedy_decode"] is True and r["decoder"] is False
assert D.GruCopyingDecoderModel.greedy_decode is not original
assert D.GruCopyingDecoder is not None and D.GruCopyingDecoder.__module__.startswith("ptgnn.")   # the decoder module stays the reference's
calls = []
decoding.greedy_decode = lambda model, **kw: calls.append((model, sorted(kw))) or "native"
model = D.GruCopyingDecoderModel(hidden_size=32)
assert model.greedy_decode(input_concrete_values=[], input_memories=None, input_memories_origin_idx=None, initial_states=None,
                           neural_model=None) == "native"
assert calls == [(model, ["initial_states", "input_concrete_values", "input_memories", "input_memories_origin_idx", "neural_model"])]
ov.uninstall()
assert D.GruCopyingDecoderModel.greedy_decode is original
print("ok")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr
