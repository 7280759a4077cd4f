"""graph2seq beam search on the CPU: the float64 restatement (beam_decode_reference.py) with beam width 1 against the reference's own
greedy_decode fixtures, the restatement's ordering with wider beams, the host-side backtrack of ``NativeBeamDecode.result`` on a
constructed state, the refusals, which come before any launch, and the overlay's opt-in ``beam_decode`` methods."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import beam_decode_reference as BR
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


def restated(f, K):
    return BR.beam_decode(f["sd"], f["vocab_obj"], int(f["max_seq_len"]), f["value_list"], f["memories"], f["origin"],
                          f["initial_states"], K)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_with_width_one_reproduces_reference_greedy_decode(name):
    f = load(name)
    out = restated(f, 1)
    assert [hs[0][0] for hs in out] == f["ref_tokens"]
    ref = f["out_logprobs"].astype(np.float64)
    got = np.array([hs[0][1] for hs in out])
    assert np.all(np.abs(got - ref) <= 1e-5 * np.maximum(1.0, np.abs(ref))), (name, got, ref)


@pytest.mark.parametrize("K", [2, 3])
def test_restatement_results_are_sorted_distinct_and_no_worse_than_greedy(K):
    f = load("greedy_end")
    out = restated(f, K)
    greedy = restated(f, 1)
    for hs, g1 in zip(out, greedy):
        totals = [t for _, t in hs]
        assert totals == sorted(totals, reverse=True) and 1 <= len(hs) <= K
        assert len({tuple(t) for t, _ in hs}) == len(hs)
        assert totals[0] >= g1[0][1] - 1e-12


def test_result_backtracks_the_state_on_the_host():
    """A constructed state of 2 graphs, 3 slots and 3 steps: backpointers and keys walk back from each final slot; END and a done
    slot's passing through append nothing; empty slots are left out; keys >= V name out-of-vocabulary copies."""
    from ptgnn_b200.decoding import CopyGroups, NativeBeamDecode

    vocab = GR.TokenVocab([GR.UNK, GR.START, GR.END, "a", "b", "c"])
    V, G, K, T = 6, 2, 3, 3
    dec = object.__new__(NativeBeamDecode)
    dec.G, dec.K, dec.V, dec.max_len, dec.vocab, dec.end_id = G, K, V, T, vocab, 2
    dec.groups = CopyGroups(["a", "zz"], np.array([0, 0]), G, vocab)      # key V + 0 is "zz"
    bp = np.full((T, G, K), -1, dtype=np.int32)
    kt = np.full((T, G, K), -1, dtype=np.int32)
    bp[0, 0, :2], kt[0, 0, :2] = [0, 0], [3, V]          # step 0: graph 0 takes a and zz
    bp[1, 0], kt[1, 0] = [1, 0, 0], [2, 4, 5]            # step 1: zz END (done), a b, a c
    bp[2, 0], kt[2, 0] = [0, 1, 2], [-1, 3, 2]           # step 2: the done slot passes through, a b a, a c END
    bp[0, 1, 0], kt[0, 1, 0] = 0, 4                      # graph 1: one hypothesis, b b b
    bp[1, 1, 0], kt[1, 1, 0] = 0, 4
    bp[2, 1, 0], kt[2, 1, 0] = 0, 4
    total = np.array([[-1.0, -2.0, -3.0], [-0.5, -np.inf, -np.inf]], dtype=np.float32)
    length = np.array([[1, 3, 2], [3, 0, 0]], dtype=np.int32)
    done = np.array([[1, 0, 1], [0, 0, 0]], dtype=np.int32)
    empty = np.array([[0, 0, 0], [0, 1, 1]], dtype=np.int32)
    buf = np.concatenate([bp.ravel(), kt.ravel(), total.view(np.int32).ravel(), length.ravel(), done.ravel(), empty.ravel()])

    class State:
        buffer = torch.from_numpy(buf)

    out = dec.result(State())
    assert out == [[(["zz"], np.float32(-1.0)), (["a", "b", "a"], np.float32(-2.0)), (["a", "c"], np.float32(-3.0))],
                   [(["b", "b", "b"], np.float32(-0.5))]]
    assert all(isinstance(lp, np.float32) for hs in out for _, lp in hs)


def test_unsupported_beam_width_and_hidden_size_are_refused_before_any_launch():
    import ptgnn_b200 as P
    from ptgnn_b200 import _native as N
    from ptgnn_b200 import decoding

    vocab = GR.TokenVocab([GR.UNK, GR.START, GR.END, "a"])
    launches = N.launch_count()
    for H, width, err in ((32, 0, ValueError), (32, -1, ValueError), (32, 9, NotImplementedError), (48, 2, NotImplementedError)):
        module = P.GruCopyingDecoder(len(vocab), 8, H, 16, unk_id=0, dropout_rate=0.0)
        with pytest.raises(err, match="beam_width" if H == 32 else "hidden_size"):
            decoding.beam_decode(GR.DecoderModelStub(vocab, 4), input_concrete_values=["a"], input_memories=torch.zeros(1, 16),
                                 input_memories_origin_idx=torch.zeros(1, dtype=torch.int64), initial_states=torch.zeros(1, H),
                                 neural_model=module, beam_width=width)
    assert N.launch_count() == launches


@pytest.mark.skipif(not reference_available(), reason="the reference tree is not available")
def test_overlay_binds_beam_decode_only_when_asked():
    code = f"""
import sys
sys.path.insert(0, {ROOT!r})
from oracle.refimport import import_reference
import_reference()
import types
import ptgnn.neuralmodels.sequence.grucopydecoder as D
import ptgnn.implementations.graph2seq.graph2seq as G2
import ptgnn_b200.overlay as ov
from ptgnn_b200 import decoding
greedy = D.GruCopyingDecoderModel.greedy_decode
r = ov.install(force_torch_scatter=True)
assert r["beam_decode"] is False and not hasattr(D.GruCopyingDecoderModel, "beam_decode") and not hasattr(G2.Graph2Seq, "beam_decode")
ov.uninstall()
r = ov.install(force_torch_scatter=True, native_beam_decode=True)
assert r["beam_decode"] is True and r["greedy_decode"] is False and D.GruCopyingDecoderModel.greedy_decode is greedy
calls = []
decoding.beam_decode = lambda model, **kw: calls.append((model, sorted(kw))) or [[(["x"], 0.0)]] * len(kw["initial_states"])
model = D.GruCopyingDecoderModel(hidden_size=32)
assert model.beam_decode(input_concrete_values=[], input_memories=None, input_memories_origin_idx=None, initial_states=[1, 2],
                         neural_model=None, beam_width=3) == [[(["x"], 0.0)]] * 2
assert calls == [(model, ["beam_width", "initial_states", "input_concrete_values", "input_memories", "input_memories_origin_idx",
                          "neural_model"])]
# Graph2Seq.beam_decode: the minibatch walk, on stand-ins for the model's parts
import torch
g2s = object.__new__(G2.Graph2Seq)
g2s._Graph2Seq__decoder_model = model
samples = [dict(node_labels=["A", "B", "C"], backbone_sequence=[2, 0]), dict(node_labels=["D"], backbone_sequence=[0])]
g2s.tensorize_dataset = lambda it, return_input_data: list(it)
g2s.minibatch_iterator = lambda data, device, max_minibatch_size: [({{"encoder_mb_data": {{}}}}, data)]
out = types.SimpleNamespace(output_node_representations=torch.arange(8.0).view(4, 2), node_idx_references={{"backbone_nodes": torch.tensor([2, 0, 3])}},
                            node_graph_idx_reference={{"backbone_nodes": torch.tensor([0, 0, 1])}})
net = types.SimpleNamespace(_gnn=lambda **kw: out, _get_initial_decoder_states=lambda o: [10, 20], _decoder="dec")
seen = []
decoding.beam_decode = lambda m, **kw: seen.append(kw) or [[(["y"], 1.0)], [(["z"], 2.0)]]
assert G2.Graph2Seq.beam_decode(g2s, samples, net, "cpu", 4) == [[(["y"], 1.0)], [(["z"], 2.0)]]
kw = seen[0]
assert kw["input_concrete_values"] == ["c", "a", "d"] and kw["beam_width"] == 4 and kw["neural_model"] == "dec"
assert kw["input_memories"].tolist() == [[4.0, 5.0], [0.0, 1.0], [6.0, 7.0]] and kw["input_memories_origin_idx"].tolist() == [0, 0, 1]
ov.uninstall()
assert not hasattr(D.GruCopyingDecoderModel, "beam_decode") and not hasattr(G2.Graph2Seq, "beam_decode")
print("ok")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr
