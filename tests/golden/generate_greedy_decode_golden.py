"""Generates the graph2seq greedy-decoding fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_greedy_decode_golden.py          # writes tests/golden/greedy_*.npz

The reference's ``GruCopyingDecoderModel`` and ``GruCopyingDecoder`` (``neuralmodels/sequence/grucopydecoder.py``) are imported
read-only through ``oracle/refimport.py``; its vocabulary is the ``dpu_utils`` stand-in under ``oracle/refstubs``.  The model's own
``build_neural_module`` builds the decoder and ``greedy_decode`` runs on CPU in eval mode.  Each fixture stores the state_dict (keys
prefixed ``sd::``), the inputs (``memories``, ``origin``, ``initial_states``), the vocabulary's tokens in id order, the concrete values
of the memory rows, and the returned tokens (``out_tokens`` flat, ``out_lengths`` per graph) and log-probabilities (``out_logprobs``).

* ``greedy_small``: V < 100; copied values in and out of the vocabulary, repeated within a graph.
* ``greedy_rank``:  V = 300 with ``vocab_bias`` fixing the vocabulary ranks, and copied tokens at ranks 98 to 101 (0-based): the top
  100 holds ranks 0 to 99, so some copies merge with their vocabulary entry and the next ones just outside it do not.
* ``greedy_end``:   a graph without memories, and a graph whose END wins at a step after the first.
"""
import os
import sys
from collections import Counter

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from dpu_utils.mlutils import Vocabulary  # noqa: E402  (the stand-in under oracle/refstubs)
from ptgnn.neuralmodels.sequence.grucopydecoder import GruCopyingDecoderModel  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def build(words, H, E, D, max_len):
    """The reference model with the output vocabulary UNK, START, END, words (in this id order) and its decoder module."""
    model = GruCopyingDecoderModel(max_seq_len=max_len, hidden_size=H, embedding_size=E, memories_hidden_dim=D, dropout_rate=0.2)
    counts = Counter({model.START: 10 ** 7, model.END: 10 ** 7 - 1})
    counts.update({w: 10 ** 6 - i for i, w in enumerate(words)})
    vocab = Vocabulary.create_vocabulary(counts, max_size=len(words) + 3, count_threshold=1)
    model._GruCopyingDecoderModel__output_vocabulary = vocab
    module = model.build_neural_module()
    module.eval()
    return model, module, vocab


def decode(model, module, values, memories, origin, h0):
    with torch.no_grad():
        return model.greedy_decode(input_concrete_values=values, input_memories=memories, input_memories_origin_idx=origin,
                                   initial_states=h0, neural_model=module)


def save(name, model, module, vocab, values, memories, origin, h0, result):
    tokens = [t for toks, _ in result for t in toks]
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(
        path, memories=memories.numpy(), origin=origin.numpy(), initial_states=h0.numpy(),
        vocab=np.array([vocab.get_name_for_id(i) for i in range(len(vocab))]), values=np.array(values),
        out_tokens=np.array(tokens, dtype=np.str_).reshape(-1), out_lengths=np.array([len(t) for t, _ in result]),
        out_logprobs=np.array([lp for _, lp in result], dtype=np.float32), max_seq_len=np.array(model.max_seq_len),
        logprob_dtype=np.array(str(np.asarray(result[0][1]).dtype)),
        **{"sd::" + k: v.detach().numpy() for k, v in module.state_dict().items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB; " + "; ".join(f"{' '.join(t)} ({lp:.4f})" for t, lp in result))


def shuffled_origin(counts, gen):
    origin = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    return origin[torch.randperm(origin.numel(), generator=gen)]


def small():
    torch.manual_seed(11)
    gen = torch.Generator().manual_seed(12)
    words = [f"w{i}" for i in range(57)]
    model, module, vocab = build(words, 32, 16, 24, 6)
    counts = [7, 3, 12, 1, 9]
    origin = shuffled_origin(counts, gen)
    pool = ["w3", "w3", "w17", "w40", "foo", "bar", "foo", "baz", "w3", "qux", "w56", "foo"]
    values = [pool[int(i)] for i in torch.randint(0, len(pool), (origin.numel(),), generator=gen)]
    memories = torch.randn(origin.numel(), 24, generator=gen) * 2
    h0 = torch.randn(len(counts), 32, generator=gen)
    result = decode(model, module, values, memories, origin, h0)
    save("greedy_small", model, module, vocab, values, memories, origin, h0, result)


def rank():
    torch.manual_seed(21)
    gen = torch.Generator().manual_seed(22)
    words = [f"t{i}" for i in range(297)]
    model, module, vocab = build(words, 32, 16, 24, 5)
    V = len(vocab)
    with torch.no_grad():
        rank_of = torch.randperm(V, generator=gen)                  # vocabulary id -> rank
        module._GruCopyingDecoder__vocab_bias.copy_(-0.01 * rank_of.float())
        module._GruCopyingDecoder__hidden_to_vocab.mul_(1e-3)     # the projection moves logits by << the 0.01 rank spacing
        module._GruCopyingDecoder__memories_to_copy_attention.weight.mul_(0.05)
    by_rank = torch.argsort(rank_of)
    at = {r: vocab.get_name_for_id(int(by_rank[r])) for r in (98, 99, 100, 101)}
    print("rank 98-101:", at)
    # graph g copies the token at rank 98 + g (two or three rows), plus out-of-vocabulary filler
    counts, values = [], []
    for g, r in enumerate((98, 99, 100, 101)):
        vals = [at[r]] * (2 + g % 2) + ["oov_a", "oov_b"][: g % 3]
        counts.append(len(vals))
        values.append(vals)
    origin = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    flat = [v for vals in values for v in vals]
    perm = torch.randperm(origin.numel(), generator=gen)
    origin, flat = origin[perm], [flat[int(i)] for i in perm]
    memories = torch.randn(origin.numel(), 24, generator=gen)
    h0 = torch.randn(len(counts), 32, generator=gen)
    result = decode(model, module, flat, memories, origin, h0)
    save("greedy_rank", model, module, vocab, flat, memories, origin, h0, result)


def end():
    words = [f"e{i}" for i in range(77)]
    for seed in range(100):
        torch.manual_seed(31 + seed)
        gen = torch.Generator().manual_seed(32 + seed)
        model, module, vocab = build(words, 32, 16, 24, 8)
        with torch.no_grad():
            bias = module._GruCopyingDecoder__vocab_bias
            bias.normal_(0.0, 1.0, generator=gen)
            bias[vocab.get_id_or_unk(model.END)] = bias.max() + 0.05        # END near the top: it wins at some steps only
        counts = [5, 0, 8, 4, 6]                # graph 1 has no memories
        origin = shuffled_origin(counts, gen)
        values = [f"e{int(i)}" if i < 77 else f"x{int(i)}" for i in torch.randint(0, 90, (origin.numel(),), generator=gen)]
        memories = torch.randn(origin.numel(), 24, generator=gen)
        h0 = torch.randn(len(counts), 32, generator=gen) * 2
        result = decode(model, module, values, memories, origin, h0)
        lengths = [len(t) for t, _ in result]
        if any(1 <= n <= 5 for n in lengths) and any(n == 8 for n in lengths):
            print(f"greedy_end: seed {seed}, lengths {lengths}")
            save("greedy_end", model, module, vocab, values, memories, origin, h0, result)
            return
    raise RuntimeError("no seed gives an END mid-sequence")


if __name__ == "__main__":
    small()
    rank()
    end()
