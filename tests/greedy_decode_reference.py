"""float64 restatement of graph2seq's greedy decoding (the reference's GruCopyingDecoderModel.greedy_decode, grucopydecoder.py:375-457),
written from the contract of DESIGN.md §3.18 rather than from the reference's code:

* Z = logsumexp(logits ∪ {lse_copy}), lp = logits - Z, c = copy scores - Z;
* T = the K = min(100, V) largest lp, the lower id first among equal values;
* an ordered dictionary, as the reference's: the members of T in that order, then every memory row of the graph in row order merged
  into the entry of its key with logaddexp (a new key is appended); the winner is the first entry with the highest score;
* the state update: a done graph feeds END; otherwise the score is added, END marks the graph done and anything else is appended.

Keys are integers: a value in the output vocabulary has its id, any other string ``V + j`` for the minibatch's j-th such string.  The
vocabulary and decoder-model stand-ins below give the native decoding what it reads from the reference's classes, so GPU tests run
without the reference tree.
"""
import math
from typing import Dict, List, Sequence

import numpy as np
import torch

import decoder_reference as DR

TOP_K = 100
START, END, UNK = "%START%", "%END%", "%UNK%"


class TokenVocab:
    """The part of dpu_utils' Vocabulary that decoding reads, over a fixed token list (UNK included)."""

    def __init__(self, tokens: Sequence[str]):
        self.tokens = list(tokens)
        self.ids = {t: i for i, t in enumerate(self.tokens)}

    def __len__(self):
        return len(self.tokens)

    @staticmethod
    def get_unk():
        return UNK

    def is_unk(self, token):
        return token not in self.ids

    def get_id_or_unk(self, token):
        return self.ids.get(token, self.ids[UNK])

    def get_name_for_id(self, token_id):
        return self.tokens[token_id]


class DecoderModelStub:
    """What greedy decoding reads from the reference's GruCopyingDecoderModel: START, END, max_seq_len and the output vocabulary."""

    START, END = START, END

    def __init__(self, vocab: TokenVocab, max_seq_len: int):
        self.max_seq_len = max_seq_len
        self._GruCopyingDecoderModel__output_vocabulary = vocab


def row_keys(values: Sequence[str], vocab) -> List[int]:
    V, oov, keys = len(vocab), {}, []
    for v in values:
        keys.append(vocab.get_id_or_unk(v) if not vocab.is_unk(v) else V + oov.setdefault(v, len(oov)))
    return keys


def logaddexp(a: float, b: float) -> float:
    return float(np.logaddexp(np.float64(a), np.float64(b)))


def select(lp: np.ndarray, c: np.ndarray, origin: np.ndarray, keys: Sequence[int]):
    """One step's selection from lp [G, V] and c [M] (float64): per graph (winning key, score, margin, entries), margin = the gap
    between the best and the second-best dictionary entry (inf with a single entry), entries = the dictionary {key: score}."""
    G, V = lp.shape
    K = min(TOP_K, V)
    out = []
    for g in range(G):
        order = np.lexsort((np.arange(V), -lp[g]))[:K]        # larger lp first, then lower id
        entries: Dict[int, float] = {int(v): float(lp[g, v]) for v in order}
        for i in np.flatnonzero(origin == g):
            k = int(keys[i])
            entries[k] = logaddexp(entries.get(k, -math.inf), float(c[i]))
        best_key, best = None, -math.inf
        for k, s in entries.items():
            if best_key is None or s > best:
                best_key, best = k, s
        second = max((s for k, s in entries.items() if k != best_key), default=-math.inf)
        out.append((best_key, best, best - second, entries))
    return out


def select_from_logits(x: np.ndarray, s: np.ndarray, lse_copy: np.ndarray, origin: np.ndarray, keys: Sequence[int]):
    """(Z [G], per-graph (key, score, margin, entries)) from logits x [G, V], copy scores s [M] and lse_copy [G], in float64."""
    x, s, lse_copy = (np.asarray(a, dtype=np.float64) for a in (x, s, lse_copy))
    m = np.maximum(x.max(axis=1), lse_copy)
    Z = m + np.log(np.exp(x - m[:, None]).sum(axis=1) + np.exp(lse_copy - m))
    return Z, select(x - Z[:, None], s - Z[origin], origin, keys)


def update(state, picks, end_id: int, unk_id: int, V: int):
    """Applies one step's picks to state = (tokens lists, logprobs, done flags); returns the next input ids."""
    tokens, logprobs, done = state
    nxt = []
    for g, (k, score, *_) in enumerate(picks):
        if done[g]:
            nxt.append(end_id)
            continue
        logprobs[g] += score
        if k == end_id:
            done[g] = True
        else:
            tokens[g].append(k)
        nxt.append(k if k < V else unk_id)
    return nxt


def greedy_decode(sd, vocab: TokenVocab, max_seq_len: int, values: Sequence[str], memories, origin, initial_states):
    """The whole decode in float64 from a state_dict ``sd`` (reference names): (token strings per graph, logprobs [G], the margin of
    every graph's pick at every step [max_seq_len, G] (inf once a graph is done))."""
    sd = {k: torch.as_tensor(v).double() for k, v in sd.items()}
    memories, initial_states = torch.as_tensor(memories).double(), torch.as_tensor(initial_states).double()
    origin = torch.as_tensor(origin)
    G, V = initial_states.shape[0], len(vocab)
    keys = row_keys(values, vocab)
    end_id, unk_id = vocab.get_id_or_unk(END), vocab.get_id_or_unk(UNK)
    state = ([[] for _ in range(G)], [0.0] * G, [False] * G)
    ids = [vocab.get_id_or_unk(START)] * G
    h = initial_states
    margins = np.full((max_seq_len, G), np.inf)
    oov = {k: v for v, k in zip(values, keys) if k >= V}
    with torch.no_grad():
        for t in range(max_seq_len):
            copy_lp, target_lp, h_new = DR.compute_logprobs(sd, h, memories, origin, torch.tensor(ids)[:, None])
            h = h_new[0]
            picks = select(target_lp[:, 0].numpy(), copy_lp[:, 0].numpy(), origin.numpy(), keys)
            margins[t] = [np.inf if state[2][g] else p[2] for g, p in enumerate(picks)]
            ids = update(state, picks, end_id, unk_id, V)
    names = [[vocab.get_name_for_id(k) if k < V else oov[k] for k in toks] for toks in state[0]]
    return names, np.array(state[1]), margins
