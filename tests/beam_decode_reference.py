"""float64 restatement of graph2seq's beam search (DESIGN.md §3.19, ``ptgnn_b200.decoding.beam_decode``), written from its contract:

* K slots per graph, each live, done or empty.  At step 0 slot 0 is live with START, total 0 and the graph's initial state; the others
  are empty.
* A live slot's candidates are greedy decoding's dictionary for its step (greedy_decode_reference.select: the top min(100, V) of
  lp = x - Z, lower id first among equal values, then every memory row of the graph merged into the entry of its key with logaddexp);
  within the slot they are ordered by score descending, then by their position in that dictionary.  The slot keeps its K best.  A
  candidate's total is cum + score.  A key >= V is an out-of-vocabulary copy and feeds UNK.
* A done slot has one candidate, itself (key -1 here: nothing appended), with its total unchanged; it feeds END.  An empty slot has none.
* Per graph the K best candidates by (total descending, source slot ascending, rank within the slot ascending) become the new slots in
  that order; a selected END makes its slot done; if fewer than K exist, the rest are empty.
* After max_seq_len steps each graph's result lists its non-empty slots best first, unfinished ones included, unnormalised.

``slot_candidates`` / ``merge`` restate one step from given logits and copy scores (the kernel-level checks); ``compute_logprobs_beams``
runs decoder_reference.compute_logprobs on G·K rows with the memories replicated per beam (the whole-decode checks).
"""
import math
from typing import List, Sequence, Tuple

import numpy as np
import torch

import decoder_reference as DR
import greedy_decode_reference as GR

LIVE, DONE, EMPTY = 0, 1, 2
DONE_KEY = -1


def dictionary(lp: np.ndarray, c: np.ndarray, rows: Sequence[int], keys: Sequence[int]):
    """The reference's dictionary of one hypothesis as a list of (key, score) in dictionary order: lp [V] and c [M] in float64, rows
    the memory rows of its graph in row order."""
    V = lp.shape[0]
    order = np.lexsort((np.arange(V), -lp))[:min(GR.TOP_K, V)]
    entries = {int(v): float(lp[v]) for v in order}
    for i in rows:
        k = int(keys[i])
        entries[k] = GR.logaddexp(entries.get(k, -math.inf), float(c[i]))
    return list(entries.items())


def ranked(entries) -> List[Tuple[int, float]]:
    """Greedy's order within one slot: score descending, then dictionary position."""
    return [e for _, e in sorted(enumerate(entries), key=lambda pe: (-pe[1][1], pe[0]))]


def slot_candidates(status: int, cum: float, lp, c, rows, keys, K: int) -> List[Tuple[int, float, float]]:
    """A slot's candidates as (key, score, total), best first."""
    if status == EMPTY:
        return []
    if status == DONE:
        return [(DONE_KEY, 0.0, cum)]
    return [(k, s, cum + s) for k, s in ranked(dictionary(lp, c, rows, keys))[:K]]


def merge(cands: Sequence[Sequence[Tuple[int, float, float]]], K: int):
    """All of one graph's candidates, ordered by (total descending, slot, rank): a list of (total, slot, rank, key); the first K are the
    selection."""
    flat = [(total, s, r, key) for s, cs in enumerate(cands) for r, (key, _, total) in enumerate(cs)]
    return sorted(flat, key=lambda e: (-e[0], e[1], e[2]))


def normaliser(x: np.ndarray, lse: float) -> float:
    m = max(float(x.max()), lse)
    return m + math.log(float(np.exp(x - m).sum()) + math.exp(lse - m)) if m != -math.inf else -math.inf


def step_from_logits(x, s, lse, origin, keys, status, cum, K):
    """One step in float64 from logits x [G·K, V], copy scores s [M, K], lse [G, K] and per-slot status / cum [G, K]: per graph the
    merged candidate list (``merge``), and Z [G, K] (NaN for a slot that is not live)."""
    x, s, lse = (np.asarray(a, dtype=np.float64) for a in (x, s, lse))
    G = lse.shape[0]
    Z = np.full((G, K), np.nan)
    out = []
    for g in range(G):
        rows = np.flatnonzero(origin == g)
        cands = []
        for k in range(K):
            if status[g][k] == LIVE:
                Z[g, k] = normaliser(x[g * K + k], lse[g, k])
            cands.append(slot_candidates(status[g][k], cum[g][k], x[g * K + k] - Z[g, k], s[:, k] - Z[g, k], rows, keys, K))
        out.append(merge(cands, K))
    return out, Z


def replicate(memories: torch.Tensor, origin: torch.Tensor, K: int):
    """The memories of graph g repeated for each of its K beams: row block k holds the rows of beam g·K + k."""
    return memories.repeat(K, 1), torch.cat([origin * K + k for k in range(K)])


def compute_logprobs_beams(sd, h, memories_rep, origin_rep, ids, M: int, K: int):
    """decoder_reference.compute_logprobs on G·K rows (``replicate``'s memories): (lp [G·K, V], c [K, M], new h [G·K, H]), c[k, i] the
    copy log-probability of memory row i for beam g(i)·K + k."""
    copy_lp, target_lp, h_new = DR.compute_logprobs(sd, h, memories_rep, origin_rep, torch.tensor(ids)[:, None])
    return target_lp[:, 0].numpy(), copy_lp[:, 0].numpy().reshape(K, M), h_new[0]


def beam_decode(sd, vocab, max_seq_len: int, values: Sequence[str], memories, origin, initial_states, K: int):
    """The whole beam search in float64 from a state_dict ``sd`` (reference names): per graph a list of (token strings, total), best
    first."""
    sd = {k: torch.as_tensor(v).double() for k, v in sd.items()}
    memories, h = torch.as_tensor(memories).double(), torch.as_tensor(initial_states).double()
    origin = torch.as_tensor(origin)
    G, V, M = h.shape[0], len(vocab), origin.numel()
    keys = GR.row_keys(values, vocab)
    oov = {k: v for v, k in zip(values, keys) if k >= V}
    end_id, unk_id = vocab.get_id_or_unk(GR.END), vocab.get_id_or_unk(GR.UNK)
    mem_rep, org_rep = replicate(memories, origin, K)
    h = h.repeat_interleave(K, 0)
    status = [[LIVE if k == 0 else EMPTY for k in range(K)] for _ in range(G)]
    cum = [[0.0] * K for _ in range(G)]
    seqs = [[[] for _ in range(K)] for _ in range(G)]
    ids = [vocab.get_id_or_unk(GR.START)] * (G * K)
    with torch.no_grad():
        for _ in range(max_seq_len):
            lp, c, h_new = compute_logprobs_beams(sd, h, mem_rep, org_rep, ids, M, K)
            gather, ids = [], []
            for g in range(G):
                rows = np.flatnonzero(origin.numpy() == g)
                m = merge([slot_candidates(status[g][k], cum[g][k], lp[g * K + k], c[k], rows, keys, K) for k in range(K)], K)[:K]
                new_status, new_cum, new_seqs = [EMPTY] * K, [0.0] * K, [[] for _ in range(K)]
                for j in range(K):
                    if j >= len(m):
                        gather.append(g * K + j)
                        ids.append(end_id)
                        continue
                    total, src, _, key = m[j]
                    gather.append(g * K + src)
                    new_cum[j] = total
                    done = key == DONE_KEY or key == end_id
                    new_status[j] = DONE if done else LIVE
                    new_seqs[j] = seqs[g][src] + ([] if done else [key])
                    ids.append(end_id if done else key if key < V else unk_id)
                status[g], cum[g], seqs[g] = new_status, new_cum, new_seqs
            h = h_new[gather]
    names = lambda s: [vocab.get_name_for_id(k) if k < V else oov[k] for k in s]      # noqa: E731
    return [[(names(seqs[g][k]), cum[g][k]) for k in range(K) if status[g][k] != EMPTY] for g in range(G)]
