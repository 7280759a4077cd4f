"""Greedy decoding of graph2seq (the reference's ``GruCopyingDecoderModel.greedy_decode``, ``neuralmodels/sequence/grucopydecoder.py:375-457``)
with the decode loop on the device (DESIGN §3.18).

The reference runs ``_compute_logprobs`` for one step ``max_seq_len`` times, recomputing both ``[M, H]`` memory projections each time,
copies the top 100 vocabulary entries and every copy log-probability to the host, and merges them in Python dictionaries keyed by
string.  Here, once per minibatch, the memory rows are given integer *keys* (the vocabulary id of a value in the output vocabulary,
else ``V + j`` for the minibatch's j-th out-of-vocabulary string) and grouped per graph in one host pass; the tables reach the device
in one copy; ``A = memories W_stdᵀ`` and ``C = memories W_copyᵀ`` are computed once.  Each step then runs the module's embedding and
``nn.GRU`` for one step, the two attention kernels of ``decoder.py``, the vocabulary einsum as the reference writes it, and
``ptgnn_b200_decode_select`` -- which merges copies into the vocabulary entries, picks the winner and updates the per-graph state on the
device.  Nothing synchronises with the host until the final copy of the tokens, lengths and log-probabilities.

Tie order: ``torch.topk``'s order among equal values is unspecified; here the lower vocabulary id comes first, both for membership
of the top 100 and for the dictionary order that breaks ties between equal scores.

``beam_decode`` (DESIGN §3.19) is beam search on the same per-minibatch work: K hypotheses per graph run as the attention kernels' K
query rows, and ``ptgnn_b200_beam_select`` builds each live hypothesis's dictionary as greedy decoding does, keeps its K best entries and
merges the K² candidates of a graph into its next K hypotheses on the device.  Its semantics are written out in ``beam_decode``.
"""
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _native as N
from . import composed as C
from .decoder import _padded_steps, native_copy_attention
from .reduceops import graph_plan, native_attention_readout

HIDDEN_SIZES = (32, 64, 128, 256)


class CopyGroups:
    """The memory rows of a minibatch grouped by (graph, key), built on the host in one pass over the rows.

    ``keys[i]`` is row i's key; the groups of graph g are ``group_ptr[g] .. group_ptr[g + 1]`` in first-occurrence order, group j has
    key ``group_key[j]`` and the rows ``member_rows[member_ptr[j] .. member_ptr[j + 1]]`` in row order.  ``oov`` lists the
    out-of-vocabulary strings in first-occurrence order (key ``V + j`` is ``oov[j]``)."""

    def __init__(self, concrete_values: Sequence[str], origin: np.ndarray, num_graphs: int, vocab):
        V = len(vocab)
        self.num_graphs, self.vocab_size = num_graphs, V
        self.oov: List[str] = []
        oov_ids: Dict[str, int] = {}
        keys = np.empty(len(concrete_values), dtype=np.int64)
        per_graph: List[Dict[int, List[int]]] = [{} for _ in range(num_graphs)]
        for i, (value, g) in enumerate(zip(concrete_values, origin.tolist())):
            if not vocab.is_unk(value):
                k = vocab.get_id_or_unk(value)
            else:
                j = oov_ids.get(value)
                if j is None:
                    j = oov_ids[value] = len(self.oov)
                    self.oov.append(value)
                k = V + j
            keys[i] = k
            per_graph[g].setdefault(k, []).append(i)      # dicts keep first-occurrence order
        self.keys = keys
        self.group_ptr = np.zeros(num_graphs + 1, dtype=np.int32)
        group_key, member_ptr, member_rows = [], [0], []
        for g, groups in enumerate(per_graph):
            for k, rows in groups.items():
                group_key.append(k)
                member_rows.extend(rows)
                member_ptr.append(len(member_rows))
            self.group_ptr[g + 1] = len(group_key)
        self.group_key = np.asarray(group_key, dtype=np.int32)
        self.member_ptr = np.asarray(member_ptr, dtype=np.int32)
        self.member_rows = np.asarray(member_rows, dtype=np.int32)

    def name(self, key: int, vocab) -> str:
        return vocab.get_name_for_id(key) if key < self.vocab_size else self.oov[key - self.vocab_size]

    def to_device(self, device) -> Tuple[torch.Tensor, ...]:
        """(group_ptr, group_key, member_ptr, member_rows) as views of one device tensor, filled by one asynchronous copy."""
        parts = (self.group_ptr, self.group_key, self.member_ptr, self.member_rows)
        host = torch.from_numpy(np.concatenate(parts)).pin_memory()
        dev = host.to(device, non_blocking=True)
        out, at = [], 0
        for p in parts:
            out.append(dev[at:at + len(p)])
            at += len(p)
        return tuple(out)


class DecodeState:
    """The per-graph decoding state the selection kernel updates: tokens [G, max_len], length, done and logprob in one int32 buffer
    (one copy brings them to the host), next_ids [G] int64 (the next step's embedding input), and the kernel's workspace, which holds
    (Z, winning score) per graph after each step."""

    def __init__(self, num_graphs: int, max_len: int, vocab_size: int, start_id: int, device):
        G = num_graphs
        self.num_graphs, self.max_len = G, max_len
        self.buffer = torch.zeros(G * (max_len + 3), dtype=torch.int32, device=device)
        self.tokens = self.buffer[:G * max_len].view(G, max_len)
        self.length = self.buffer[G * max_len:G * (max_len + 1)]
        self.done = self.buffer[G * (max_len + 1):G * (max_len + 2)]
        self.logprob = self.buffer[G * (max_len + 2):].view(torch.float32)
        self.next_ids = torch.full((G,), start_id, dtype=torch.int64, device=device)
        ws_bytes = N.lib().ptgnn_b200_decode_select_workspace_bytes(G, vocab_size)
        self.workspace = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
        self.workspace_bytes = ws_bytes

    def stats(self) -> torch.Tensor:
        """[G, 2] fp32: the normaliser Z and the winning score of the last step (NaN for a graph that was already done)."""
        return self.workspace[:self.num_graphs * 8].view(torch.float32).view(self.num_graphs, 2)


def check_vocab_size(V: int) -> None:
    if not N.lib().ptgnn_b200_decode_select_supported(V):
        raise NotImplementedError(f"the decode selection kernel takes a vocabulary of 1 to 65536 tokens, got {V}")


def decode_select(logits: torch.Tensor, copy_scores: torch.Tensor, lse_copy: torch.Tensor, groups: Tuple[torch.Tensor, ...],
                  state: DecodeState, step: int, end_id: int, unk_id: int) -> None:
    """``ptgnn_b200_decode_select`` for one step: logits [G, V] fp32, copy_scores [M] fp32 (the copy attention's scores in row
    order), lse_copy [G] fp32, ``groups`` from ``CopyGroups.to_device``; updates ``state`` in place."""
    x = N.require_cuda(logits, "logits", torch.float32)
    s = N.require_cuda(copy_scores, "copy_scores", torch.float32)
    lse = N.require_cuda(lse_copy, "lse_copy", torch.float32)
    G, V = x.shape
    check_vocab_size(V)
    num_rows = s.numel()
    group_ptr, group_key, member_ptr, member_rows = groups
    if G != state.num_graphs or lse.numel() != G or group_ptr.numel() != G + 1 or member_rows.numel() != num_rows:
        raise ValueError(f"decode_select: logits [{G}, {V}], lse_copy {tuple(lse.shape)}, {num_rows} copy scores and the group tables "
                         "disagree")
    N.call("ptgnn_b200_decode_select", x.device, N.ptr(x), G, V, N.ptr(s) if num_rows else None, num_rows, N.ptr(lse), N.ptr(group_ptr),
           N.ptr(group_key), N.ptr(member_ptr), N.ptr(member_rows), end_id, unk_id, step, state.max_len, N.ptr(state.done),
           N.ptr(state.length), N.ptr(state.logprob), N.ptr(state.tokens), N.ptr(state.next_ids), N.ptr(state.workspace),
           state.workspace_bytes)


def check_hidden_size(H: int) -> None:
    if H not in HIDDEN_SIZES:
        raise NotImplementedError(f"native decoding takes hidden_size in {{32, 64, 128, 256}} (the attention kernels' set), got {H}")


class _NativeDecode:
    """What greedy and beam decoding share: the constructor checks the shapes and builds the copy groups on the host (reading the origin
    map is its one host synchronisation); ``_minibatch`` does the once-per-minibatch device work."""

    def __init__(self, decoder_model, neural_model, input_concrete_values: List[str], input_memories, input_memories_origin_idx,
                 initial_states):
        self.vocab = vocab = decoder_model._GruCopyingDecoderModel__output_vocabulary
        self.module = neural_model
        gru = neural_model._GruCopyingDecoder__output_gru
        embedding = neural_model._GruCopyingDecoder__embedding_layer
        self.G, self.V, self.max_len = int(initial_states.shape[0]), len(vocab), int(decoder_model.max_seq_len)
        assert len(input_concrete_values) == input_memories.shape[0]
        check_hidden_size(gru.hidden_size)
        check_vocab_size(self.V)
        if embedding.num_embeddings != self.V:
            raise ValueError(f"the decoder embeds {embedding.num_embeddings} tokens but the output vocabulary has {self.V}")
        if input_memories.dim() != 2:
            raise ValueError(f"input_memories must be [num_inputs, D], got {tuple(input_memories.shape)}")
        self.start_id, self.end_id = vocab.get_id_or_unk(decoder_model.START), vocab.get_id_or_unk(decoder_model.END)
        self.unk_id = vocab.get_id_or_unk(vocab.get_unk())
        self.memories, self.origin_idx, self.initial_states = input_memories, input_memories_origin_idx, initial_states
        origin = input_memories_origin_idx.cpu().numpy()
        if origin.size and (origin.min() < 0 or origin.max() >= self.G):
            raise IndexError(f"input_memories_origin_idx outside [0, {self.G})")
        self.groups = CopyGroups(input_concrete_values, origin, self.G, vocab)

    def _minibatch(self):
        """Once per minibatch (call under no_grad): the group tables (one copy), the two memory projections on the native linear (rounded
        to bf16 for bf16 memories, as ``_compute_logprobs`` does) and the graph plan."""
        m = self.module
        groups = self.groups.to_device(self.memories.device)
        bf16 = self.memories.dtype == torch.bfloat16
        memories = self.memories.float() if bf16 else self.memories
        std_reps = C.linear(memories, m._GruCopyingDecoder__memories_to_standard_attention.weight, None)
        copy_reps = C.linear(memories, m._GruCopyingDecoder__memories_to_copy_attention.weight, None)
        if bf16:
            std_reps, copy_reps = std_reps.to(torch.bfloat16), copy_reps.to(torch.bfloat16)
        return groups, std_reps, copy_reps, graph_plan(self.origin_idx, self.G)


class NativeGreedyDecode(_NativeDecode):
    """One minibatch of native greedy decoding in three parts: the constructor checks the shapes and builds the copy groups on the host
    (reading the origin map is its one host synchronisation), ``run()`` enqueues all device work without synchronising, and ``result``
    copies the state back once and maps the keys to strings."""

    def run(self) -> DecodeState:
        m = self.module
        embedding = m._GruCopyingDecoder__embedding_layer
        gru = m._GruCopyingDecoder__output_gru
        dropout = m._GruCopyingDecoder__dropout
        hidden_to_vocab, vocab_bias = m._GruCopyingDecoder__hidden_to_vocab, m._GruCopyingDecoder__vocab_bias
        G, V, device = self.G, self.V, self.memories.device
        with torch.no_grad():
            groups, std_reps, copy_reps, plan = self._minibatch()
            state = DecodeState(G, self.max_len, V, self.start_id, device)
            h = self.initial_states.unsqueeze(0)
            for step in range(self.max_len):
                # one step of _compute_logprobs (decoder.py), with its dropouts
                emb = dropout(embedding(state.next_ids.unsqueeze(1)))          # [G, 1, E]
                o, h = gru(emb, h)                                              # [G, 1, H], [1, G, H]
                o = o.contiguous()
                ctx = native_attention_readout(std_reps, plan, o, 1)[0]        # [G, 1, H]
                s, lse = native_copy_attention(dropout(copy_reps), plan, o)    # [M, 1], [G, 1]
                target_scores = (
                    torch.einsum("blh,hd,vd->blv", torch.cat((dropout(ctx), o), dim=-1), hidden_to_vocab, dropout(embedding.weight))
                    + vocab_bias
                )                                                               # [G, 1, V]
                decode_select(target_scores.view(G, V), s.view(-1), lse.view(-1), groups, state, step, self.end_id, self.unk_id)
            plan.poll()
        return state

    def result(self, state: DecodeState) -> List[Tuple[List[str], float]]:
        G, T = self.G, self.max_len
        host = state.buffer.cpu()           # the one copy back: tokens, lengths, done flags and log-probabilities
        tokens = host[:G * T].view(G, T).numpy()
        length = host[G * T:G * (T + 1)].numpy()
        logprob = host[G * (T + 2):].view(torch.float32).numpy()
        return [([self.groups.name(int(k), self.vocab) for k in tokens[g, :length[g]]], np.float32(logprob[g])) for g in range(G)]


def greedy_decode(decoder_model, *, input_concrete_values: List[str], input_memories, input_memories_origin_idx, initial_states,
                  neural_model) -> List[Tuple[List[str], float]]:
    """The reference's ``GruCopyingDecoderModel.greedy_decode`` (same arguments and result) with the selection on the device.
    ``decoder_model`` is the reference's ``GruCopyingDecoderModel`` (its vocabulary, ``START``, ``END`` and ``max_seq_len`` are read);
    ``neural_model`` the reference's or this package's ``GruCopyingDecoder`` (parameters are read by their mangled names, which are the
    same in both).  fp32 or bf16 memories; hidden size in {32, 64, 128, 256}; vocabulary of 1 to 65536 tokens."""
    dec = NativeGreedyDecode(decoder_model, neural_model, input_concrete_values, input_memories, input_memories_origin_idx, initial_states)
    if dec.G == 0 or dec.max_len == 0:
        return [([], 0.0) for _ in range(dec.G)]
    return dec.result(dec.run())


# ---- beam search (DESIGN §3.19) ----------------------------------------------------------------------------------------------------
MAX_BEAM_WIDTH = 8


def check_beam_width(beam_width: int) -> None:
    if beam_width < 1:
        raise ValueError(f"beam_width must be at least 1, got {beam_width}")
    if beam_width > MAX_BEAM_WIDTH:
        raise NotImplementedError(f"beam search takes beam_width up to {MAX_BEAM_WIDTH} (the attention kernels' query rows), got {beam_width}")


class BeamState:
    """The beam state the selection kernels update, for G graphs, K slots and max_len steps: one int32 buffer (one copy brings it to the
    host) holding the per-step backpointers and keys [max_len, G, K] and the per-slot totals (fp32), lengths, done and empty flags
    [G, K]; next_ids [G·K] int64 (the next step's embedding input); gather_idx [G·K] int64 (the row of each slot's parent, for the
    hidden-state reorder); and the kernels' workspace, which starts with Z per (graph, slot) after each step."""

    def __init__(self, num_graphs: int, beam_width: int, max_len: int, vocab_size: int, start_id: int, device):
        G, K, T = num_graphs, beam_width, max_len
        self.num_graphs, self.beam_width, self.max_len = G, K, T
        gk = G * K
        self.buffer = torch.zeros(gk * (2 * T + 4), dtype=torch.int32, device=device)
        self.backpointers = self.buffer[:T * gk].view(T, G, K)
        self.keys = self.buffer[T * gk:2 * T * gk].view(T, G, K)
        self.total = self.buffer[2 * T * gk:(2 * T + 1) * gk].view(torch.float32).view(G, K)
        self.length = self.buffer[(2 * T + 1) * gk:(2 * T + 2) * gk].view(G, K)
        self.done = self.buffer[(2 * T + 2) * gk:(2 * T + 3) * gk].view(G, K)
        self.empty = self.buffer[(2 * T + 3) * gk:].view(G, K)
        self.next_ids = torch.full((gk,), start_id, dtype=torch.int64, device=device)
        self.gather_idx = torch.arange(gk, dtype=torch.int64, device=device)
        ws_bytes = N.lib().ptgnn_b200_beam_select_workspace_bytes(G, vocab_size, K)
        self.workspace = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
        self.workspace_bytes = ws_bytes

    def stats(self) -> torch.Tensor:
        """[G, K] fp32: the normaliser Z of each slot at the last step (NaN for a slot that was done or empty)."""
        gk = self.num_graphs * self.beam_width
        return self.workspace[:gk * 4].view(torch.float32).view(self.num_graphs, self.beam_width)


def beam_select(logits: torch.Tensor, copy_scores: torch.Tensor, lse_copy: torch.Tensor, groups: Tuple[torch.Tensor, ...],
                state: BeamState, step: int, end_id: int, unk_id: int) -> None:
    """``ptgnn_b200_beam_select`` for one step: logits [G·K, V] fp32 (rows graph-major), copy_scores [M, K] fp32 (the copy attention's
    scores in row order, one column per slot), lse_copy [G, K] fp32, ``groups`` from ``CopyGroups.to_device``; updates ``state``."""
    x = N.require_cuda(logits, "logits", torch.float32)
    s = N.require_cuda(copy_scores, "copy_scores", torch.float32)
    lse = N.require_cuda(lse_copy, "lse_copy", torch.float32)
    G, K = state.num_graphs, state.beam_width
    V = x.shape[1]
    check_vocab_size(V)
    num_rows = s.shape[0]
    group_ptr, group_key, member_ptr, member_rows = groups
    if (x.shape[0] != G * K or tuple(lse.shape) != (G, K) or s.dim() != 2 or s.shape[1] != K or group_ptr.numel() != G + 1
            or member_rows.numel() != num_rows):
        raise ValueError(f"beam_select: logits {tuple(x.shape)}, lse_copy {tuple(lse.shape)}, copy scores {tuple(s.shape)}, {G} graphs "
                         f"of {K} slots and the group tables disagree")
    N.call("ptgnn_b200_beam_select", x.device, N.ptr(x), G, V, K, N.ptr(s) if num_rows else None, num_rows, N.ptr(lse),
           N.ptr(group_ptr), N.ptr(group_key), N.ptr(member_ptr), N.ptr(member_rows), end_id, unk_id, step, state.max_len,
           N.ptr(state.buffer), N.ptr(state.next_ids), N.ptr(state.gather_idx), N.ptr(state.workspace), state.workspace_bytes)


class NativeBeamDecode(_NativeDecode):
    """One minibatch of native beam search, in the three parts of ``NativeGreedyDecode``: the constructor (host work, one read of the
    origin map), ``run()`` (all device work, no synchronisation) and ``result`` (one copy back, then the backtrack on the host)."""

    def __init__(self, decoder_model, neural_model, input_concrete_values: List[str], input_memories, input_memories_origin_idx,
                 initial_states, beam_width: int):
        check_beam_width(beam_width)
        self.K = int(beam_width)
        super().__init__(decoder_model, neural_model, input_concrete_values, input_memories, input_memories_origin_idx, initial_states)

    def run(self) -> BeamState:
        m = self.module
        embedding = m._GruCopyingDecoder__embedding_layer
        gru = m._GruCopyingDecoder__output_gru
        dropout = m._GruCopyingDecoder__dropout
        hidden_to_vocab, vocab_bias = m._GruCopyingDecoder__hidden_to_vocab, m._GruCopyingDecoder__vocab_bias
        G, K, V, device = self.G, self.K, self.V, self.memories.device
        heads = _padded_steps(K)
        with torch.no_grad():
            groups, std_reps, copy_reps, plan = self._minibatch()
            state = BeamState(G, K, self.max_len, V, self.start_id, device)
            h = self.initial_states.repeat_interleave(K, dim=0).unsqueeze(0)            # [1, G·K, H], rows graph-major
            for step in range(self.max_len):
                # one step of _compute_logprobs (decoder.py) on G·K rows, the K slots as the attention kernels' query rows
                emb = dropout(embedding(state.next_ids.unsqueeze(1)))                  # [G·K, 1, E]
                o, h = gru(emb, h)                                                      # [G·K, 1, H], [1, G·K, H]
                o = o.contiguous().view(G, K, -1)                                       # [G, K, H]
                queries = o if heads == K else torch.nn.functional.pad(o, (0, 0, 0, heads - K))
                ctx = native_attention_readout(std_reps, plan, queries, heads)[0][:, :K]     # [G, K, H]
                s, lse = native_copy_attention(dropout(copy_reps), plan, o)            # [M, K], [G, K]
                target_scores = (
                    torch.einsum("blh,hd,vd->blv", torch.cat((dropout(ctx), o), dim=-1), hidden_to_vocab, dropout(embedding.weight))
                    + vocab_bias
                )                                                                       # [G, K, V]
                beam_select(target_scores.view(G * K, V), s, lse, groups, state, step, self.end_id, self.unk_id)
                h = h.index_select(1, state.gather_idx)
            plan.poll()
        return state

    def result(self, state: BeamState) -> List[List[Tuple[List[str], np.float32]]]:
        G, K, T = self.G, self.K, self.max_len
        gk = G * K
        host = state.buffer.cpu()           # the one copy back: backpointers, keys, totals, lengths, done and empty flags
        bp = host[:T * gk].view(T, G, K).numpy()
        keys = host[T * gk:2 * T * gk].view(T, G, K).numpy()
        total = host[2 * T * gk:(2 * T + 1) * gk].view(torch.float32).view(G, K).numpy()
        length = host[(2 * T + 1) * gk:(2 * T + 2) * gk].view(G, K).numpy()
        empty = host[(2 * T + 3) * gk:].view(G, K).numpy()
        out = []
        for g in range(G):
            hyps = []
            for k in range(K):              # the slots are in rank order: best first, by total and then slot
                if empty[g, k]:
                    continue
                path, j = [], k
                for t in range(T - 1, -1, -1):
                    key = int(keys[t, g, j])
                    if key >= 0 and key != self.end_id:
                        path.append(key)
                    j = int(bp[t, g, j])
                assert len(path) == length[g, k], (g, k, path, length[g, k])
                hyps.append(([self.groups.name(key, self.vocab) for key in reversed(path)], np.float32(total[g, k])))
            out.append(hyps)
        return out


def beam_decode(decoder_model, *, input_concrete_values: List[str], input_memories, input_memories_origin_idx, initial_states,
                neural_model, beam_width: int) -> List[List[Tuple[List[str], np.float32]]]:
    """Beam search with the selection on the device (DESIGN §3.19): the arguments of ``greedy_decode`` plus ``beam_width`` K in [1, 8].

    Per graph, K slots; each is live, done or empty.  At step 0 slot 0 is live with START, total 0 and the graph's initial state, the
    others empty.  A live slot's candidates are greedy decoding's dictionary for its step (the top 100 of ``lp = x - Z`` merged with
    its copy groups), each with total ``fl(cum + score)`` in fp32; a done slot has one candidate, itself, unchanged, and feeds END; an
    empty slot has none.  Per graph the K best candidates, by total descending, then source slot ascending, then greedy's order within
    the slot (score descending, members of the top 100 by lp descending and id ascending, then groups outside it in first-occurrence
    order), become the new slots; a selected END makes its slot done; if fewer than K exist the rest stay empty.  All ``max_seq_len``
    steps run.  Returns, per graph, its non-empty slots best first (total descending, then slot): (tokens, fp32 total), unfinished
    hypotheses included, without length normalisation.  With K = 1 this is ``greedy_decode`` exactly.

    ``beam_width < 1`` raises ValueError; ``beam_width > 8``, a hidden size outside {32, 64, 128, 256} or a vocabulary outside 1 to 65536
    tokens raise NotImplementedError, all before any launch."""
    dec = NativeBeamDecode(decoder_model, neural_model, input_concrete_values, input_memories, input_memories_origin_idx, initial_states,
                           beam_width)
    if dec.G == 0 or dec.max_len == 0:
        return [[([], np.float32(0.0))] for _ in range(dec.G)]
    return dec.result(dec.run())
