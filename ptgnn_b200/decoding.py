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
"""
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _native as N
from . import composed as C
from .decoder import native_copy_attention
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


class NativeGreedyDecode:
    """One minibatch of native greedy decoding in three parts: the constructor checks the shapes and builds the copy groups on the host
    (reading the origin map is its one host synchronisation), ``run()`` enqueues all device work without synchronising, and ``result``
    copies the state back once and maps the keys to strings."""

    def __init__(self, decoder_model, neural_model, input_concrete_values: List[str], input_memories, input_memories_origin_idx,
                 initial_states):
        self.vocab = vocab = decoder_model._GruCopyingDecoderModel__output_vocabulary
        self.module = neural_model
        gru = neural_model._GruCopyingDecoder__output_gru
        embedding = neural_model._GruCopyingDecoder__embedding_layer
        self.G, self.V, self.max_len = int(initial_states.shape[0]), len(vocab), int(decoder_model.max_seq_len)
        assert len(input_concrete_values) == input_memories.shape[0]
        if gru.hidden_size not in HIDDEN_SIZES:
            raise NotImplementedError(f"native greedy decoding takes hidden_size in {{32, 64, 128, 256}} (the attention kernels' set), "
                                      f"got {gru.hidden_size}")
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

    def run(self) -> DecodeState:
        m = self.module
        embedding = m._GruCopyingDecoder__embedding_layer
        gru = m._GruCopyingDecoder__output_gru
        dropout = m._GruCopyingDecoder__dropout
        hidden_to_vocab, vocab_bias = m._GruCopyingDecoder__hidden_to_vocab, m._GruCopyingDecoder__vocab_bias
        G, V, device = self.G, self.V, self.memories.device
        with torch.no_grad():
            # once per minibatch: the group tables (one copy), the memory projections on the native linear, the graph plan
            groups = self.groups.to_device(device)
            bf16 = self.memories.dtype == torch.bfloat16
            memories = self.memories.float() if bf16 else self.memories
            std_reps = C.linear(memories, m._GruCopyingDecoder__memories_to_standard_attention.weight, None)
            copy_reps = C.linear(memories, m._GruCopyingDecoder__memories_to_copy_attention.weight, None)
            if bf16:
                std_reps, copy_reps = std_reps.to(torch.bfloat16), copy_reps.to(torch.bfloat16)
            plan = graph_plan(self.origin_idx, G)
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
