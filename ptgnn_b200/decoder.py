"""The graph2seq decoder, ``GruCopyingDecoder`` (reference ``neuralmodels/sequence/grucopydecoder.py:29-212``), with its attention over
the memories on native kernels (DESIGN §3.11).

For sample g, step l and memory row i of g, with O the GRU outputs ``[G, L, H]``, A = ``memories W_stdᵀ`` and
C = ``dropout(memories W_copyᵀ)`` (``[M, H]`` each):

* standard attention ``ctx[g, l] = Σ_i softmax_i(O[g, l]·A_i) A_i`` is the attention readout (``native_attention_readout``, §3.7) with
  x = A and the steps as heads: L is padded with zero query rows to the next head count it takes;
* copy attention ``s[i, l] = C_i·O[g(i), l]`` and ``lse[g, l] = log Σ_i exp s[i, l]`` is ``ptgnn_b200_copy_attention``, with ``s``
  written in the caller's memory-row order.

So the reference's ``[M, L, H]`` gathered decoder states, and the products autograd keeps of that size, are never formed.  The token
embedding, the GRU, the vocabulary projection and the normalisation stay library ops, written as the reference writes them, and the
loss makes no ``torch_scatter`` call.  Constructor, parameter creation order and (name-mangled) ``state_dict`` keys are the
reference's.  Forward in fp32, or with bf16 memories (A and C rounded to bf16 for the kernels, fp32 outputs); gradients in fp32.
"""
import math

import torch
import torch.nn as nn

from . import _native as N
from . import autograd as _ag
from . import composed as C
from .edgeplan import EdgePlan, plan_for
from .reduceops import graph_plan, native_attention_readout

_STEPS = "the decoder's attention kernels take at most 8 steps"


def _padded_steps(L: int) -> int:
    """The attention readout's head count for L steps: L rounded up to {1, 2, 4, 8}."""
    if L > 8:
        raise NotImplementedError(f"{_STEPS}, got {L}")
    return 1 << (L - 1).bit_length()


def native_copy_attention(copy_reps: torch.Tensor, plan: EdgePlan, o: torch.Tensor):
    """``ptgnn_b200_copy_attention``: (s [M, L] fp32 in row order, lse [G, L] fp32) with s[i, l] = c_i . o[graph(i), l].  fp32 or bf16
    copy_reps [M, H]; o [G, L, H] fp32; H in {32, 64, 128, 256}, L in [1, 8]."""
    bf16 = copy_reps.dtype == torch.bfloat16
    c = N.require_cuda(copy_reps, "copy_reps", torch.bfloat16 if bf16 else torch.float32)
    q = N.require_cuda(o, "o", torch.float32)
    G = plan.num_nodes
    if c.dim() != 2 or q.dim() != 3 or q.shape[0] != G or q.shape[2] != c.shape[1]:
        raise ValueError(f"copy_reps [M, H] and o [{G}, L, H] disagree: {tuple(c.shape)}, {tuple(q.shape)}")
    num_rows, H = c.shape
    L = q.shape[1]
    if plan.num_edges != num_rows:
        raise ValueError("input_memories_origin_idx and the memories disagree on the number of rows")
    lib = N.lib()
    if not lib.ptgnn_b200_copy_attention_supported(int(bf16), H, L):
        raise NotImplementedError(f"the copy attention kernel takes H in {{32, 64, 128, 256}} and at most 8 steps, got H={H}, L={L}")
    ws_bytes = lib.ptgnn_b200_copy_attention_workspace_bytes(num_rows, G, H, L)
    s = torch.empty(num_rows, L, dtype=torch.float32, device=c.device)
    lse = torch.empty(G, L, dtype=torch.float32, device=c.device)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=c.device)
    with torch.cuda.device(c.device):
        rc = lib.ptgnn_b200_copy_attention(int(bf16), N.ptr(c), num_rows, H, L, N.ptr(plan.row_ptr), N.ptr(plan.perm) if num_rows else None,
                                           G, N.ptr(q), N.ptr(s), N.ptr(lse), N.ptr(ws), ws_bytes, N.current_stream(c.device))
    N.check(rc, "ptgnn_b200_copy_attention")
    return s, lse


def native_copy_attention_backward(copy_reps: torch.Tensor, plan: EdgePlan, o: torch.Tensor, lse: torch.Tensor, d_s: torch.Tensor,
                                   d_lse: torch.Tensor):
    """``ptgnn_b200_copy_attention_backward_f32``: (d_copy_reps [M, H], d_o [G, L, H]) from d_s [M, L] and d_lse [G, L].  fp32 only."""
    c = N.require_cuda(copy_reps, "copy_reps", torch.float32)
    q = N.require_cuda(o, "o", torch.float32)
    num_rows, H = c.shape
    G, L = q.shape[0], q.shape[1]
    tabs = [N.require_cuda(t, n, torch.float32) for t, n in ((lse, "lse"), (d_s, "d_s"), (d_lse, "d_lse"))]
    for t, n, shape in zip(tabs, ("lse", "d_s", "d_lse"), ((G, L), (num_rows, L), (G, L))):
        if tuple(t.shape) != shape:                 # raw pointers cross the C ABI next
            raise ValueError(f"{n} must be {shape}, got {tuple(t.shape)}")
    lib = N.lib()
    ws_bytes = lib.ptgnn_b200_copy_attention_workspace_bytes(num_rows, G, H, L)
    if ws_bytes == 0:
        raise NotImplementedError(f"the copy attention kernel takes H in {{32, 64, 128, 256}} and at most 8 steps, got H={H}, L={L}")
    d_c = torch.empty_like(c)
    d_o = torch.empty(G, L, H, dtype=torch.float32, device=c.device)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=c.device)
    with torch.cuda.device(c.device):
        rc = lib.ptgnn_b200_copy_attention_backward_f32(N.ptr(c), num_rows, H, L, N.ptr(plan.row_ptr), N.ptr(plan.perm) if num_rows else None,
                                                        G, N.ptr(q), N.ptr(tabs[0]), N.ptr(tabs[1]), N.ptr(tabs[2]), N.ptr(d_c), N.ptr(d_o),
                                                        N.ptr(ws), ws_bytes, N.current_stream(c.device))
    N.check(rc, "ptgnn_b200_copy_attention_backward_f32")
    return d_c, d_o


def segment_logsumexp(src: torch.Tensor, index: torch.Tensor, num_segments: int) -> torch.Tensor:
    """``torch_scatter.scatter_logsumexp(src, index, dim_size=num_segments, eps=0)`` for 1-D fp32 ``src``, differentiable: a segment
    without elements gives -inf, and no NaN reaches ``src``'s gradient (an empty segment has no element to pass it to).  The sums run
    on the native segmented reduce over the plan of ``index`` (elements in order, no float atomics), so they repeat bit for bit."""
    mx = torch.full((num_segments,), -math.inf, dtype=src.dtype, device=src.device)
    mx = mx.scatter_reduce(0, index, src.detach(), "amax", include_self=True)
    mx = torch.where(torch.isinf(mx), torch.zeros_like(mx), mx)
    terms = nn.functional.pad(torch.exp(src - mx[index]).unsqueeze(1), (0, 3))      # the reduce takes widths that are multiples of 4
    total = _ag._SegmentReduceFn.apply(terms, plan_for([(index, index)], num_segments), "sum")[:, 0]
    return torch.log(total) + mx


class GruCopyingDecoder(nn.Module):
    def __init__(
        self,
        vocabulary_size: int,
        embedding_size: int,
        hidden_size: int,
        memories_hidden_dim: int,
        unk_id: int,
        dropout_rate: float,
    ):
        super().__init__()
        self.__embedding_layer = nn.Embedding(num_embeddings=vocabulary_size, embedding_dim=embedding_size)
        self.__output_gru = nn.GRU(input_size=embedding_size, hidden_size=hidden_size, num_layers=1, batch_first=True)

        self.__unk_id = unk_id

        self.__memories_to_standard_attention = nn.Linear(in_features=memories_hidden_dim, out_features=hidden_size, bias=False)
        self.__memories_to_copy_attention = nn.Linear(in_features=memories_hidden_dim, out_features=hidden_size, bias=False)
        self.__hidden_to_vocab = nn.Parameter(0.01 * torch.randn((2 * hidden_size, embedding_size)))
        self.__vocab_bias = nn.Parameter(torch.zeros(vocabulary_size))
        self.__dropout = nn.Dropout(dropout_rate)

    def _compute_logprobs(self, initial_states, input_memories, input_memories_origin_idx, input_token_ids):
        """
        :param input_memories: [num-inputs-flattened, D]
        :param input_memories_origin_idx: [num-inputs-flattened]
        :param initial_states: [num-targets, H]
        :param input_token_ids: [num-targets, max-seq-size-1]

        :return: the logprobs for all copying locations and the logprobs for all elements in the vocabulary
        """
        if input_memories.dim() != 2:
            raise ValueError(f"input_memories must be [num_inputs, D], got {tuple(input_memories.shape)}")
        grad = _ag.needs_grad(self, input_memories) or (torch.is_grad_enabled() and initial_states.requires_grad)
        bf16 = input_memories.dtype == torch.bfloat16
        if grad and bf16:
            raise NotImplementedError("GruCopyingDecoder with gradients: fp32 memories only (call it under torch.no_grad() for bf16)")
        L = input_token_ids.shape[1]
        heads = _padded_steps(L)
        H = self.__output_gru.hidden_size
        if not N.lib().ptgnn_b200_copy_attention_supported(int(bf16), H, L):
            raise NotImplementedError(f"the decoder's attention kernels take hidden_size in {{32, 64, 128, 256}}, got {H}")

        target_token_embeddings = self.__dropout(self.__embedding_layer(input_token_ids))  # [num-targets, max-seq-size - 1, E]
        output_states, output_gru_state = self.__output_gru(target_token_embeddings, initial_states.unsqueeze(0))
        output_states = output_states.contiguous()  # [num-targets, max-seq-size - 1, H]
        G = output_states.shape[0]
        plan = graph_plan(input_memories_origin_idx, G)

        # Standard and copy attention representations [num-inputs-flattened, H] on the native dense kernel (exact up-cast of bf16)
        memories = input_memories.float() if bf16 else input_memories
        linear = _ag._LinearFn.apply if grad else C.linear
        standard_attention_reps = linear(memories, self.__memories_to_standard_attention.weight, None)
        copy_attention_reps = self.__dropout(linear(memories, self.__memories_to_copy_attention.weight, None))
        if bf16:
            standard_attention_reps = standard_attention_reps.to(torch.bfloat16)
            copy_attention_reps = copy_attention_reps.to(torch.bfloat16)

        # Standard attention: the attention readout with the steps as heads (zero query rows pad L up to the head count)
        queries = output_states if heads == L else nn.functional.pad(output_states, (0, 0, 0, heads - L))
        if grad:
            ctx = _ag.attention_readout_with_grad(plan, heads, standard_attention_reps, queries)
        else:
            ctx = native_attention_readout(standard_attention_reps, plan, queries, heads)[0]
        standard_attention_out = ctx[:, :L].contiguous()  # [num-targets, max-seq-size - 1, H]

        # Copy attention: the scores [num-inputs-flattened, max-seq-size - 1] and their per-sample logsumexp
        if grad:
            copy_attention_scores, total_copy_scores = _ag.copy_attention_with_grad(plan, copy_attention_reps, output_states)
        else:
            copy_attention_scores, total_copy_scores = native_copy_attention(copy_attention_reps, plan, output_states)
        plan.poll()
        # the [M, H] operands are not needed past here (autograd keeps what it saved): a forward without gradients frees them before
        # the [G, L, V] vocabulary tensors exist
        del standard_attention_reps, copy_attention_reps, ctx

        target_scores = (
            torch.einsum(
                "blh,hd,vd->blv",
                torch.cat((self.__dropout(standard_attention_out), output_states), dim=-1),
                self.__hidden_to_vocab,
                self.__dropout(self.__embedding_layer.weight),
            )
            + self.__vocab_bias
        )  # [num-targets, max-seq-size - 1, vocab-size]

        # A "manual" log_softmax over [num-targets, max-seq-size - 1, vocab-size + 1]
        normalizing_const = torch.logsumexp(torch.cat((target_scores, total_copy_scores.unsqueeze(-1)), dim=-1), dim=-1)

        target_logprobs = target_scores - normalizing_const.unsqueeze(-1)  # [num-targets, max-seq-size - 1, vocab-size]
        copy_logprobs = copy_attention_scores - _ag.gather_by_graph(plan, input_memories_origin_idx, normalizing_const)  # [num-inputs-flattened, max-seq-size - 1]
        return copy_logprobs, target_logprobs, output_gru_state

    def forward(
        self,
        *,
        input_memories,
        input_memories_origin_idx,
        initial_states,
        target_token_ids,
        copyable_elements_idxs,
        copyable_elements_sample_idxs,
        target_lengths
    ):
        """
        :param input_memories: [num-inputs-flattened, D]
        :param input_memories_origin_idx: [num-inputs-flattened]
        :param initial_states: [num-targets, H]
        :param target_token_ids: [num-targets, max-seq-size]
        :param target_lengths: [num-targets]
        :param copyable_elements_idxs: [num-copyable-elements]
        :param copyable_elements_sample_idxs: [num-copyable-elements]

        :return: the loss function.
        """
        copy_logprobs, target_logprobs, _ = self._compute_logprobs(
            initial_states, input_memories, input_memories_origin_idx, target_token_ids[:, :-1]
        )
        num_locations = target_token_ids.shape[0] * (target_token_ids.shape[1] - 1)

        # Get loss. UNKs are only predicted if we cannot copy.
        num_valid_copy_actions = torch.zeros(
            num_locations, dtype=copyable_elements_sample_idxs.dtype, device=copyable_elements_sample_idxs.device
        ).index_add_(0, copyable_elements_sample_idxs, torch.ones_like(copyable_elements_sample_idxs))
        locations_with_valid_copy_actions = (
            num_valid_copy_actions.reshape(target_token_ids.shape[0], target_token_ids.shape[1] - 1) > 0
        )
        unk_prediction_locations = target_token_ids[:, 1:] == self.__unk_id
        mask = locations_with_valid_copy_actions & unk_prediction_locations

        correct_generation_logprobs = torch.gather(
            target_logprobs, index=target_token_ids[:, 1:].unsqueeze(-1), dim=-1
        ).squeeze(-1)  # [num-targets, max-seq-size - 1]
        correct_generation_logprobs.masked_fill_(mask, -math.inf)

        correct_copy_logprobs = segment_logsumexp(
            copy_logprobs.flatten()[copyable_elements_idxs], copyable_elements_sample_idxs, num_locations
        )  # [num-targets * (max-seq-size - 1)]
        correct_copy_logprobs = correct_copy_logprobs.view(target_token_ids.shape[0], target_token_ids.shape[1] - 1)

        any_correct_action_logprob = torch.logsumexp(
            torch.stack((correct_generation_logprobs, correct_copy_logprobs)), dim=0
        )  # [num-targets, max-seq-size - 1]

        mask = torch.arange(any_correct_action_logprob.shape[1], device=target_lengths.device).unsqueeze(0) < target_lengths.unsqueeze(1)
        per_seq_loss = (any_correct_action_logprob * mask.float()).sum(dim=-1) / mask.float().sum(dim=-1)

        return -per_seq_loss.mean()
