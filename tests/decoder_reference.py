"""A restatement of the reference's graph2seq decoder (``GruCopyingDecoder``, grucopydecoder.py:59-212) in plain torch ops, for the
tests: run in float64 it is the yardstick of the native decoder, and it reproduces the reference's fixtures (tests/golden/decoder_*.npz).

Parameters come as a dict keyed like the module's ``state_dict`` (the ``_GruCopyingDecoder__`` prefix is added here).  ``masks``, when
given, are the four dropout multipliers (0 or 1 / (1 - p)) in the reference's order: token embeddings [G, L, E], copy representations
[M, H], standard attention output [G, L, H], embedding weight [V, E]; None is eval mode.
"""
import math

import torch

P = "_GruCopyingDecoder__"
PARAMS = ("embedding_layer.weight", "output_gru.weight_ih_l0", "output_gru.weight_hh_l0", "output_gru.bias_ih_l0", "output_gru.bias_hh_l0",
          "memories_to_standard_attention.weight", "memories_to_copy_attention.weight", "hidden_to_vocab", "vocab_bias")


def gru(x, h, w_ih, w_hh, b_ih, b_hh):
    """torch.nn.GRU (one layer, batch_first, gate order r, z, n): (outputs [G, L, H], last state [G, H])."""
    outs = []
    for t in range(x.shape[1]):
        gi = x[:, t] @ w_ih.t() + b_ih
        gh = h @ w_hh.t() + b_hh
        ir, iz, i_n = gi.chunk(3, dim=1)
        hr, hz, hn = gh.chunk(3, dim=1)
        r, z = torch.sigmoid(ir + hr), torch.sigmoid(iz + hz)
        n = torch.tanh(i_n + r * hn)
        h = (1 - z) * n + z * h
        outs.append(h)
    return torch.stack(outs, dim=1), h


def segment_logsumexp(src, index, n):
    """scatter_logsumexp(src, index, dim=0, dim_size=n, eps=0) for src [K] or [K, L]: an empty segment gives -inf."""
    shape = (n,) + tuple(src.shape[1:])
    idx = index.reshape((-1,) + (1,) * (src.dim() - 1)).expand(src.shape)
    mx = torch.full(shape, -math.inf, dtype=src.dtype).scatter_reduce(0, idx, src.detach(), "amax", include_self=True)
    mx = torch.where(torch.isinf(mx), torch.zeros_like(mx), mx)
    total = torch.zeros(shape, dtype=src.dtype).index_add(0, index, torch.exp(src - mx[index]))
    return torch.log(total) + mx


def compute_logprobs(sd, initial_states, memories, origin, token_ids, masks=None):
    """_compute_logprobs: (copy_logprobs [M, L], target_logprobs [G, L, V], gru_state [1, G, H])."""
    w = {k: sd[P + k] for k in PARAMS}
    drop = (lambda t, i: t) if masks is None else (lambda t, i: t * masks[i])
    emb = drop(w["embedding_layer.weight"][token_ids], 0)
    out, h = gru(emb, initial_states, w["output_gru.weight_ih_l0"], w["output_gru.weight_hh_l0"], w["output_gru.bias_ih_l0"],
                 w["output_gru.bias_hh_l0"])
    G, L, H = out.shape
    A = memories @ w["memories_to_standard_attention.weight"].t()
    C = drop(memories @ w["memories_to_copy_attention.weight"].t(), 1)
    per_row = out[origin]                                                           # [M, L, H]
    z = torch.einsum("ilh,ih->il", per_row, A)
    p = torch.exp(z - segment_logsumexp(z, origin, G)[origin])
    ctx = torch.zeros(G, L, H, dtype=out.dtype).index_add(0, origin, p[:, :, None] * A[:, None, :])
    s = torch.einsum("ilh,ih->il", per_row, C)
    lse = segment_logsumexp(s, origin, G)
    target_scores = torch.einsum("blh,hd,vd->blv", torch.cat((drop(ctx, 2), out), dim=-1), w["hidden_to_vocab"],
                                 drop(w["embedding_layer.weight"], 3)) + w["vocab_bias"]
    norm = torch.logsumexp(torch.cat((target_scores, lse.unsqueeze(-1)), dim=-1), dim=-1)
    return s - norm[origin], target_scores - norm.unsqueeze(-1), h.unsqueeze(0)


def loss(sd, unk_id, memories, origin, initial_states, target_token_ids, copyable_elements_idxs, copyable_elements_sample_idxs,
         target_lengths, masks=None):
    """forward: the decoder's loss."""
    copy_lp, target_lp, _ = compute_logprobs(sd, initial_states, memories, origin, target_token_ids[:, :-1], masks)
    G, L = target_token_ids.shape[0], target_token_ids.shape[1] - 1
    valid = torch.zeros(G * L, dtype=torch.int64).index_add(0, copyable_elements_sample_idxs, torch.ones_like(copyable_elements_sample_idxs))
    mask = (valid.reshape(G, L) > 0) & (target_token_ids[:, 1:] == unk_id)
    gen = torch.gather(target_lp, index=target_token_ids[:, 1:].unsqueeze(-1), dim=-1).squeeze(-1).masked_fill(mask, -math.inf)
    cp = segment_logsumexp(copy_lp.flatten()[copyable_elements_idxs], copyable_elements_sample_idxs, G * L).view(G, L)
    anyc = torch.logsumexp(torch.stack((gen, cp)), dim=0)
    keep = (torch.arange(L).unsqueeze(0) < target_lengths.unsqueeze(1)).to(anyc.dtype)
    return -((anyc * keep).sum(dim=-1) / keep.sum(dim=-1)).mean()
