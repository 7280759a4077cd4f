"""Generates the graph2seq decoder fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_decoder_golden.py          # writes tests/golden/decoder_*.npz

The reference's ``GruCopyingDecoder`` (``neuralmodels/sequence/grucopydecoder.py``) is imported read-only through
``oracle/refimport.py``, whose ``torch_scatter`` stand-in is differentiable, so ``loss.backward()`` reaches every parameter.  Each
fixture stores the seeded inputs, the module's ``state_dict`` (keys prefixed ``sd::``), the outputs of ``_compute_logprobs`` in eval
mode (``copy_logprobs``, ``target_logprobs``, ``gru_state``), the loss, and the autograd gradients of the loss w.r.t. the memories
(``grad::memories``), the initial states (``grad::initial_states``) and every parameter (``grad::<name>``).

The memory rows of sample g are shuffled among the other samples' (an unsorted origin map); one sample has no memory and is not
the last (the reference's ``scatter_add`` sizes its output by the largest id); the samples hold 1, 31, 33 and more than 64 rows.
Every sample gets copyable rows at some steps and none at others, one step predicts UNK with a valid copy, one predicts UNK
without, and the target lengths are shorter than the batch maximum for most samples.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.sequence.grucopydecoder import GruCopyingDecoder  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
UNK = 0

# name -> (hidden H, steps L, memory rows per sample, memories D, embedding E, vocabulary V)
CASES = {
    "decoder_h32_l1": (32, 1, [1, 0, 31, 33, 70], 24, 16, 50),
    "decoder_h32_l4": (32, 4, [33, 1, 0, 70, 31], 24, 16, 50),
    "decoder_h128_l4": (128, 4, [1, 65, 0, 31, 33], 64, 48, 300),
    "decoder_h128_l7": (128, 7, [70, 31, 0, 33, 1, 5], 64, 48, 300),
}


def make_inputs(H, L, counts, D, V, gen):
    """(memories, origin, initial_states, target_token_ids, copyable_elements_idxs, copyable_elements_sample_idxs, target_lengths)
    in the layout of GruCopyingDecoderModel.finalize_minibatch: a copyable row i at step t of sample g is the flat index i * L + t of
    copy_logprobs [M, L] and the location g * L + t."""
    G = len(counts)
    origin = torch.repeat_interleave(torch.arange(G), torch.tensor(counts))
    origin = origin[torch.randperm(origin.numel(), generator=gen)]
    M = origin.numel()
    memories = torch.randn(M, D, generator=gen)
    initial_states = torch.randn(G, H, generator=gen) * 0.5
    tokens = torch.randint(1, V, (G, L + 1), generator=gen)
    ce, ces = [], []
    for g in range(G):
        rows = torch.nonzero(origin == g).flatten()
        for t in range(L):
            if len(rows) == 0 or torch.rand(1, generator=gen).item() < 0.4:
                continue                                   # a step with no copyable element
            pick = rows[torch.rand(len(rows), generator=gen) < 0.3]
            if len(pick) == 0:
                pick = rows[:1]
            ce += (pick * L + t).tolist()
            ces += [g * L + t] * len(pick)
    ce, ces = torch.tensor(ce, dtype=torch.int64), torch.tensor(ces, dtype=torch.int64)
    with_copy = set(ces.tolist())
    # one UNK target with a valid copy, one without
    unk_copy = next(loc for loc in sorted(with_copy))
    tokens[unk_copy // L, unk_copy % L + 1] = UNK
    unk_none = next(loc for loc in range(G * L) if loc not in with_copy)
    tokens[unk_none // L, unk_none % L + 1] = UNK
    lengths = torch.randint(1, L + 2, (G,), generator=gen)
    lengths[0] = L + 1
    return memories, origin, initial_states, tokens, ce, ces, lengths


def run(module, memories, origin, initial_states, tokens, ce, ces, lengths):
    """(copy_logprobs, target_logprobs, gru_state) in eval mode, the loss and its gradients."""
    module.eval()
    with torch.no_grad():
        copy_lp, target_lp, gru_state = module._compute_logprobs(initial_states, memories, origin, tokens[:, :-1])
    mem, h0 = memories.clone().requires_grad_(True), initial_states.clone().requires_grad_(True)
    module.zero_grad()
    loss = module(input_memories=mem, input_memories_origin_idx=origin, initial_states=h0, target_token_ids=tokens,
                  copyable_elements_idxs=ce, copyable_elements_sample_idxs=ces, target_lengths=lengths)
    loss.backward()
    grads = {"grad::memories": mem.grad.numpy(), "grad::initial_states": h0.grad.numpy()}
    grads.update({"grad::" + n: p.grad.numpy() for n, p in module.named_parameters()})
    return copy_lp, target_lp, gru_state, loss.detach(), grads


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def main():
    for i, (name, (H, L, counts, D, E, V)) in enumerate(CASES.items()):
        torch.manual_seed(7000 + i)
        module = GruCopyingDecoder(V, E, H, D, unk_id=UNK, dropout_rate=0.2)
        gen = torch.Generator().manual_seed(8000 + i)
        inputs = make_inputs(H, L, counts, D, V, gen)
        copy_lp, target_lp, gru_state, loss, grads = run(module, *inputs)
        assert all(np.isfinite(g).all() for g in grads.values()), f"{name}: non-finite gradient"
        names = ("memories", "origin", "initial_states", "target_token_ids", "copyable_elements_idxs", "copyable_elements_sample_idxs",
                 "target_lengths")
        state = {"sd::" + k: v.detach().numpy() for k, v in module.state_dict().items()}
        config = dict(hidden=np.array(H), steps=np.array(L), memories_dim=np.array(D), embedding=np.array(E), vocabulary=np.array(V),
                      unk_id=np.array(UNK), dropout=np.array(0.2))
        save(name, **dict(zip(names, (t.numpy() for t in inputs))), copy_logprobs=copy_lp.numpy(), target_logprobs=target_lp.numpy(),
             gru_state=gru_state.numpy(), loss=loss.numpy(), **grads, **state, **config)
        if name == "decoder_h128_l7":
            # the reference's bf16 path: the fp32 module under torch.autocast("cpu", bfloat16), and in fp32, on the same bf16-rounded memories
            memories, origin, initial_states, tokens = inputs[:4]
            mb = memories.to(torch.bfloat16).float()
            with torch.no_grad():
                c32, t32, _ = module._compute_logprobs(initial_states, mb, origin, tokens[:, :-1])
                with torch.autocast("cpu", dtype=torch.bfloat16):
                    cac, tac, _ = module._compute_logprobs(initial_states, mb, origin, tokens[:, :-1])
            gap = (cac.float() - c32).abs()
            print(f"decoder_h128_l7_bf16ac: autocast dtypes {cac.dtype} / {tac.dtype}; copy logprobs autocast vs fp32 max {gap.max():.3e}")
            save("decoder_h128_l7_bf16ac", memories=mb.numpy(), origin=origin.numpy(), initial_states=initial_states.numpy(),
                 target_token_ids=tokens.numpy(), copy_autocast=cac.float().numpy(), target_autocast=tac.float().numpy(),
                 copy_fp32_rounded_inputs=c32.numpy(), target_fp32_rounded_inputs=t32.numpy(), **state, **config)


if __name__ == "__main__":
    main()
