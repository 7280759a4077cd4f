"""Generates the node-embedder fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_embedding_golden.py          # writes tests/golden/embed_*.npz

The reference's ``TokenUnitEmbedder`` and ``SubtokenUnitEmbedder`` (``neuralmodels/embeddings/strelementrepresentationmodel.py``) are
imported read-only through ``oracle/refimport.py``.  Each fixture stores the seeded ids and lengths, the module's ``state_dict`` (keys
prefixed ``sd::``), the eval-mode output, an upstream gradient ``grad_out`` and the autograd gradients of ``(out * grad_out).sum()``
w.r.t. every parameter (``grad::<name>``).

The ids are Zipf-like over the first 35 of 50 tokens, so 15 tokens never occur and token 0 occurs more than 2 * 32 times; row 0 has
length 1, row 1 and others the full length, and every padding slot holds a non-zero in-range id (a kernel that ignores ``lengths``
fails).  ``embed_sub_mean_dense_d64_bf16ac`` is the same module under ``torch.autocast("cpu", bfloat16)``.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.embeddings.strelementrepresentationmodel import SubtokenUnitEmbedder, TokenUnitEmbedder  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
B, S, V, USED = 160, 5, 50, 35

# name -> (kind or None for token mode, use_dense_output, D)
CASES = {
    "embed_token_d128": (None, False, 128),
    "embed_token_d63": (None, False, 63),
    "embed_sub_sum_dense_d64": ("sum", True, 64),
    "embed_sub_mean_dense_d64": ("mean", True, 64),
    "embed_sub_max_dense_d64": ("max", True, 64),
    "embed_sub_sum_d64": ("sum", False, 64),
    "embed_sub_mean_d64": ("mean", False, 64),
    "embed_sub_max_d64": ("max", False, 64),
    "embed_sub_mean_dense_d128": ("mean", True, 128),
    "embed_sub_sum_d63": ("sum", False, 63),
    "embed_sub_max_d63": ("max", False, 63),
}


def zipf_ids(shape, gen):
    p = 1.0 / torch.arange(1, USED + 1, dtype=torch.float64)
    return torch.multinomial(p / p.sum(), int(np.prod(shape)), replacement=True, generator=gen).reshape(shape)


def make_inputs(token_mode, gen):
    if token_mode:
        ids = zipf_ids((B,), gen)
        ids[::2] = 0                                                         # token 0 fills more than two chunks of the backward
        return ids, None
    ids = zipf_ids((B, S), gen)
    lengths = torch.randint(1, S + 1, (B,), generator=gen)
    lengths[0], lengths[1] = 1, S
    pad = torch.arange(S)[None, :] >= lengths[:, None]
    ids[pad] = torch.randint(1, USED, (int(pad.sum()),), generator=gen)      # non-zero, in range, never to be read
    return ids, lengths


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items() if v is not None})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def main():
    for i, (name, (kind, dense, D)) in enumerate(CASES.items()):
        torch.manual_seed(9000 + i)
        module = TokenUnitEmbedder(V, D, 0.2) if kind is None else SubtokenUnitEmbedder(V, D, 0.2, kind, use_dense_output=dense)
        module.eval()
        gen = torch.Generator().manual_seed(9500 + i)
        ids, lengths = make_inputs(kind is None, gen)
        args = (ids,) if kind is None else (ids, lengths)
        grad_out = torch.randn(B, D, generator=gen)
        out = module(*args)
        (out * grad_out).sum().backward()
        grads = {"grad::" + n: p.grad.numpy() for n, p in module.named_parameters()}
        assert all(np.isfinite(g).all() for g in grads.values()), f"{name}: non-finite gradient"
        state = {"sd::" + k: v.detach().numpy() for k, v in module.state_dict().items()}
        config = dict(kind=np.array(kind or "token"), dense=np.array(dense), vocabulary=np.array(V), dim=np.array(D))
        save(name, token_idxs=ids.numpy(), lengths=None if lengths is None else lengths.numpy(), out=out.detach().numpy(),
             grad_out=grad_out.numpy(), **grads, **state, **config)
        if name == "embed_sub_mean_dense_d64":
            with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16):
                out_ac = module(*args)
            print(f"{name}_bf16ac: autocast dtype {out_ac.dtype}; autocast vs fp32 max {(out_ac.float() - out).abs().max():.3e}")
            save(name + "_bf16ac", token_idxs=ids.numpy(), lengths=lengths.numpy(), out_autocast=out_ac.float().numpy(),
                 out_fp32=out.detach().numpy(), **state, **config)


if __name__ == "__main__":
    main()
