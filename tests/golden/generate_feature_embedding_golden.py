"""Generates the feature-embedder fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_feature_embedding_golden.py       # writes tests/golden/feature_embed_*.npz

The reference's ``LinearFeatureEmbedder`` (``neuralmodels/embeddings/linearmapembedding.py:13-29``) is imported read-only through
``oracle/refimport.py`` (pure torch: no ``torch_scatter`` is needed) and run on the CPU in fp32.

* ``feature_embed_f{F}`` for F in {1, 50, 121}: seeded features ``x`` [29, F]; for D in {8, 64, 256} the weight of a module built under
  ``torch.manual_seed`` (``w_d{D}``, the reference's ``_LinearFeatureEmbedder__linear_map.weight``) and, for each activation (none, relu,
  tanh, gelu), the module's output ``out_d{D}_{act}``.  At D = 64, an upstream gradient ``grad_out_{act}`` and the autograd gradients of
  ``(out * grad_out).sum()`` w.r.t. the weight (``grad_w_{act}``) and the features (``grad_x_{act}``).
* ``feature_embed_bf16ac``: F = 50, D = 64 (PPI's shape), each activation under ``torch.autocast("cpu", bfloat16)`` (``out_{act}``).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.embeddings.linearmapembedding import LinearFeatureEmbedder  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
ROWS = 29
ACTIVATIONS = {"none": lambda: None, "relu": torch.nn.ReLU, "tanh": torch.nn.Tanh, "gelu": torch.nn.GELU}
KEY = "_LinearFeatureEmbedder__linear_map.weight"


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def module(F, D, act, seed):
    torch.manual_seed(seed)
    return LinearFeatureEmbedder(F, D, ACTIVATIONS[act]())


def feature_fixture(F):
    gen = torch.Generator().manual_seed(8000 + F)
    x = torch.randn(ROWS, F, generator=gen)
    arrays = {"x": x.numpy()}
    for D in (8, 64, 256):
        seed = 8100 + F * 7 + D
        arrays[f"w_d{D}"] = module(F, D, "none", seed).state_dict()[KEY].numpy()
        for act in ACTIVATIONS:
            m = module(F, D, act, seed)
            assert torch.equal(m.state_dict()[KEY], torch.from_numpy(arrays[f"w_d{D}"])), "same seed, same weight"
            if D != 64:
                with torch.no_grad():
                    arrays[f"out_d{D}_{act}"] = m(x).numpy()
                continue
            xg = x.clone().requires_grad_(True)
            out = m(xg)
            grad_out = torch.randn(ROWS, D, generator=gen)
            (out * grad_out).sum().backward()
            arrays[f"out_d{D}_{act}"] = out.detach().numpy()
            arrays[f"grad_out_{act}"] = grad_out.numpy()
            arrays[f"grad_w_{act}"] = dict(m.named_parameters())[KEY].grad.numpy()
            arrays[f"grad_x_{act}"] = xg.grad.numpy()
    save(f"feature_embed_f{F}", **arrays)


def bf16_fixture():
    F, D = 50, 64
    gen = torch.Generator().manual_seed(8900)
    x = torch.randn(ROWS, F, generator=gen)
    arrays = {"x": x.numpy()}
    for act in ACTIVATIONS:
        m = module(F, D, act, 8950)
        arrays["w"] = m.state_dict()[KEY].numpy()
        with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16):
            out = m(x)
        assert out.dtype == torch.bfloat16
        arrays[f"out_{act}"] = out.float().numpy()
    save("feature_embed_bf16ac", **arrays)


def main():
    for F in (1, 50, 121):
        feature_fixture(F)
    bf16_fixture()


if __name__ == "__main__":
    main()
