"""Generates the char-embedder fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_char_embedding_golden.py          # writes tests/golden/char_*.npz

The reference's ``CharUnitEmbedder`` (``neuralmodels/embeddings/strelementrepresentationmodel.py:100-142``) is imported read-only through
``oracle/refimport.py`` and run on the CPU in fp32.  Each fixture stores the configuration, the seeded ids, the module's parameters
(``sd::<key>``, the reference's mangled ``state_dict`` keys) and eval-mode outputs.

* ``char_default``: the default ``CnnConfig(256, 3, 128, 3, 3)`` at C = 101, L = 15, one module seeded at D = 128; the outputs at
  D = 63 and D = 127 (``out_d63``, ``out_d127``) are the reference module of that size with the same W1, b1, W2, b2 and the first D rows
  of W3.  ``out_minl``: the first 7 characters of every token (the minimal L: one output position).  ``out_bf16ac_d127``: the D = 127
  module under ``torch.autocast("cpu", bfloat16)``.
* ``char_cfg_a``: ``CnnConfig(64, 1, 256, 5, 2)``, C = 40, L = 12, D = 63.
* ``char_cfg_b``: ``CnnConfig(128, 2, 64, 4, 5)``, C = 101, L = 20, D = 100, with an upstream gradient ``grad_out`` and the autograd
  gradients of ``(out * grad_out).sum()`` w.r.t. all five parameters (``grad::<key>``); its max has no ties (checked here).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.embeddings.strelementrepresentationmodel import CharUnitEmbedder, CnnConfig  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
B = 96
PRE = "_CharUnitEmbedder__"


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def state(module):
    return {"sd::" + k: v.detach().numpy() for k, v in module.state_dict().items()}


def config_arrays(C, cfg, D, L):
    return dict(num_chars=np.array(C), cnn=np.array(list(cfg)), dim=np.array(D), max_chars=np.array(L))


def default_fixture():
    C, L, cfg = 101, 15, CnnConfig(256, 3, 128, 3, 3)
    torch.manual_seed(7100)
    big = CharUnitEmbedder(C, 128, cfg, 0.2).eval()
    gen = torch.Generator().manual_seed(7150)
    chars = torch.randint(0, C, (B, L), generator=gen)
    outs = {}
    with torch.no_grad():
        outs["out_d128"] = big(chars).numpy()
        outs["out_minl"] = big(chars[:, :7].contiguous()).numpy()
        for D in (63, 127):
            m = CharUnitEmbedder(C, D, cfg, 0.2).eval()
            sd = {k: (v[:D] if k.endswith("conv_l3.weight") else v) for k, v in big.state_dict().items()}
            m.load_state_dict(sd, strict=True)
            outs[f"out_d{D}"] = m(chars).numpy()
            if D == 127:
                with torch.autocast("cpu", dtype=torch.bfloat16):
                    ac = m(chars)
                print(f"char_default bf16 autocast: dtype {ac.dtype}, max |autocast - fp32| {(ac.float() - m(chars)).abs().max():.3e}")
                outs["out_bf16ac_d127"] = ac.float().numpy()
    save("char_default", chars=chars.numpy(), **outs, **state(big), **config_arrays(C, cfg, 128, L))


def config_fixture(name, C, cfg, D, L, seed, with_grad):
    torch.manual_seed(seed)
    m = CharUnitEmbedder(C, D, cfg, 0.2).eval()
    gen = torch.Generator().manual_seed(seed + 50)
    chars = torch.randint(0, C, (B, L), generator=gen)
    extra = {}
    if with_grad:
        out = m(chars)
        grad_out = torch.randn(B, D, generator=gen)
        (out * grad_out).sum().backward()
        extra["grad_out"] = grad_out.numpy()
        extra.update({"grad::" + k: p.grad.numpy() for k, p in m.named_parameters()})
        with torch.no_grad():      # no ties in the max: the backward's routing is then unique
            l1 = m._CharUnitEmbedder__conv_l1(torch.nn.functional.one_hot(chars, C).transpose(1, 2).float())
            l3 = m._CharUnitEmbedder__conv_l3(torch.relu(m._CharUnitEmbedder__conv_l2(torch.relu(l1))))
            top2 = l3.topk(2, dim=-1).values
            assert bool((top2[..., 0] > top2[..., 1]).all()), f"{name}: a tie in the max"
    else:
        with torch.no_grad():
            out = m(chars)
    save(name, chars=chars.numpy(), out=out.detach().numpy(), **extra, **state(m), **config_arrays(C, cfg, D, L))


def main():
    default_fixture()
    config_fixture("char_cfg_a", 40, CnnConfig(64, 1, 256, 5, 2), 63, 12, 7200, False)
    config_fixture("char_cfg_b", 101, CnnConfig(128, 2, 64, 4, 5), 100, 20, 7300, True)


if __name__ == "__main__":
    main()
