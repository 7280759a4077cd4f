"""Generates the self-attention layer fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_selfattention_golden.py          # writes tests/golden/selfatt_*.npz

The reference's ``MultiHeadSelfAttentionMessagePassing`` is imported read-only through ``oracle/refimport.py`` (it runs on the CPU
through the ``torch_scatter`` stub); every fixture stores the seeded inputs, the module's ``state_dict`` (keys prefixed ``sd::``), its
configuration and the reference's output.  Graph sizes straddle the 64-row tiles and the chunk lengths; every node -> graph map has
a graph id without nodes, and all but one are unsorted (the reference takes each graph's rows from the counts, not from the ids).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.gnn.messagepassing.selfattmessagepassing import MultiHeadSelfAttentionMessagePassing  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
IN_DIM, OUT_DIM, INTER = 16, 16, 32

# name -> (heads, dk, dv, max_num_nodes, node counts per graph id (0 = a graph id without nodes), shuffle the map)
CASES = {
    "selfatt_h1_d16": (1, 16, 16, 250, [1, 16, 17, 0, 64, 65, 249, 250, 251], True),
    "selfatt_h3_d32": (3, 32, 32, 64, [65, 1, 0, 250, 17, 64], True),
    "selfatt_h8_d16": (8, 16, 16, 250, [2500, 0, 64, 1], False),
    "selfatt_h4_dk64_dv32": (4, 64, 32, 1000, [251, 1100, 0, 16], True),
    "selfatt_h2_dk128_dv64": (2, 128, 64, 250, [251, 249, 1, 0, 65], True),
}


def node_to_graph(counts, shuffle, gen):
    n2g = torch.cat([torch.full((c,), g, dtype=torch.int64) for g, c in enumerate(counts)])
    if shuffle:
        n2g = n2g[torch.randperm(n2g.numel(), generator=gen)]
    return n2g


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def main():
    for i, (name, (heads, dk, dv, L, counts, shuffle)) in enumerate(CASES.items()):
        torch.manual_seed(5000 + i)
        gen = torch.Generator().manual_seed(6000 + i)
        module = MultiHeadSelfAttentionMessagePassing(IN_DIM, dk, dv, OUT_DIM, INTER, heads, max_num_nodes=L).eval()
        n2g = node_to_graph(counts, shuffle, gen)
        x = torch.randn(n2g.numel(), IN_DIM, generator=gen)
        with torch.no_grad():
            out = module(x, [], n2g, {}, {}, [])
        state = {"sd::" + k: v.detach().numpy() for k, v in module.state_dict().items()}
        config = dict(heads=np.array(heads), dk=np.array(dk), dv=np.array(dv), max_num_nodes=np.array(L), in_dim=np.array(IN_DIM),
                      out_dim=np.array(OUT_DIM), inter=np.array(INTER))
        save(name, x=x.numpy(), n2g=n2g.numpy(), out=out.numpy(), **config, **state)
        if name == "selfatt_h8_d16":
            # the reference's bf16 path: the fp32 module under torch.autocast("cpu", bfloat16), and in fp32, on the same bf16-rounded states
            xb = x.to(torch.bfloat16).float()
            with torch.no_grad():
                out32 = module(xb, [], n2g, {}, {}, [])
                with torch.autocast("cpu", dtype=torch.bfloat16):
                    out_ac = module(xb, [], n2g, {}, {}, [])
            gap = (out_ac.float() - out32).abs()
            print(f"selfatt_h8_d16_bf16ac: autocast output dtype {out_ac.dtype}; autocast vs fp32: max {gap.max():.3e} mean {gap.mean():.3e}")
            save("selfatt_h8_d16_bf16ac", x=xb.numpy(), n2g=n2g.numpy(), out_autocast=out_ac.float().numpy(),
                 out_fp32_rounded_inputs=out32.numpy(), **config, **state)


if __name__ == "__main__":
    main()
