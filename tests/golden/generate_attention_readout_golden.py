"""Generates the attention-reducer fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_attention_readout_golden.py          # writes tests/golden/attn_*.npz

Like ``generate_global_exchange_golden.py``: the reference's ``SelfAttentionVarSizedElementReduce`` and
``MultiheadSelfAttentionVarSizedElementReduce`` are imported read-only through ``oracle/refimport.py``; every fixture stores the
seeded inputs, the module's ``state_dict`` (keys prefixed ``sd::``), its configuration and the reference's output.  The node -> graph
map is the global-exchange fixtures': unsorted, with a gap (graph 3 has no node) and two 1-node graphs.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from generate_global_exchange_golden import node_to_graph  # noqa: E402
from ptgnn.neuralmodels.reduceops.varsizedsummary import (  # noqa: E402
    ElementsToSummaryRepresentationInput,
    MultiheadSelfAttentionVarSizedElementReduce,
    SelfAttentionVarSizedElementReduce,
    SimpleVarSizedElementReduce,
    WeightedSumVarSizedElementReduce,
)

OUT = os.path.dirname(os.path.abspath(__file__))
N, D, HIDDEN, OUT_DIM = 100, 64, 64, 32

# name -> (class, heads, use_value_layer, query summarizer kind)
CASES = {
    "attn_mh1": ("multihead", 1, False, "max"),
    "attn_mh1_value": ("multihead", 1, True, "max"),
    "attn_mh4": ("multihead", 4, False, "mean"),
    "attn_mh4_value": ("multihead", 4, True, "max"),
    "attn_mh8": ("multihead", 8, False, "max"),
    "attn_mh8_value": ("multihead", 8, True, "sum"),
    "attn_self_weighted": ("self", 1, False, "weighted"),
}


def build(cls, heads, value, query):
    q = WeightedSumVarSizedElementReduce(D) if query == "weighted" else SimpleVarSizedElementReduce(query)
    if cls == "self":
        return SelfAttentionVarSizedElementReduce(D, HIDDEN, OUT_DIM, q)
    return MultiheadSelfAttentionVarSizedElementReduce(D, HIDDEN, OUT_DIM, heads, q, use_value_layer=value)


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def main():
    for i, (name, (cls, heads, value, query)) in enumerate(CASES.items()):
        torch.manual_seed(3000 + i)
        gen = torch.Generator().manual_seed(4000 + i)
        module = build(cls, heads, value, query).eval()
        x = torch.randn(N, D, generator=gen)
        n2g = node_to_graph(gen)
        with torch.no_grad():
            out = module(ElementsToSummaryRepresentationInput(x, n2g, n2g.max() + 1))
        state = {"sd::" + k: v.detach().numpy() for k, v in module.state_dict().items()}
        config = dict(cls=np.array(cls), heads=np.array(heads), value=np.array(value), query=np.array(query))
        save(name, x=x.numpy(), n2g=n2g.numpy(), out=out.numpy(), **config, **state)
        if name == "attn_mh8":
            # the reference's bf16 path: the fp32 module under torch.autocast("cpu", bfloat16), and in fp32, on the same bf16-rounded states
            xb = x.to(torch.bfloat16).float()
            with torch.no_grad():
                out32 = module(ElementsToSummaryRepresentationInput(xb, n2g, n2g.max() + 1))
                with torch.autocast("cpu", dtype=torch.bfloat16):
                    out_ac = module(ElementsToSummaryRepresentationInput(xb, n2g, n2g.max() + 1))
            gap = (out_ac.float() - out32).abs()
            print(f"attn_mh8_bf16ac: autocast output dtype {out_ac.dtype}; autocast vs fp32: max {gap.max():.3e} mean {gap.mean():.3e}")
            save("attn_mh8_bf16ac", x=xb.numpy(), n2g=n2g.numpy(), out_autocast=out_ac.float().numpy(), out_fp32_rounded_inputs=out32.numpy(),
                 **config, **state)


if __name__ == "__main__":
    main()
