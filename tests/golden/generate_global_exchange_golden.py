"""Generates the GruGlobalStateUpdate fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_global_exchange_golden.py          # writes tests/golden/global_*.npz

Like ``generate_golden.py``: the reference's ``GruGlobalStateUpdate`` and its reducers are imported read-only through
``oracle/refimport.py``; every fixture stores the seeded inputs, the reference module's ``state_dict``, the reference's readout
``g`` and the layer's output.  The node -> graph map is unsorted, has a gap (graph 3 has no node) and two 1-node graphs.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.gnn.messagepassing.globalgraphexchange import GruGlobalStateUpdate  # noqa: E402
from ptgnn.neuralmodels.reduceops.varsizedsummary import (  # noqa: E402
    ElementsToSummaryRepresentationInput,
    SimpleVarSizedElementReduce,
    WeightedSumVarSizedElementReduce,
)

OUT = os.path.dirname(os.path.abspath(__file__))
N, H = 100, 64


def node_to_graph(gen):
    """Graphs 0 and 5 have one node each, graph 3 none; the others share the rest; the order is shuffled."""
    ids = torch.tensor([0, 5] + [(1, 2, 4, 6)[i % 4] for i in range(N - 2)], dtype=torch.int64)
    return ids[torch.randperm(N, generator=gen)]


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def main():
    cases = [("weighted", None), ("simple", "sum"), ("simple", "mean"), ("simple", "max")]
    for i, (reducer_kind, agg) in enumerate(cases):
        torch.manual_seed(1000 + i)
        gen = torch.Generator().manual_seed(2000 + i)
        reducer = WeightedSumVarSizedElementReduce(H) if reducer_kind == "weighted" else SimpleVarSizedElementReduce(agg)
        layer = GruGlobalStateUpdate(reducer, input_state_size=H, summarized_state_size=H).eval()
        h = torch.randn(N, H, generator=gen)
        n2g = node_to_graph(gen)
        with torch.no_grad():
            g = reducer(ElementsToSummaryRepresentationInput(h, n2g, n2g.max() + 1))
            out = layer(h, [], n2g, {}, {}, [])
        kind = "weighted" if reducer_kind == "weighted" else agg
        state = {"sd::" + k: v.detach().numpy() for k, v in layer.state_dict().items()}
        save(f"global_{kind}", h=h.numpy(), n2g=n2g.numpy(), g=g.numpy(), out=out.numpy(), kind=np.array(kind), **state)
        if kind == "weighted":
            # the reference's bf16 path: fp32 module under torch.autocast("cpu", bfloat16), and in fp32, on the same bf16-rounded states
            hb = h.to(torch.bfloat16).float()
            with torch.no_grad():
                out32 = layer(hb, [], n2g, {}, {}, [])
                with torch.autocast("cpu", dtype=torch.bfloat16):
                    out_ac = layer(hb, [], n2g, {}, {}, [])
            gap = (out_ac.float() - out32).abs()
            print(f"global_weighted_bf16ac: autocast output dtype {out_ac.dtype}; autocast vs fp32: max {gap.max():.3e} mean {gap.mean():.3e}, "
                  f"within 1e-2: {(gap <= 1e-2 * out32.abs().clamp(min=1)).float().mean():.4f}")
            save("global_weighted_bf16ac", h=hb.numpy(), n2g=n2g.numpy(), out_autocast=out_ac.float().numpy(),
                 out_fp32_rounded_inputs=out32.numpy(), kind=np.array(kind), **state)


if __name__ == "__main__":
    main()
