"""Generates the GraphNorm fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_graphnorm_golden.py          # writes tests/golden/graphnorm_*.npz

The reference's ``GraphNorm`` is imported read-only through ``oracle/refimport.py`` (it runs on the CPU through the ``torch_scatter``
stub, whose ``scatter_mean`` is differentiable).  Every fixture stores the seeded inputs, the module's ``state_dict`` (keys prefixed
``sd::``; gamma, alpha and bias are set away from their defaults 1, 1, 0, where alpha and bias mistakes would not show), the
reference's output, and its autograd gradients for a seeded ``dy``.  Every node -> graph map is unsorted and has a graph id without
nodes, one-node graphs and a graph of several 32-row chunks.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.gnn.messagepassing.graphnorm import GraphNorm  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

# name -> (D, node counts per graph id (0 = a graph id without nodes))
CASES = {
    "graphnorm_d32": (32, [1, 33, 0, 100, 1, 7, 64]),
    "graphnorm_d64": (64, [5, 1, 0, 97, 32, 1]),
    "graphnorm_d128": (128, [70, 1, 1, 0, 31, 129]),
    "graphnorm_d256": (256, [1, 0, 65, 3, 40]),
}


def node_to_graph(counts, gen):
    n2g = torch.cat([torch.full((c,), g, dtype=torch.int64) for g, c in enumerate(counts)])
    return n2g[torch.randperm(n2g.numel(), generator=gen)]


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def run(module, x, n2g, dy):
    module.zero_grad()
    x = x.clone().requires_grad_(True)
    out = module(x, [], n2g, {}, {}, [])
    out.backward(dy)
    grads = {"d_x": x.grad.numpy(), **{"d_" + n: p.grad.numpy() for n, p in module.named_parameters()}}
    return out.detach(), grads


def main():
    for i, (name, (D, counts)) in enumerate(CASES.items()):
        torch.manual_seed(7000 + i)
        gen = torch.Generator().manual_seed(8000 + i)
        module = GraphNorm(D)
        with torch.no_grad():
            module.gamma.copy_(1.0 + 0.5 * torch.randn(1, D, generator=gen))
            module.alpha.copy_(torch.rand(1, D, generator=gen) * 1.5)
            module.bias.copy_(0.3 * torch.randn(1, D, generator=gen))
        n2g = node_to_graph(counts, gen)
        G = len(counts)
        x = torch.randn(n2g.numel(), D, generator=gen) * 2.0 + torch.randn(G, D, generator=gen)[n2g]
        dy = torch.randn(n2g.numel(), D, generator=gen)
        out, grads = run(module, x, n2g, dy)
        state = {"sd::" + k: v.detach().numpy() for k, v in module.state_dict().items()}
        save(name, x=x.numpy(), n2g=n2g.numpy(), dy=dy.numpy(), out=out.numpy(), **grads, **state)
        if name == "graphnorm_d128":
            # the reference fed bf16 states, and in fp32 on the same bf16-rounded states
            xb = x.to(torch.bfloat16)
            with torch.no_grad():
                out_bf16 = module(xb, [], n2g, {}, {}, [])
                out32 = module(xb.float(), [], n2g, {}, {}, [])
            gap = (out_bf16.float() - out32).abs()
            print(f"graphnorm_d128_bf16: output dtype {out_bf16.dtype}; bf16 vs fp32: max {gap.max():.3e} mean {gap.mean():.3e}")
            save("graphnorm_d128_bf16", x=xb.float().numpy(), n2g=n2g.numpy(), out_bf16=out_bf16.float().numpy(),
                 out_fp32_rounded_inputs=out32.numpy(), **state)


if __name__ == "__main__":
    main()
