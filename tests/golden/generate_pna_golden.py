"""Generates the PnaMessageAggregation fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_pna_golden.py          # writes tests/golden/pna_*.npz

The reference's ``PnaMessageAggregation`` is imported read-only through ``oracle/refimport.py`` (its ``torch_scatter`` calls run on the
CPU stub).  Every forward fixture stores the seeded messages, their unsorted targets, the target count, ``delta`` and the reference's
output, and the winning edge ids of max and min that the reference's ``torch_scatter`` (here the stub) returns with them.  The
targets include targets without messages (a run of them too), one-message targets, a hub of several hundred messages,
a target whose messages are nearly equal (the std's cancellation), exactly tied maxima and minima, and one NaN message element.

``pna_grad_d8`` also stores the reference's autograd gradient for a seeded ``d_out``.  The stub's max / min keep torch_scatter's arg
routing under autograd on their sequential path (at most 4,096 elements), and a tie would split the gradient there differently from
torch_scatter, so this fixture has 480 x 8 elements, no ties and no NaN.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
import torch_scatter  # noqa: E402  (the stub the reference imports)
from ptgnn.neuralmodels.gnn.messagepassing.pna_aggregation import PnaMessageAggregation  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

# name -> (D, delta, bf16 messages)
CASES = {
    "pna_d8_delta1": (8, 1.0, False),
    "pna_d8_delta2.3": (8, 2.3, False),
    "pna_d64_delta1": (64, 1.0, False),
    "pna_d64_delta2.3": (64, 2.3, False),
    "pna_d128_delta1": (128, 1.0, False),
    "pna_d128_delta2.3": (128, 2.3, False),
    "pna_d256_delta1": (256, 1.0, False),
    "pna_d256_delta2.3": (256, 2.3, False),
    "pna_d128_bf16": (128, 2.3, True),
}
HUB, TIED, FLAT = 6, 7, 9     # target ids: the hub, the target with tied rows, the nearly constant one


def degrees(gen):
    counts = [0, 1, 3, 0, 0, 0, 300, 7, 1, 12, 2, 16, 17, 0, 33, 1]
    return counts + torch.randint(0, 9, (16,), generator=gen).tolist()


def targets_for(counts, gen):
    t = torch.cat([torch.full((c,), v, dtype=torch.int64) for v, c in enumerate(counts)])
    return t[torch.randperm(t.numel(), generator=gen)]


def messages_for(targets, D, gen, nan=True):
    m = torch.randn(targets.numel(), D, generator=gen) * 1.5 + 0.3
    flat = (targets == FLAT).nonzero().flatten()
    m[flat] = 2.0 + 1e-4 * torch.randn(flat.numel(), D, generator=gen)
    tied = (targets == TIED).nonzero().flatten()
    m[tied[3]] = m[tied[1]]           # rows 1 and 3 of the target equal: every column's max / min tie if row 1 wins
    m[tied[5]] = m[tied[1]]
    if nan:
        hub = (targets == HUB).nonzero().flatten()
        m[hub[10], D // 2] = float("nan")
    return m


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def main():
    for i, (name, (D, delta, bf16)) in enumerate(CASES.items()):
        gen = torch.Generator().manual_seed(9100 + i)
        counts = degrees(gen)
        targets = targets_for(counts, gen)
        m = messages_for(targets, D, gen)
        if bf16:
            m = m.to(torch.bfloat16)
        out = PnaMessageAggregation(delta=delta)(m, targets, len(counts))
        assert out.dtype == torch.float32
        arg_max = torch_scatter.scatter_max(m.float(), targets, dim=0, dim_size=len(counts))[1]
        arg_min = torch_scatter.scatter_min(m.float(), targets, dim=0, dim_size=len(counts))[1]
        save(name, messages=m.float().numpy(), targets=targets.numpy(), num_nodes=len(counts), delta=delta, bf16=bf16, out=out.numpy(),
             arg_max=arg_max.int().numpy(), arg_min=arg_min.int().numpy())
    # gradients: 480 messages x 8 columns, no ties, no NaN
    gen = torch.Generator().manual_seed(9200)
    counts = [0, 1, 2, 0, 1, 120, 17, 16, 33, 3, 1, 0] + [5] * 52 + [2] * 13
    targets = targets_for(counts, gen)
    D, delta = 8, 2.3
    m = messages_for(targets, D, gen, nan=False)
    m[(targets == TIED).nonzero().flatten()] += 1e-3 * torch.randn(counts[TIED], D, generator=gen)    # untie
    assert targets.numel() == 480
    x = m.clone().requires_grad_(True)
    out = PnaMessageAggregation(delta=delta)(x, targets, len(counts))
    d_out = torch.randn(out.shape, generator=gen)
    out.backward(d_out)
    save("pna_grad_d8", messages=m.numpy(), targets=targets.numpy(), num_nodes=len(counts), delta=delta, bf16=False,
         out=out.detach().numpy(), d_out=d_out.numpy(), d_messages=x.grad.numpy())


if __name__ == "__main__":
    main()
