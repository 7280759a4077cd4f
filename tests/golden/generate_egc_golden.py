"""Generates the EGCMessagePassingLayer fixtures of the fused path by running the UNMODIFIED reference class.

    python tests/golden/generate_egc_golden.py      # writes tests/golden/egc_grad_*.npz, egc_*_bf16ac.npz

The reference is imported read-only through ``oracle/refimport.py``, as in ``generate_golden.py``.

* ``egc_grad_{sum,mean,max,min}``: a shape the fused kernel takes (H = out = 64, 8 heads, 4 bases, T = 3 with an empty type, and
  targets without in-edges); the fp32 output and the autograd gradients of ``h``, every ``bases[t].weight`` and ``weight_coeffs``'
  weight and bias for a seeded ``d out``.  Each (source, target, type) edge occurs once and the states are random: no two messages
  of one target tie, so the max / min routing of the reference's scatter is unambiguous.
* ``egc_{sum,max}_bf16ac``: the reference under CPU autocast bf16 next to its fp32 output on the same bf16-rounded states.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.gnn.messagepassing.egcmessagepassing import EGCMessagePassingLayer  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from generate_golden import pack, run_layer, save, state  # noqa: E402


def unique_graph(gen, n_tgt, n_src, counts):
    """Per type: `count` distinct (source, target) pairs, targets in [0, n_tgt) (nodes >= n_tgt receive nothing)."""
    adj = []
    for c in counts:
        if c == 0:
            adj.append((torch.zeros(0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64)))
            continue
        keys = torch.randperm(n_src * n_tgt, generator=gen)[:c]
        adj.append((keys // n_tgt, keys % n_tgt))
    return adj


def main():
    for i, agg in enumerate(["sum", "mean", "max", "min"]):
        gen = torch.Generator().manual_seed(1100 + i)
        torch.manual_seed(1200 + i)
        n, H, out, heads, bases, counts = 320, 64, 64, 8, 4, [1400, 0, 900]
        adj = unique_graph(gen, n - 24, n, counts)
        layer = EGCMessagePassingLayer(H, out, len(counts), agg, num_bases=bases, num_heads=heads).eval()
        h = torch.randn(n, H, generator=gen).requires_grad_(True)
        d_out = torch.randn(n, out, generator=gen)
        feats = [torch.empty(a[0].shape[0], 0) for a in adj]
        y = layer(node_states=h, adjacency_lists=adj, node_to_graph_idx=torch.zeros(n, dtype=torch.int64), reference_node_ids={},
                  reference_node_graph_idx={}, edge_features=feats)
        params = dict(layer.named_parameters())
        names = sorted(params)
        grads = torch.autograd.grad(y, [h] + [params[k] for k in names], d_out)
        save(f"egc_grad_{agg}", h=h.detach().numpy(), out=y.detach().numpy(), d_out=d_out.numpy(), d_h=grads[0].numpy(),
             agg=agg, heads=heads, bases=bases, **{"grad::" + k: g.numpy() for k, g in zip(names, grads[1:])}, **pack("", adj),
             **state(layer))

    for i, agg in enumerate(["sum", "max"]):
        gen = torch.Generator().manual_seed(1300 + i)
        torch.manual_seed(1400 + i)
        n, H, counts = 384, 64, [900, 0, 500, 260]
        adj = unique_graph(gen, n - 16, n, counts)
        layer = EGCMessagePassingLayer(H, H, len(counts), agg, num_bases=4, num_heads=8)
        h = torch.randn(n, H, generator=gen)
        out32 = run_layer(layer, h, adj)
        hb = h.to(torch.bfloat16)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            out_ac = run_layer(layer, hb, adj)
        out32_on_rounded = run_layer(layer, hb.float(), adj)
        gap = (out_ac.float() - out32_on_rounded).abs()
        print(f"egc_{agg}_bf16ac: autocast output dtype {out_ac.dtype}; autocast vs fp32 (same rounded inputs): max {gap.max():.3e} "
              f"mean {gap.mean():.3e}")
        save(f"egc_{agg}_bf16ac", h=h.numpy(), out_autocast=out_ac.float().numpy(), out_fp32=out32.numpy(),
             out_fp32_rounded_inputs=out32_on_rounded.numpy(), agg=agg, **pack("", adj), **state(layer))


if __name__ == "__main__":
    main()
