"""Times the native VarMisuse head (DESIGN.md §3.16) against the reference's torch formulation, forward plus backward, with CUDA events.

    python tools/heads_time.py [--iters 200] [--json OUT]

The shape is a VarMisuse training minibatch of the reference's defaults (implementations/varmisuse/train.py: H = 64, 300 samples per
minibatch, up to 80000 nodes): N = 80000 node states, 300 slots with 2 to 20 candidates each.  The torch formulation is the reference's
head written with differentiable library ops (index, cat, Linear, a per-slot log-softmax from scatter_reduce / scatter_add, the NLL
mean); the native one is ``ptgnn_b200.VarMisuseGraphModel``'s head.  Both start from the same fp32 node states and weight, and both
include the loss's backward into d h and d w.  Prints the card name and power limit with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from ptgnn_b200 import autograd as AG  # noqa: E402
from ptgnn_b200 import heads as HD  # noqa: E402
from ptgnn_b200.edgeplan import EdgePlan  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name()
    return out.splitlines()[0] if out else torch.cuda.get_device_name()


def inputs(num_nodes=80000, H=64, slots=300, seed=0):
    gen = torch.Generator().manual_seed(seed)
    sizes = torch.randint(2, 21, (slots,), generator=gen)
    slot_of = torch.repeat_interleave(torch.arange(slots), sizes)
    cand = torch.randint(0, num_nodes, (slot_of.shape[0],), generator=gen)
    slot_nodes = torch.randint(0, num_nodes, (slots,), generator=gen)
    starts = torch.cumsum(sizes, 0) - sizes
    correct = starts + (torch.rand(slots, generator=gen) * sizes).long()
    h = torch.randn(num_nodes, H, generator=gen)
    w = torch.randn(1, 2 * H, generator=gen) / H ** 0.5
    return [t.cuda() for t in (h, cand, slot_of, slot_nodes, correct, w)]


def torch_head(h, cand, slot_of, slot_nodes, correct, w):
    J = slot_nodes.shape[0]
    score = torch.nn.functional.linear(torch.cat((h[cand], h[slot_nodes][slot_of]), dim=-1), w).squeeze(-1)
    mx = torch.full((J,), -torch.inf, device=h.device).scatter_reduce(0, slot_of, score, "amax")
    centred = score - mx[slot_of]
    lse = torch.zeros(J, device=h.device).scatter_add(0, slot_of, centred.exp()).log()
    return -(centred - lse[slot_of])[correct].mean()


def native_head(h, cand, slot_of, slot_nodes, correct, w, hits):
    ops = HD.varmisuse_inputs(h, cand, slot_of, slot_nodes, correct, w)
    return AG.varmisuse_with_grad(ops, hits, h, w)


def time_step(fn, h, w, iters):
    for _ in range(10):
        h.grad = w.grad = None
        fn().backward()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        h.grad = w.grad = None
        fn().backward()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters * 1000.0


def time_forward(fn, iters):
    for _ in range(10):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters * 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "heads_time.py measures on the GPU"
    h, cand, slot_of, slot_nodes, correct, w = inputs()
    h.requires_grad_(True)
    w.requires_grad_(True)
    hits = torch.zeros(1, dtype=torch.int64, device="cuda")
    ref = lambda: torch_head(h, cand, slot_of, slot_nodes, correct, w)          # noqa: E731
    nat = lambda: native_head(h, cand, slot_of, slot_nodes, correct, w, hits)   # noqa: E731
    node_ids = torch.cat([cand, slot_nodes])
    node_plan = lambda: EdgePlan([(node_ids, node_ids)], h.shape[0]).perm      # noqa: E731  (the plan the native backward builds)
    rows, fwd = {}, {}
    for rep in range(3):                 # alternate the two, three times: the spread shows in the repeats
        rows.setdefault("torch_us", []).append(time_step(ref, h, w, args.iters))
        rows.setdefault("native_us", []).append(time_step(nat, h, w, args.iters))
        with torch.no_grad():            # the forward alone, so that the backward's share shows
            fwd.setdefault("torch_us", []).append(time_forward(ref, args.iters))
            fwd.setdefault("native_us", []).append(time_forward(nat, args.iters))
            fwd.setdefault("native_backward_node_plan_us", []).append(time_forward(node_plan, args.iters))
    result = {"card": card(), "shape": {"N": h.shape[0], "H": h.shape[1], "slots": slot_nodes.shape[0], "candidates": cand.shape[0]},
              "forward_backward_us": {k: [round(v, 1) for v in vs] for k, vs in rows.items()},
              "forward_us": {k: [round(v, 1) for v in vs] for k, vs in fwd.items()}}
    print(json.dumps(result))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
