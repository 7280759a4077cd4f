"""One training step of the gated stacks of the reference's Typilus and VarMisuse training scripts with per-edge dropout, at the
config-2 batch: the three-kernel dropout path (the layers' own routing at these widths) against ``autograd.gated_forward_composed``
(the gathered rows, torch's dropout mask, per-type Linear, segmented reduce), which the layers take when the native dropout paths are
switched off for the run, alternating the two in the same process.

  typilus:   7 x GatedMessagePassingLayer(H = D = 64, max, p = 0.1), ConcatResidualLayer, GatedMessagePassingLayer(H = 128, D = 64)
  varmisuse: GatedMessagePassingLayer(H = D = 64, sum, p = 0.01) x 2, GruGlobalStateUpdate, the same layer again

Reports forward time, backward time and peak memory per stack and path, with the card's name and power limit.  Writes nothing;
prints one JSON line."""
import json
import os
import subprocess
import sys
from unittest import mock

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200.synthetic import graph2class_batch  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 5


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as exc:   # the numbers are still reported, with what was not read
        return f"{torch.cuda.get_device_name()} (power limit not read: {exc})"


def typilus(T):
    mp = P.GatedMessagePassingLayer(64, 64, T, "max", dropout_rate=0.1)
    r = P.ConcatResidualLayer(64)
    return [r.pass_through_dummy_layer()] + [mp] * 7 + [r, P.GatedMessagePassingLayer(128, 64, T, "max", dropout_rate=0.1)]


def varmisuse(T):
    mp = P.GatedMessagePassingLayer(64, 64, T, "sum", dropout_rate=0.01)
    return [mp, mp, P.GruGlobalStateUpdate(P.WeightedSumVarSizedElementReduce(64), 64, 64, dropout_rate=0.1), mp]


b = graph2class_batch()
n2g = b.node_to_graph_idx.cuda()
T = 2 * len(b.adjacency_lists) + 1            # with the backward and self edges the container adds
stacks = {}
for name, make in (("typilus", typilus), ("varmisuse", varmisuse)):
    torch.manual_seed(0)
    stacks[name] = P.GraphNeuralNetwork(make(T), torch.nn.Identity(), True, True).cuda().train()
adj = stacks["typilus"].expand_adjacency([(s.cuda(), t.cuda()) for s, t in b.adjacency_lists], b.num_nodes, "cuda")
h0 = torch.randn(b.num_nodes, 64).cuda()


def step(gnn, composed):
    for q in gnn.parameters():
        q.grad = None
    h = h0.clone().requires_grad_(True)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with mock.patch("ptgnn_b200.messagepassing._native_dropout", lambda lib, H, D: not composed):
        ev[0].record()
        loss = gnn.gnn(h, adj, None, n2g, {}, {}).mean()
        ev[1].record()
        loss.backward()
        ev[2].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), (torch.cuda.max_memory_allocated() - base) / 2**20


def median(xs):
    return sorted(xs)[len(xs) // 2]


out = {"card": card(), "nodes": b.num_nodes, "edges": sum(int(s.shape[0]) for s, _ in adj), "reps": REPS}
for name, gnn in stacks.items():
    paths = {"three_kernel": False, "composed": True}
    for c in paths.values():        # warm-up: module loads, plan build, library algorithm choice
        step(gnn, c)
        step(gnn, c)
    res = {k: [] for k in paths}
    for _ in range(REPS):
        for k, c in paths.items():
            res[k].append(step(gnn, c))
    out[name] = {k: {"forward_ms": round(median([r[0] for r in rows]), 3), "backward_ms": round(median([r[1] for r in rows]), 3),
                     "peak_mib_above_inputs": round(max(r[2] for r in rows), 1)} for k, rows in res.items()}
print(json.dumps(out))
