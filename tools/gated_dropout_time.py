"""One training step of 8 gated layers with per-edge dropout p = 0.1 at the config-2 batch: the fused path (the layer's own routing)
against ``autograd.gated_forward_composed`` called directly (the gathered rows, torch's dropout mask, per-type Linear, segmented
reduce), in the same process, alternating the two.  Reports forward time, backward time and peak memory per path, with the card's
name and power limit.  Writes nothing; prints one JSON line."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import autograd as A  # noqa: E402
from ptgnn_b200.synthetic import graph2class_batch  # noqa: E402

LAYERS, P_DROP, REPS = 8, 0.1, int(sys.argv[1]) if len(sys.argv) > 1 else 5


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as exc:   # the numbers are still reported, with what was not read
        return f"{torch.cuda.get_device_name()} (power limit not read: {exc})"


b = graph2class_batch()
torch.manual_seed(0)
layers = [P.GatedMessagePassingLayer(128, 128, 17, "sum", dropout_rate=P_DROP) for _ in range(LAYERS)]
gnn = P.GraphNeuralNetwork(layers, torch.nn.Identity(), True, True).cuda().train()
adj = gnn.expand_adjacency([(s.cuda(), t.cuda()) for s, t in b.adjacency_lists], b.num_nodes, "cuda")
h0 = torch.randn(b.num_nodes, 128).cuda()


def composed_forward(h):
    for layer in layers:
        lins = layer._GatedMessagePassingLayer__edge_message_transformation_layers
        h = A.gated_forward_composed([lin.weight for lin in lins], layer._GatedMessagePassingLayer__state_update, h, adj, None, "sum", P_DROP)
    return h


def fused_forward(h):
    return gnn.gnn(h, adj, None, None, {}, {})


def step(forward):
    for q in gnn.parameters():
        q.grad = None
    h = h0.clone().requires_grad_(True)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ev[0].record()
    loss = forward(h).mean()
    ev[1].record()
    loss.backward()
    ev[2].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), (torch.cuda.max_memory_allocated() - base) / 2**20


paths = {"fused": fused_forward, "composed": composed_forward}
for f in paths.values():        # warm-up: module loads, plan build, library algorithm choice
    step(f)
    step(f)
res = {k: [] for k in paths}
for _ in range(REPS):
    for k, f in paths.items():
        res[k].append(step(f))


def median(xs):
    return sorted(xs)[len(xs) // 2]


out = {"card": card(), "layers": LAYERS, "p": P_DROP, "nodes": b.num_nodes, "edges": sum(int(s.shape[0]) for s, _ in adj), "reps": REPS}
for k, rows in res.items():
    out[k] = {"forward_ms": round(median([r[0] for r in rows]), 3), "backward_ms": round(median([r[1] for r in rows]), 3),
              "peak_mib_above_inputs": round(max(r[2] for r in rows), 1)}
print(json.dumps(out))
