"""Whole-step time of the config-2 layer loop (8 GatedMessagePassingLayers, plan build included, states resident), CUDA events:
    [PTGNN_TOOLS_LIB=tools/_variants/lib....so] python tools/step_time.py [f32|bf16] [label]
A/B tool: variants of the library are timed on the SAME box in one session (box-to-box spread is several percent)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ctypes  # noqa: E402

import torch  # noqa: E402

from ptgnn_b200 import _native as N  # noqa: E402

chain = True
if os.environ.get("PTGNN_TOOLS_LIB"):
    N.LIB_PATH = os.path.join(ROOT, os.environ["PTGNN_TOOLS_LIB"])
    probe = ctypes.CDLL(N.LIB_PATH)
    for name in list(N.SIGNATURES):          # older builds lack the newest entry points
        if not hasattr(probe, name):
            del N.SIGNATURES[name]
            chain = False
import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import edgeplan, globalexchange, gnn as gnn_module, messagepassing  # noqa: E402
from ptgnn_b200.synthetic import graph2class_batch  # noqa: E402

if not chain:                                   # older builds: no packed-state hand-off between layers
    for module in (edgeplan, messagepassing, globalexchange, gnn_module):
        module.current_state_chain = lambda: None
dtype = sys.argv[1] if len(sys.argv) > 1 else "f32"
label = sys.argv[2] if len(sys.argv) > 2 else ""
b = graph2class_batch()
torch.manual_seed(0)
if os.environ.get("STEP_LAYERS") == "mlp":        # the VarMisuse-style stack; STEP_NOCACHE=1: training mode (derived weights re-made per call)
    layers = [P.MlpMessagePassingLayer(128, 128, 128, 17, "max") for _ in range(8)]
else:
    layers = [P.GatedMessagePassingLayer(128, 128, 17, "sum") for _ in range(8)]
gnn = P.GraphNeuralNetwork(layers, torch.nn.Identity(), True, True).cuda().eval()
if os.environ.get("STEP_NOCACHE") == "1":
    gnn.train()
h = torch.randn(b.num_nodes, 128).cuda()
if dtype == "bf16":
    h = h.to(torch.bfloat16)
raw = [(s.cuda(), t.cuda()) for s, t in b.adjacency_lists]
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def step():
    P.clear_plan_cache()
    adj = gnn.expand_adjacency(raw, b.num_nodes, "cuda")
    return gnn.gnn(h, adj, None, None, {}, {})


with torch.no_grad():
    for _ in range(5):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(20):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
times.sort()
N.kernel_timing(True)
N.read_kernel_timing()
with torch.no_grad():
    for _ in range(5):
        step()
kt = N.read_kernel_timing()
N.kernel_timing(False)
print("   kernels: " + "  ".join(f"{k} {v[0] / max(v[1], 1):.4f} ms x{v[1] // 5}" for k, v in kt.items() if v[1]))
print(f"{dtype} chain={int(chain)} {label}: step median {times[len(times) // 2]:.3f} ms  min {times[0]:.3f}  p90 {times[17]:.3f}")
