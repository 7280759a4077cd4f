"""Kernel time of the fused aggregation / GRU kernels at config 2 (one Gated layer, library-side CUDA events):
    python tools/fused_time.py [f32|bf16] [label]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200.synthetic import graph2class_batch  # noqa: E402

if os.environ.get("PTGNN_TOOLS_LIB"):          # A/B against another build of the library (tools only; the package never reads this)
    N.LIB_PATH = os.path.join(ROOT, os.environ["PTGNN_TOOLS_LIB"])
dtype = sys.argv[1] if len(sys.argv) > 1 else "f32"
label = sys.argv[2] if len(sys.argv) > 2 else ""
b = graph2class_batch()
torch.manual_seed(0)
layer = P.GatedMessagePassingLayer(128, 128, 17, "sum").cuda().eval()
gnn = P.GraphNeuralNetwork([layer], torch.nn.Identity(), True, True).cuda().eval()
h = torch.randn(b.num_nodes, 128).cuda()
if dtype == "bf16":
    h = h.to(torch.bfloat16)
adj = gnn.expand_adjacency([(s.cuda(), t.cuda()) for s, t in b.adjacency_lists], b.num_nodes, "cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
with torch.no_grad():
    for _ in range(5):
        layer(h, adj)
    torch.cuda.synchronize()
    N.kernel_timing(True)
    N.read_kernel_timing()
    for _ in range(20):
        flush.zero_()
        layer(h, adj)
    torch.cuda.synchronize()
    kt = N.read_kernel_timing()
    N.kernel_timing(False)
print(f"{dtype} {label}: " + "  ".join(f"{k} {v[0] / max(v[1], 1):.4f} ms x{v[1]}" for k, v in kt.items() if v[1]))
