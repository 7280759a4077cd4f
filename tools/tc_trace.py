"""Debug: dump the CTA-0 timeline of one tensor-core pipeline launch (PTGNN_TC_TRACE=<category>, 1 = message, 3 = gru)."""
import ctypes, os, sys
sys.path.insert(0, os.getcwd())
import numpy as np, torch
import bench
from ptgnn_b200 import _native as N
batch = bench.make_batch("graph2class")
gnn = bench.build_model(17, "sum").cuda()
h = torch.randn(batch.num_nodes, 128).cuda()
if os.environ.get("TRACE_DTYPE") == "bf16":
    h = h.bfloat16()
adj = [(s.cuda(), t.cuda()) for s, t in batch.adjacency_lists]
ident = torch.arange(batch.num_nodes, device="cuda")
ex = list(adj) + [(t, s) for s, t in adj] + [(ident, ident)]
with torch.no_grad():
    for _ in range(3): gnn.gnn(h, ex, None, None, {}, {})
torch.cuda.synchronize()
lib = ctypes.CDLL(N.LIB_PATH)
buf = np.zeros(3 * 2048, dtype=np.uint64)
assert lib.ptgnn_b200_debug_trace(buf.ctypes.data_as(ctypes.c_void_p)) == 1
names = {1: "G wait empty", 2: "G empty ok", 3: "P wait landed", 4: "P cp.async ok", 5: "P landed ok", 6: "P full arrived(prev)",
         10: "M tile", 11: "M setup done", 12: "M tmem_empty ok", 13: "M wait full", 14: "M full ok", 16: "M landed ok", 15: "M committed",
         20: "E wait tmem_full", 21: "E tmem_full ok", 22: "E drained+released", 23: "E stored"}
ev = []
for r in range(3):
    for v in buf[r * 2048:(r + 1) * 2048]:
        if v: ev.append((int(v) >> 8, int(v) & 0xFF))
ev.sort()
t0 = ev[0][0]
lo, hi = int(os.environ.get("TRACE_FROM", 400)), int(os.environ.get("TRACE_TO", 560))
for t, tag in ev[lo:hi]:
    print(f"{t - t0:9d} ns  {names.get(tag, tag)}")
