"""Timeline of the fused aggregation kernel (CTA 0) at config 2: python tools/fused_trace.py [f32|bf16] [label]
Sets PTGNN_FUSED_TRACE=1, runs one Gated layer a few times, prints the per-phase cycle breakdown of the last launch (clock64 of
the SM) and dumps the raw events to <dir>/fused_trace_<dtype>[_<label>].txt, <dir> = $PTGNN_TRACE_DIR or the system temporary
directory.  PTGNN_TOOLS_LIB selects another build of the library (tools only).  The roles and tags are listed above `trace_mark` in ptgnn_b200/csrc/fused_mp.cu."""
import ctypes
import os
import sys
import tempfile

os.environ["PTGNN_FUSED_TRACE"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200.synthetic import graph2class_batch  # noqa: E402

if os.environ.get("PTGNN_TOOLS_LIB"):
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
with torch.no_grad():
    for _ in range(3):
        layer(h, adj)
torch.cuda.synchronize()
lib = N.lib()
lib.ptgnn_b200_debug_fused_trace.argtypes = [ctypes.c_void_p]
cap = lib.ptgnn_b200_debug_fused_trace(None)
assert cap > 0, "tracing is off"
roles = ["gather", "wg0", "wg1", "reducer"]
buf = (ctypes.c_ulonglong * (len(roles) * cap))()
lib.ptgnn_b200_debug_fused_trace(buf)
ev = {}
for r, name in enumerate(roles):
    ev[name] = [((v >> 24), (v >> 8) & 0xFFFF, v & 0xFF) for v in buf[r * cap:(r + 1) * cap] if v]
out_dir = os.environ.get("PTGNN_TRACE_DIR") or tempfile.gettempdir()
os.makedirs(out_dir, exist_ok=True)
out_path = os.path.join(out_dir, f"fused_trace_{dtype}{'_' + label if label else ''}.txt")
t0 = min(e[0][0] for e in ev.values() if e)
with open(out_path, "w") as f:
    for name in roles:
        for clk, step, tag in ev[name]:
            f.write(f"{name} {clk - t0} {step} {tag}\n")


def by_step(name, tags):
    """step -> {tag: clock} over the events of `name` whose tag is in `tags` (steps and sub-groups are numbered separately)"""
    by = {}
    for clk, step, tag in ev[name]:
        if tag in tags:
            by.setdefault(step, {})[tag] = clk
    return by


def line(label, d, total=None):
    if not d:
        return
    d = sorted(d)
    s = sum(d)
    share = f"  {100.0 * s / total:5.1f} % of span" if total else ""
    print(f"  {label:40s} n={len(d):5d} mean {s / len(d):8.0f}  p50 {d[len(d) // 2]:7d}  p90 {d[int(len(d) * 0.9)]:7d}  sum {s:10d}{share}")


print(f"== {dtype} {label}: events recorded", {k: len(v) for k, v in ev.items()}, "raw events:", out_path)
g = by_step("gather", (1, 2, 3, 4))
print("gather (per step):")
line("wait x_empty", [v[2] - v[1] for v in g.values() if 1 in v and 2 in v])
line("issue cp.async", [v[3] - v[2] for v in g.values() if 2 in v and 3 in v])
for name in ("wg0", "wg1"):
    evs = ev[name]
    if not evs:
        continue
    span = max(c for c, _, _ in evs) - min(c for c, _, _ in evs)
    st = by_step(name, (10, 11, 12, 13, 14))
    sub = by_step(name, (20, 21, 22))
    print(f"{name}: span {span} cycles, {len(st)} steps, {len(sub)} sub-groups, "
          f"weights reloaded on {sum(1 for v in st.values() if 11 in v)} steps")
    order = sorted(evs)
    # fragment loads are issued in line (after the step's 10) or, with a look-ahead, after the previous step's 14
    line("weight fetch issue (prev event -> 11)", [c - order[i - 1][0] for i, (c, _, t) in enumerate(order) if t == 11 and i > 0], span)
    line("x_full wait (10 or 11 -> 12)", [v[12] - max(v[10], v.get(11, 0)) for v in st.values() if 10 in v and 12 in v], span)
    line("MMA issue, new weights (12->13)", [v[13] - v[12] for v in st.values() if 11 in v and 12 in v and 13 in v], span)
    line("MMA issue, same weights (12->13)", [v[13] - v[12] for v in st.values() if 11 not in v and 12 in v and 13 in v], span)
    line("MMA retire (13->14)", [v[14] - v[13] for v in st.values() if 13 in v and 14 in v], span)
    line("acc_empty wait (20->21)", [v[21] - v[20] for v in sub.values() if 20 in v and 21 in v], span)
    line("staging (21->22)", [v[22] - v[21] for v in sub.values() if 21 in v and 22 in v], span)
    # from the previous event to a step's begin (10): loop overhead, block-table waits
    line("before step begin (prev event -> 10)", [c - order[i - 1][0] for i, (c, _, t) in enumerate(order) if t == 10 and i > 0], span)
evs = ev["reducer"]
if evs:
    span = max(c for c, _, _ in evs) - min(c for c, _, _ in evs)
    sub = by_step("reducer", (30, 31, 32))
    wo = [(c, t) for c, _, t in evs if t in (33, 34)]
    print(f"reducer: span {span} cycles, {len(sub)} sub-groups, {sum(1 for _, t in wo if t == 33)} write-outs")
    line("acc_full wait (30->31)", [v[31] - v[30] for v in sub.values() if 30 in v and 31 in v], span)
    line("column walk (31->32)", [v[32] - v[31] for v in sub.values() if 31 in v and 32 in v], span)
    begins = [c for c, t in wo if t == 33]
    ends = [c for c, t in wo if t == 34]
    line("write-out incl. barriers (33->34)", [b_ - a for a, b_ in zip(begins, ends)], span)
