"""Times EGCMessagePassingLayer on its fused slabs (DESIGN.md §3.14) against the composed path (edge_messages + segment_reduce +
linear, the [E, bases * out] message tensor), on the same card in the same run.

Shapes: config 2 (Graph2Class, 204,800 nodes, E = 1,105,920 after backward and self edges, T = 17, sum) and config 3 (VarMisuse,
80,000 nodes, E = 480,000, T = 23, max), with H = out = 128, 8 heads, 4 bases; fp32 and bf16 states (bf16: fused only, the composed
path takes fp32 states).  Per case: eval forward per call (CUDA events, median and 10th / 90th percentile; fused and composed calls
alternate), the library's kernel time and launch count per call (ptgnn_b200_kernel_timing_*), the peak memory above the inputs, the
fused training forward + backward per call (fp32), max |fused - composed| / max |composed|, and an HBM floor for the fused forward:
per slab, the gathered source rows (E rows of the packed states) + the output columns; the card's bandwidth from the H100 SXM data
sheet.  The card's name, power limit and clock are read in the same run.

    python tools/egc_time.py [--calls 20] [--out /tmp/egc_time.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200.synthetic import graph2class_batch, varmisuse_batch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet
H, OUT, HEADS, BASES = 128, 128, 8, 4


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()


def time_alternating(fns, calls, warmup=3):
    for _ in range(warmup):
        for f in fns:
            f()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(calls):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[i].append(a.elapsed_time(b))
    out = []
    for t in times:
        t = sorted(t)
        out.append({"median_ms": statistics.median(t), "p10_ms": t[len(t) // 10], "p90_ms": t[(9 * len(t)) // 10]})
    return out


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def kernel_time(fn, calls=10):
    torch.cuda.synchronize()
    N.kernel_timing(True)
    N.read_kernel_timing()
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    kt = N.read_kernel_timing()
    N.kernel_timing(False)
    return {k: {"ms_per_call": v[0] / calls, "launches_per_call": v[1] / calls} for k, v in kt.items() if v[1]}


def with_fp32_mode(value, fn):
    """fn under PTGNN_B200_FP32_MODE=value: "tf32" selects the composed path for fp32 states, "" the fused slabs."""
    def run():
        old = os.environ.get("PTGNN_B200_FP32_MODE")
        os.environ["PTGNN_B200_FP32_MODE"] = value
        try:
            return fn()
        finally:
            if old is None:
                del os.environ["PTGNN_B200_FP32_MODE"]
            else:
                os.environ["PTGNN_B200_FP32_MODE"] = old
    return run


def case(name, batch, agg, calls):
    torch.manual_seed(0)
    T = 2 * len(batch.adjacency_lists) + 1
    layer = P.EGCMessagePassingLayer(H, OUT, T, agg, num_bases=BASES, num_heads=HEADS).cuda().eval()
    gnn = P.GraphNeuralNetwork([layer], torch.nn.Identity(), True, True).cuda()
    adj = gnn.expand_adjacency([(s.cuda(), t.cuda()) for s, t in batch.adjacency_lists], batch.num_nodes, "cuda")
    n, E = batch.num_nodes, sum(int(s.numel()) for s, _ in adj)
    h32 = torch.randn(n, H, device="cuda")
    res = {"nodes": n, "edges": E, "types": T, "aggregation": agg}
    plan = P.EdgePlan(adj, n)
    with torch.no_grad(), P.edgeplan.shared_plan(plan):
        for dtype in ("fp32", "bf16"):
            h = h32 if dtype == "fp32" else h32.to(torch.bfloat16)
            fused = with_fp32_mode("", lambda: layer(h, adj))
            r = {}
            if dtype == "fp32":
                composed = with_fp32_mode("tf32", lambda: layer(h, adj))
                tf, tc = time_alternating([fused, composed], calls)
                r["fused_forward"], r["composed_forward"] = tf, tc
                a, b = fused(), composed()
                r["max_abs_diff_over_max_abs_composed"] = float((a - b).abs().max() / b.abs().max())
                r["composed_kernels"] = kernel_time(composed)
                r["composed_peak_mib"] = peak_bytes(composed) / 2**20
            else:
                (r["fused_forward"],) = time_alternating([fused], calls)
            r["fused_kernels"] = kernel_time(fused)
            r["fused_peak_mib"] = peak_bytes(fused) / 2**20
            row = H * (4 if dtype == "fp32" else 2)            # packed (hi | lo') fp16 rows of 4H bytes, or bf16 rows of 2H bytes
            slabs = BASES * OUT // 128
            floor_bytes = slabs * (E * row + n * (128 // BASES) * (4 if dtype == "fp32" else 2))
            r["hbm_floor_ms"] = floor_bytes / HBM_BYTES_PER_S * 1e3
            res[dtype] = r
    # training forward + backward (fp32)
    layer.train()
    g = torch.randn(n, OUT, device="cuda")
    x = h32.clone().requires_grad_(True)

    def train_step():
        layer.zero_grad(set_to_none=True)
        x.grad = None
        layer(x, adj).backward(g)

    (res["fp32"]["fused_forward_backward"],) = time_alternating([train_step], max(calls // 4, 3), warmup=2)
    layer.eval()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("egc_time.py measures on the GPU; no CUDA device found")
    result = {"card": card(), "torch": torch.__version__, "layer": dict(H=H, out=OUT, heads=HEADS, bases=BASES),
              "config2": case("config2", graph2class_batch(), "sum", args.calls),
              "config3": case("config3", varmisuse_batch(), "max", args.calls)}
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
