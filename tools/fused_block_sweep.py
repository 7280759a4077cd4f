"""Fused aggregation kernel time against the target-block size B at config 2 (one Gated layer, library-side CUDA events):
    python tools/fused_block_sweep.py [B ...]
For fp32 and bf16 states and every B (default 64 88 120 144 176) it times the fused kernel per launch and the block-plan build,
fits the kernel time to a + b / B (least squares) and prints the fit with its prediction at B = 224 and B = 240.  The card
name and power limit are printed with the numbers."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200.synthetic import graph2class_batch  # noqa: E402

Bs = [int(x) for x in sys.argv[1:]] or [64, 88, 120, 144, 176]
PREDICT = (224, 240)
REPS = 20


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi not available"
    return f"{torch.cuda.get_device_name()} | {q}"


def timed(fn, reps):
    """{category: ms per launch} of `reps` calls of fn, from the library's per-launch CUDA events"""
    torch.cuda.synchronize()
    N.kernel_timing(True)
    N.read_kernel_timing()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    kt = N.read_kernel_timing()
    N.kernel_timing(False)
    return {k: v[0] / v[1] for k, v in kt.items() if v[1]}


def main():
    print("card:", card())
    b = graph2class_batch()
    torch.manual_seed(0)
    layer = P.GatedMessagePassingLayer(128, 128, 17, "sum").cuda().eval()
    gnn = P.GraphNeuralNetwork([layer], torch.nn.Identity(), True, True).cuda().eval()
    adj = gnn.expand_adjacency([(s.cuda(), t.cuda()) for s, t in b.adjacency_lists], b.num_nodes, "cuda")
    n = b.num_nodes
    print(f"nodes {n}, edges {sum(int(s.shape[0]) for s, _ in adj)}, types {len(adj)}")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for dtype in ("f32", "bf16"):
        h = torch.randn(n, 128, generator=torch.Generator().manual_seed(1)).cuda()
        if dtype == "bf16":
            h = h.to(torch.bfloat16)
        rows = []
        for B in Bs:
            plan_ms = timed(lambda: P.EdgePlan(adj, n, block_targets=B).block_plan(), 5).get("plan", float("nan"))
            plan = P.EdgePlan(adj, n, block_targets=B)
            plan.block_plan()

            def run():
                flush.zero_()
                with P.edgeplan.shared_plan(plan):
                    layer(h, adj)

            with torch.no_grad():
                for _ in range(5):
                    run()
                kt = timed(run, REPS)
            plan.validate()
            nblk = (n + B - 1) // B
            rows.append((B, nblk, kt["message"], plan_ms))
            print(f"{dtype} B={B:3d} blocks={nblk:5d}  fused {kt['message']:.4f} ms/launch  gru {kt.get('gru', float('nan')):.4f}  "
                  f"plan build {plan_ms:.4f} ms")
        x = np.array([1.0 / r[0] for r in rows])
        y = np.array([r[2] for r in rows])
        A = np.stack([np.ones_like(x), x], 1)
        (a, bb), *_ = np.linalg.lstsq(A, y, rcond=None)
        resid = y - A @ np.array([a, bb])
        print(f"{dtype} fit: t(B) = {a:.4f} + {bb:.3f} / B ms  (max |residual| {np.abs(resid).max():.4f} ms)")
        t176 = a + bb / 176
        for B in PREDICT:
            t = a + bb / B
            print(f"{dtype} predicted at B={B}: {t:.4f} ms  ({100 * (t176 - t) / t176:.1f} % below the fit at B=176, "
                  f"{(n + B - 1) // B} blocks)")


if __name__ == "__main__":
    main()
