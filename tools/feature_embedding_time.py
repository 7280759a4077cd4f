"""Times the native LinearFeatureEmbedder (csrc/feature_embed.cu, DESIGN.md §3.15) against the library's F.linear + activation, on the
same card in the same run.

Shapes: PPI-like (N = 44,906 nodes: the PPI training set, F = 50, D = 64) and a large one (N = 200,000, F = 128, D = 128), ReLU, fp32
and bf16 (autocast).  Per shape and dtype:
* the kernel time per call, from the library's per-launch event timing (category "dense"), against the HBM floor N F 4 + N D (4 or 2)
  bytes at 3.35 TB/s (H100 SXM data sheet);
* the module's eval forward and the library's F.linear + ReLU (TF32 off for fp32: true fp32; bf16 under autocast), CUDA events around
  each call, calls alternating between the variants;
* fp32: a container of the embedder and one fused gated layer (message dimension 128, 3 edge types, 4 N edges each), with and without the packed hand-off
  (``current_state_chain`` replaced by ``lambda: None``), alternating: the difference is what the first layer saves by skipping its packing pass.
Times are the median and the 10th / 90th percentile.  The card's name, power limit and max SM clock are read in the same run.

    python tools/feature_embedding_time.py [--calls 50] [--out /tmp/feature_embedding_time.json]
"""
import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F_

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200 import edgeplan, globalexchange, gnn as gnn_module, messagepassing  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SHAPES = {"ppi": (44_906, 50, 64), "large": (200_000, 128, 128)}


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()


def stats(t):
    q = statistics.quantiles(t, n=10)
    return (statistics.median(t), q[0], q[-1])


def time_alternating(fns, calls, warmup=5):
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
    return [stats(t) for t in times]


def kernel_ms(f, calls):
    """Per-launch event time of the library's "dense" kernels (the embedder's forward kernel) over `calls` calls of f."""
    f()
    torch.cuda.synchronize()
    N.read_kernel_timing()
    N.kernel_timing(True)
    per_call = []
    for _ in range(calls):
        f()
        ms, launches = N.read_kernel_timing()["dense"]
        assert launches == 1, launches
        per_call.append(ms)
    N.kernel_timing(False)
    return stats(per_call)


@contextlib.contextmanager
def no_state_chain():
    """Inside the block no layer sees a state chain: every layer packs its own input states."""
    modules = (edgeplan, messagepassing, globalexchange, gnn_module)
    current = edgeplan.current_state_chain
    for module in modules:
        module.current_state_chain = lambda: None
    try:
        yield
    finally:
        for module in modules:
            module.current_state_chain = current


def fmt(t):
    return f"{t[0]:8.4f} ms  [{t[1]:.4f}, {t[2]:.4f}]"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    result = {"card": card(), "shapes": {}}
    print("card (name, power limit, max SM clock):", result["card"])
    torch.backends.cuda.matmul.allow_tf32 = False
    for name, (n, F, D) in SHAPES.items():
        torch.manual_seed(0)
        m = P.LinearFeatureEmbedder(F, D, torch.nn.ReLU()).cuda().eval()
        w = m.state_dict()["_LinearFeatureEmbedder__linear_map.weight"]
        x = torch.randn(n, F, device="cuda")
        row = {"N": n, "F": F, "D": D}
        for dtype in ("fp32", "bf16"):
            bf16 = dtype == "bf16"
            floor_ms = (n * F * 4 + n * D * (2 if bf16 else 4)) / HBM_BYTES_PER_S * 1e3

            def native():
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
                    m(x)

            def library():
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
                    F_.relu(F_.linear(x, w))

            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
                diff = (m(x).double() - F_.relu(F_.linear(x, w)).double()).abs().max().item()
            k = kernel_ms(native, args.calls)
            call = time_alternating([native, library], args.calls)
            row[dtype] = {"kernel_ms": k, "hbm_floor_ms": floor_ms, "floor_share": floor_ms / k[0], "module_call_ms": call[0],
                          "library_linear_relu_ms": call[1], "max_abs_diff_vs_library": diff}
            print(f"\n{name} {dtype}: N={n} F={F} D={D}  HBM floor {floor_ms:.4f} ms")
            print(f"  kernel        {fmt(k)}   floor share {floor_ms / k[0]:.2f}")
            print(f"  module call   {fmt(call[0])}")
            print(f"  F.linear+relu {fmt(call[1])}   max |native - library| {diff:.2e}")
        # the first fused layer with and without the packed hand-off
        gen = torch.Generator().manual_seed(1)
        adj = [(torch.randint(0, n, (4 * n,), generator=gen).cuda(), torch.randint(0, n, (4 * n,), generator=gen).cuda()) for _ in range(3)]
        assert N.lib().ptgnn_b200_fused_supported(0, D, 128)
        gnn = P.GraphNeuralNetwork([P.GatedMessagePassingLayer(D, 128, 3, "sum")], m, False, False).cuda().eval()
        kw = dict(node_data={"features": x}, adjacency_lists=adj, edge_feature_data=[], reference_node_ids={},
                  reference_node_graph_idx={}, node_to_graph_idx=torch.zeros(n, dtype=torch.int64, device="cuda"), num_graphs=1)

        def chained():
            with torch.no_grad():
                gnn(**kw)

        def unchained():
            with torch.no_grad(), no_state_chain():
                gnn(**kw)

        with torch.no_grad():
            with_handoff = gnn(**kw).output_node_representations
            with no_state_chain():
                without = gnn(**kw).output_node_representations
            same = torch.equal(with_handoff, without)
        c = time_alternating([chained, unchained], args.calls)
        row["container_fp32"] = {"chained_ms": c[0], "unchained_ms": c[1], "saved_ms": c[1][0] - c[0][0], "bit_identical": same}
        print(f"  container (embedder + fused gated layer), fp32: hand-off {fmt(c[0])}, without {fmt(c[1])}, "
              f"saved {c[1][0] - c[0][0]:.4f} ms, bit-identical {same}")
        result["shapes"][name] = row
        del m, gnn, x, adj
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
