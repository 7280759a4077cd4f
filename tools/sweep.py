#!/usr/bin/env python
"""BASELINE.json configs[4]: edges/s sweep over single random graphs (not block diagonal).

    python tools/sweep.py [--out sweep.md] [--quick]

One GatedMessagePassingLayer and one MlpMessagePassingLayer call per point (plan build excluded, it is once per
minibatch): E in {1e4, 1e5, 1e6, 5e6}, N = E / 5, T in {1, 4, 16} (even split), H in {64, 128, 256}, sum and max.
Points with E <= 1e5 are also checked against the oracle (tests/helpers tolerance) and timed on the host CPU
(oracle port, all usable threads), so the table shows where the GPU path stops paying off.  The oracle is the
checker here, never the thing measured as "ours".
"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_time(fn, warmup=3, reps=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true")
    args = ap.parse_args()
    import ptgnn_b200 as P
    from ptgnn_b200.synthetic import single_random_graph
    from oracle import ptgnn_oracle as O
    import bench
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import helpers

    edges = [10_000, 100_000, 1_000_000, 5_000_000]
    types = [1, 4, 16]
    hidden = [64, 128, 256]
    if args.quick:
        edges, types, hidden = [10_000, 1_000_000], [4], [128]
    rows = []
    threads = bench.usable_cores() if hasattr(bench, "usable_cores") else os.cpu_count()
    torch.set_num_threads(threads)
    for i, E in enumerate(edges):
        for T in types:
            g = single_random_graph(E // 5, E, T, seed=2000 + i)
            adj_cpu = g.adjacency_lists
            adj = [(s.cuda(), t.cuda()) for s, t in adj_cpu]
            feats = [torch.zeros(len(s), 0) for s, _ in adj_cpu]
            for H in hidden:
                for agg in ("sum", "max"):
                    torch.manual_seed(0)
                    layers = {"gated": P.GatedMessagePassingLayer(H, H, T, agg).eval(),
                              "mlp": P.MlpMessagePassingLayer(H, H, H, T, agg).eval()}
                    h_cpu = torch.randn(g.num_nodes, H, generator=torch.Generator().manual_seed(7))
                    h = h_cpu.cuda()
                    for kind, layer in layers.items():
                        sd = {k: v.detach().clone() for k, v in layer.state_dict().items()}
                        layer = layer.cuda()
                        with torch.no_grad():
                            call = lambda: layer(node_states=h, adjacency_lists=adj, node_to_graph_idx=None, reference_node_ids={},
                                                 reference_node_graph_idx={}, edge_features=None)   # plan cached on `adj`
                            out = call()
                            ms = gpu_time(call)
                        err, cpu_ms = None, None
                        if E <= 100_000:
                            t0 = time.perf_counter()
                            if kind == "gated":
                                ref = O.gated_layer_forward(h_cpu, adj_cpu, feats, aggregation_fn=agg, **helpers.gated_oracle_args(sd))
                            else:
                                ref = O.mlp_layer_forward(h_cpu, adj_cpu, feats, aggregation_fn=agg, **helpers.mlp_oracle_args(sd))
                            cpu_ms = (time.perf_counter() - t0) * 1e3
                            err = float(((out.cpu() - ref).abs() / ref.abs().clamp(min=1.0)).max())
                        rows.append((E, g.num_nodes, T, H, agg, kind, ms, E / ms * 1e-6, cpu_ms, err))
                        print(rows[-1], flush=True)
    lines = ["# edges/s sweep on single random graphs (BASELINE.json configs[4]); one layer call, plan excluded", "",
             f"GPU: CUDA events, 3 warm-up + 10 timed calls. CPU: oracle port, one call, {threads} threads (only E <= 1e5). "
             "`err` = max |ours - oracle| / max(1, |oracle|) (bar 1e-5).", "",
             "| E | N | T | H | agg | layer | GPU ms | GPU G edges/s | CPU ms | GPU/CPU | err |", "|---|---|---|---|---|---|---|---|---|---|---|"]
    for E, N, T, H, agg, kind, ms, geps, cpu_ms, err in rows:
        lines.append(f"| {E:,} | {N:,} | {T} | {H} | {agg} | {kind} | {ms:.4f} | {geps:.3f} | "
                     f"{'' if cpu_ms is None else f'{cpu_ms:.1f}'} | {'' if cpu_ms is None else f'{cpu_ms / ms:.0f}x'} | {'' if err is None else f'{err:.1e}'} |")
    text = "\n".join(lines) + "\n"
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
    print(text)


if __name__ == "__main__":
    main()
