"""One training step of a stack of MlpMessagePassingLayers at config 2's shape (N = 204,800, E ~ 1.1 M after backward and self edges,
T = 17, H = D = 128) in bf16 and in fp32, and the parameter-gradient products alone: the gathered bf16 kernel (csrc/wgrad.cu)
against the fp32 path's gather-split and three fp16 GEMMs per type (``_mm_t_split``).  CUDA events around warmed-up repetitions.

    python tools/mlp_bf16_train_time.py [--layers 4] [--reduce sum] [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import autograd as AG  # noqa: E402
from ptgnn_b200.edgeplan import plan_for  # noqa: E402
from ptgnn_b200.synthetic import graph2class_batch  # noqa: E402


def _time(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--reduce", default="sum")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    b = graph2class_batch()
    raw = [(s.cuda(), t.cuda()) for s, t in b.adjacency_lists]
    result = {"gpu": gpu, "layers": args.layers, "reduce": args.reduce}
    h0 = torch.randn(b.num_nodes, 128, device="cuda")
    for name, dtype in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        torch.manual_seed(0)
        T = 2 * len(raw) + 1
        layers = [P.MlpMessagePassingLayer(128, 128, 128, T, args.reduce) for _ in range(args.layers)]
        gnn = P.GraphNeuralNetwork(layers, torch.nn.Identity(), True, True).cuda().train()
        adj = gnn.expand_adjacency(raw, b.num_nodes, "cuda")
        h = h0.to(dtype).requires_grad_(True)

        def step():
            out = gnn.gnn(h, adj, None, None, {}, {})
            out = out[-1] if isinstance(out, (list, tuple)) else out
            out.float().square().mean().backward()

        result[f"step_ms_{name}"] = round(_time(step, args.reps), 3)
        result["edges"] = sum(int(s.shape[0]) for s, _ in adj)
        del gnn, layers

    # the parameter-gradient products of one layer (use_target: [D, 2H] per type) on the same graph
    gnn = P.GraphNeuralNetwork([P.MlpMessagePassingLayer(128, 128, 128, 17, "sum")], torch.nn.Identity(), True, True)
    adj = gnn.expand_adjacency(raw, b.num_nodes, "cuda")
    plan = plan_for(adj, b.num_nodes)
    d_agg = torch.randn(b.num_nodes, 128, device="cuda") * 1e-7
    h32 = h0
    hb = h0.to(torch.bfloat16)

    def fp32_products():
        scale = AG._pow2_scale(d_agg)
        a_all = AG._split16(d_agg, plan.tgt32, scale)
        b_all, g_all = AG._split16(h32, plan.src32), AG._split16(h32, plan.tgt32)
        for t in range(plan.num_types):
            lo, hi = plan.type_off[t], plan.type_off[t + 1]
            a = AG._slice(a_all, lo, hi)
            AG._mm_t_split(a, AG._slice(b_all, lo, hi))
            AG._mm_t_split(a, AG._slice(g_all, lo, hi))

    def bf16_products():
        s, inv = AG._pow2_scale(d_agg)
        AG._weight_grad_bf16(plan, (d_agg * s).to(torch.bfloat16), plan.tgt32, inv, hb, True)

    result["weight_grad_ms_fp32_split_gemms"] = round(_time(fp32_products, args.reps * 2), 3)
    result["weight_grad_ms_bf16_kernel"] = round(_time(bf16_products, args.reps * 2), 3)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
