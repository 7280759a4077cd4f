"""Times the native node embedder (DESIGN.md §3.12) against the same module built from torch ops, on one card in one run.

Per shape: the bag kernel alone (fp32 and bf16 output) next to its algorithmic bytes ``B S 8 + B 8 + B D s_out + min(V, B S) D 4``
(ids, lengths, output, the table rows touched) and the share of the HBM floor at the data-sheet 3.35 TB/s those bytes allow (HBM
is the bound that applies: the kernel has no arithmetic to speak of); the table gradient, whole and split into the plan of the
occurrences (pairs kernel + edge-plan build) and the backward kernels on a ready plan; the
``SubtokenUnitEmbedder`` module forward (eval) and forward + backward (train) against the torch-op module (embedding, mask, sum,
Linear), the two alternating call by call; and the table-first against the pool-first dense path on each side of V = B.

Times are CUDA events around each call after a warm-up, median and 10th / 90th percentile.  The card's name and power limit are
read in the same run.  Fails without a GPU.

    python tools/embedding_time.py [--calls 50] [--out /tmp/embedding_time.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import embeddings as E  # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet
# name -> (B, S, D, V)
SHAPES = {"typilus": (204_800, 5, 64, 10_000), "typilus_d128": (204_800, 5, 128, 10_000), "one_slot_d128": (204_800, 1, 128, 10_000)}


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()


class TorchOpEmbedder(nn.Module):
    """SubtokenUnitEmbedder("mean") as the reference writes it, on library ops."""

    def __init__(self, V, D):
        super().__init__()
        self.emb, self.out = nn.Embedding(V, D), nn.Linear(D, D, bias=False)

    def forward(self, token_idxs, lengths):
        embedded = self.emb(token_idxs)
        mask = torch.arange(embedded.shape[1], device=lengths.device).unsqueeze(0) < lengths.unsqueeze(-1)
        embedded = embedded * mask.unsqueeze(-1).float()
        return self.out(embedded.sum(dim=-2) / (lengths.unsqueeze(-1).float() + 1e-10))


def time_alternating(fns, calls, warmup=10):
    """Per function: (median, p10, p90) milliseconds of one call; the functions take turns call by call."""
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
        q = statistics.quantiles(t, n=10)
        out.append((statistics.median(t), q[0], q[-1]))
    return out


def inputs(B, S, V, gen):
    p = 1.0 / torch.arange(1, V + 1, dtype=torch.float64)
    ids = torch.multinomial(p / p.sum(), B * S, replacement=True, generator=gen).reshape(B, S).cuda()
    return ids, torch.randint(1, S + 1, (B,), generator=gen).cuda()


def fmt(t):
    return f"{t[0] * 1e3:8.1f} us  [{t[1] * 1e3:.1f}, {t[2] * 1e3:.1f}]"


def step_share(calls):
    """The embedder's share of a Typilus-shaped step: GraphNeuralNetwork.forward (embedder, edge plan, 8 gated layers of width 128 on
    the 204,800-node graph2class batch of tools/step_time.py), eval forward and training forward + backward, with the native embedder
    and with the torch-op one, next to each embedder alone on the same inputs."""
    from ptgnn_b200.synthetic import graph2class_batch

    b = graph2class_batch()
    D, V, S = 128, 10_000, 5
    gen = torch.Generator().manual_seed(1)
    ids, lens = inputs(b.num_nodes, S, V, gen)
    raw = [(s.cuda(), t.cuda()) for s, t in b.adjacency_lists]
    n2g = b.node_to_graph_idx.cuda()
    torch.manual_seed(0)
    layers = [P.GatedMessagePassingLayer(D, D, 17, "sum") for _ in range(8)]
    embedders = {"native": P.SubtokenUnitEmbedder(V, D, 0.0, "mean").cuda(), "torch_ops": TorchOpEmbedder(V, D).cuda()}
    gnns = {k: P.GraphNeuralNetwork(layers, e, True, True).cuda() for k, e in embedders.items()}

    def run(m, train):
        def f():
            if not train:
                with torch.no_grad():
                    return m(ids, lens) if not isinstance(m, P.GraphNeuralNetwork) else whole(m)
            m.zero_grad(set_to_none=True)
            out = m(ids, lens) if not isinstance(m, P.GraphNeuralNetwork) else whole(m).output_node_representations
            out.square().mean().backward()
        return f

    def whole(g):
        P.clear_plan_cache()
        return g(node_data=dict(token_idxs=ids, lengths=lens), adjacency_lists=raw, edge_feature_data=[], node_to_graph_idx=n2g,
                 reference_node_ids={}, reference_node_graph_idx={}, num_graphs=b.num_graphs)

    out = {}
    for train in (False, True):
        for m in list(gnns.values()) + list(embedders.values()):
            m.train(train)
        names = ["step, native embedder", "step, torch-op embedder", "native embedder alone", "torch-op embedder alone"]
        times = time_alternating([run(gnns["native"], train), run(gnns["torch_ops"], train), run(embedders["native"], train),
                                  run(embedders["torch_ops"], train)], calls, warmup=3)
        mode = "forward + backward (train)" if train else "forward (eval)"
        for n, t in zip(names, times):
            print(f"step share, {mode:26s} {n:24s} {fmt(t)}")
        print(f"step share, {mode:26s} embedder / step: native {times[2][0] / times[0][0]:.3f}   torch ops {times[3][0] / times[1][0]:.3f}")
        out["train" if train else "eval"] = dict(zip(names, times))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("embedding_time.py needs a CUDA device")
    result = {"card": card(), "calls": args.calls, "shapes": {}}
    print("card (name, power limit, max SM clock):", result["card"])
    gen = torch.Generator().manual_seed(0)
    for name, (B, S, D, V) in SHAPES.items():
        ids, lens = inputs(B, S, V, gen)
        table, d_out = torch.randn(V, D, device="cuda"), torch.randn(B, D, device="cuda")
        r = {}
        for dtype, size in ((torch.float32, 4), (torch.bfloat16, 2)):
            out = torch.empty(B, D, dtype=dtype, device="cuda")
            t, = time_alternating([lambda: E.native_embedding_bag(table, ids, lens, "mean", dtype, out=out)], args.calls)
            nbytes = B * S * 8 + B * 8 + B * D * size + min(V, B * S) * D * 4
            floor_us = nbytes / HBM_BYTES_PER_S * 1e6
            r[f"bag_{size * 8}"] = dict(ms=t, bytes=nbytes, hbm_floor_us=floor_us, share_of_hbm_floor=floor_us / (t[0] * 1e3))
            print(f"{name:16s} bag kernel, {str(dtype)[6:]:8s} out: {fmt(t)}   {nbytes / 1e6:6.1f} MB, HBM floor {floor_us:5.1f} us, "
                  f"share of the HBM floor reached {floor_us / (t[0] * 1e3):.2f}")
        ready = E.occurrence_plan(ids, lens, V)
        t, tp, tk = time_alternating([lambda: E.native_embedding_bag_backward(d_out, ids, lens, "mean", V),
                                      lambda: E.occurrence_plan(ids, lens, V),
                                      lambda: E.native_embedding_bag_backward(d_out, ids, lens, "mean", V, plan=ready)], args.calls)
        r["table_grad"] = dict(ms=t, plan_ms=tp, kernels_on_ready_plan_ms=tk)
        print(f"{name:16s} table gradient: {fmt(t)}   = plan of the occurrences {fmt(tp)}   + backward kernels {fmt(tk)}")
        # the module against the torch-op module, alternating
        native = P.SubtokenUnitEmbedder(V, D, 0.0, "mean").cuda()
        ref = TorchOpEmbedder(V, D).cuda()

        def fwd(m):
            with torch.no_grad():
                return m(ids, lens)

        def fwd_bwd(m):
            m.zero_grad(set_to_none=True)
            (m(ids, lens) * d_out).sum().backward()

        native.eval(), ref.eval()
        tn, tr = time_alternating([lambda: fwd(native), lambda: fwd(ref)], args.calls)
        r["module_forward"] = dict(native_ms=tn, torch_ops_ms=tr)
        print(f"{name:16s} module forward (eval):   native {fmt(tn)}   torch ops {fmt(tr)}   x{tr[0] / tn[0]:.2f}")
        native.train(), ref.train()
        tn, tr = time_alternating([lambda: fwd_bwd(native), lambda: fwd_bwd(ref)], args.calls)
        r["module_forward_backward"] = dict(native_ms=tn, torch_ops_ms=tr)
        print(f"{name:16s} module forward+backward: native {fmt(tn)}   torch ops {fmt(tr)}   x{tr[0] / tn[0]:.2f}")
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fwd_bwd(native)
        peak_n = torch.cuda.max_memory_allocated() - base
        torch.cuda.reset_peak_memory_stats()
        fwd_bwd(ref)
        peak_r = torch.cuda.max_memory_allocated() - base
        r["peak_bytes"] = dict(native=peak_n, torch_ops=peak_r)
        print(f"{name:16s} peak memory of forward+backward: native {peak_n / 1e6:.0f} MB   torch ops {peak_r / 1e6:.0f} MB")
        result["shapes"][name] = r
    # table-first against pool-first on each side of V = B (the module takes table-first when V <= B)
    D, S = 64, 5
    W = torch.randn(D, D, device="cuda") * 0.1
    for B, V in ((204_800, 10_000), (4_096, 50_000)):
        ids, lens = inputs(B, S, V, gen)
        table = torch.randn(V, D, device="cuda")
        from ptgnn_b200 import composed as C

        tf, pf = time_alternating([lambda: E.native_embedding_bag(C.linear(table, W), ids, lens, "mean"),
                                   lambda: C.linear(E.native_embedding_bag(table, ids, lens, "mean"), W)], args.calls)
        result[f"dense_B{B}_V{V}"] = dict(table_first_ms=tf, pool_first_ms=pf)
        print(f"dense path B={B:7d} V={V:6d}: table first {fmt(tf)}   pool first {fmt(pf)}   (the module takes {'table' if V <= B else 'pool'} first)")
    result["step_share"] = step_share(max(args.calls // 2, 10))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
