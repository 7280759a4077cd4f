"""Times one GruGlobalStateUpdate call (WeightedSum reducer) at the VarMisuse GGNN shape (40 x 2,000 nodes, H = 64) and at config 2's
shape (80 x 2,560, H = 128), fp32 and bf16 states:

* native -- the layer: the readout kernel, the [G, 3H] input-side table, the state-only weights-stationary GRU;
* current -- what the overlay ran before the native layer: the same formula on ``ptgnn_b200.scatter_sum`` (sigmoid(Linear(x)) * x as
  torch ops, the native two-level scatter) plus ``torch.nn.GRUCell`` on the per-node gathered summaries.

Call times come from CUDA events over many calls; per-kernel times from ``ptgnn_b200_kernel_timing_*`` (readout under "reduce",
GRU under "gru").  The HBM floor counts what the layer must move: the states read twice (readout, GRU) and the new states written.

    python tools/global_exchange_time.py [--calls 200]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200.edgeplan import shared_num_graphs  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def current_path(layer, h, n2g, G):
    """The reference formula on the pre-existing native pieces (scatter_sum) and torch.nn.GRUCell."""
    reducer = layer._AbstractGlobalGraphExchange__global_graph_representation_module
    w = reducer._WeightedSumVarSizedElementReduce__weights_layer
    x = h.float()
    s = torch.sigmoid(w(x).squeeze(-1))
    g = P.scatter_sum(x * s.unsqueeze(-1), n2g, dim=0, dim_size=G)
    gru = layer._GruGlobalStateUpdate__gru_cell
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=h.dtype == torch.bfloat16):    # bf16: the reference's AMP path
        return gru(g[n2g], h)


def time_calls(fn, calls):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def kernel_times(fn, calls):
    N.read_kernel_timing()
    N.kernel_timing(True)
    for _ in range(calls):
        fn()
    N.kernel_timing(False)
    return {k: (ms / max(n, 1), n // calls) for k, (ms, n) in N.read_kernel_timing().items() if n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    args = ap.parse_args()
    print(f"card: {card()}")
    for name, G, per, H in (("varmisuse GGNN (config 3)", 40, 2000, 64), ("config 2", 80, 2560, 128)):
        for dtype in (torch.float32, torch.bfloat16):
            torch.manual_seed(0)
            Nn = G * per
            n2g = torch.repeat_interleave(torch.arange(G, device="cuda"), per)
            h = (torch.randn(Nn, H, device="cuda") * 0.5).to(dtype)
            layer = P.GruGlobalStateUpdate(P.WeightedSumVarSizedElementReduce(H), H, H).cuda().eval()
            with torch.no_grad():
                with shared_num_graphs(G):
                    native = lambda: layer(h, [], n2g, {}, {}, [])  # noqa: E731
                    t_nat = time_calls(native, args.calls)
                    k_nat = kernel_times(native, 20)
                    out_nat = native().float()
                cur = lambda: current_path(layer, h, n2g, G)  # noqa: E731
                t_cur = time_calls(cur, args.calls)
                out_cur = cur().float()
            es = 2 if dtype == torch.bfloat16 else 4
            floor_ms = 3 * Nn * H * es / HBM_BYTES_PER_S * 1e3
            diff = (out_nat - out_cur).abs().max().item()
            kn = ", ".join(f"{k} {ms:.4f} ms x{n}" for k, (ms, n) in k_nat.items())
            print(f"{name} {str(dtype).replace('torch.', '')}: N={Nn} H={H} G={G}: native {t_nat:.4f} ms/call, current {t_cur:.4f} ms/call "
                  f"({t_cur / t_nat:.2f}x); kernels: {kn}; HBM floor {floor_ms:.4f} ms; max |native - current| {diff:.2e}")


if __name__ == "__main__":
    main()
