"""Times the 8-head attention reducer at graph2seq's shape (80 x 2,560 nodes, D = 256 = the concatenated input and output states,
hidden 256, output 128, SimpleVarSizedElementReduce("max") query; graph2seq.py:55-65, 116-122), fp32 and bf16 states:

* native -- ``ptgnn_b200.MultiheadSelfAttentionVarSizedElementReduce``: the max query, the qt table, the attention readout kernel
  (3 launches), the output layer;
* shim -- the reference's forward (varsizedsummary.py:145-178) as the overlay runs it without the native class: torch ops for the
  layers and ``ptgnn_b200.torch_scatter_shim`` for ``scatter_log_softmax`` / ``scatter_sum`` (bf16: on the up-cast states);
* the max query alone (the native scatter), the forward kernel alone (``ptgnn_b200_attention_readout`` on a fixed qt) and the backward kernel alone (fp32), from CUDA events;
* the HBM floor: one read of the states at 3.35 TB/s (H100 SXM data sheet);
* the peak-memory increase of one call of each path.

    python tools/attention_readout_time.py [--calls 100]
"""
import argparse
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import torch_scatter_shim as shim  # noqa: E402
from ptgnn_b200.reduceops import graph_plan, native_attention_readout, native_attention_readout_backward, reduce_states  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet
G, PER, D, HIDDEN, OUT, HEADS = 80, 2560, 256, 256, 128, 8


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def shim_path(m, x, n2g):
    """The reference's multi-head forward on torch ops and the torch_scatter shim."""
    pre = "_MultiheadSelfAttentionVarSizedElementReduce__"
    key, out = getattr(m, pre + "key_layer"), getattr(m, pre + "output_layer")
    x = x.float()
    n = x.shape[0]
    queries = shim.scatter(x, n2g, dim=0, dim_size=G, reduce="max")[n2g].reshape(n, HEADS, HIDDEN // HEADS)
    keys = key(x).reshape(n, HEADS, HIDDEN // HEADS)
    scores = torch.einsum("bhk,bhk->bh", queries, keys) / math.sqrt(HIDDEN // HEADS)
    probs = torch.exp(shim.scatter_log_softmax(scores, index=n2g, dim=0, eps=0))
    outputs = (probs.unsqueeze(-1) * x.unsqueeze(1)).reshape(n, -1)
    return out(shim.scatter_sum(outputs, index=n2g, dim=0, dim_size=G))


def time_calls(fn, calls):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def peak_rise(fn):
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    args = ap.parse_args()
    print(f"card: {card()}")
    torch.manual_seed(0)
    n = G * PER
    n2g = torch.repeat_interleave(torch.arange(G, device="cuda"), PER)
    m = P.MultiheadSelfAttentionVarSizedElementReduce(D, HIDDEN, OUT, HEADS, P.SimpleVarSizedElementReduce("max")).cuda().eval()
    plan = graph_plan(n2g, G)
    qt = torch.randn(G, HEADS, D, device="cuda") * (4.0 / D ** 0.5)
    for dtype in (torch.float32, torch.bfloat16):
        x = (torch.randn(n, D, device="cuda") * 0.5).to(dtype)
        inputs = P.ElementsToSummaryRepresentationInput(x, n2g, G)
        with torch.no_grad():
            native = lambda: m(inputs)  # noqa: E731
            ref = lambda: shim_path(m, x, n2g)  # noqa: E731
            kernel = lambda: native_attention_readout(x, plan, qt, HEADS)  # noqa: E731
            query = lambda: reduce_states("max", None, x, n2g, plan)  # noqa: E731
            t_nat, t_ref, t_fwd = time_calls(native, args.calls), time_calls(ref, max(args.calls // 10, 5)), time_calls(kernel, args.calls)
            t_query = time_calls(query, args.calls)
            diff = ((native().float() - ref()).abs().max() / ref().abs().max()).item()
            mem_nat, mem_ref = peak_rise(native), peak_rise(ref)
            line = (f"{str(dtype).replace('torch.', '')}: N={n} D={D} heads={HEADS} G={G}: native call {t_nat:.4f} ms, shim call {t_ref:.4f} ms; "
                    f"max query {t_query:.4f} ms, forward kernel {t_fwd:.4f} ms")
            if dtype == torch.float32:
                o, lse = kernel()
                d_o = torch.randn_like(o)
                t_bwd = time_calls(lambda: native_attention_readout_backward(x, plan, qt, o, lse, d_o), args.calls)
                line += f", backward kernel {t_bwd:.4f} ms"
        es = 2 if dtype == torch.bfloat16 else 4
        floor_ms = n * D * es / HBM_BYTES_PER_S * 1e3
        print(line + f"; HBM floor (one read of x, {n * D * es / 1e6:.0f} MB) {floor_ms:.4f} ms; peak rise native {mem_nat:.1f} MiB, "
              f"shim {mem_ref:.1f} MiB; max |native - shim| / max |shim| {diff:.2e}")


if __name__ == "__main__":
    main()
