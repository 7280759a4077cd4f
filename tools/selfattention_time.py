"""Times MultiHeadSelfAttentionMessagePassing at 80 x 2,560 nodes, in = out = 128, 8 heads, dk = dv = 16, intermediate 512,
max_num_nodes 250, with fp32 and bf16 states:

* native -- ``ptgnn_b200.MultiHeadSelfAttentionMessagePassing`` (dense products on the native linear, the chunked attention kernel,
  library LayerNorms), with the graph count handed in;
* shim -- the reference's forward (selfattmessagepassing.py:59-128) as it runs without the native class: the per-graph counts
  through ``ptgnn_b200.torch_scatter_shim``, a host loop over the chunks and torch ops (bf16: on the up-cast states);
* the forward kernel alone and the fp32 backward kernels alone, from CUDA events;
* the bounds from the shapes: the HBM floor (one read of t and one write of o at 3.35 TB/s, H100 SXM data sheet) and the
  tensor-core floor (the S and O products at 989 TFLOP/s dense fp16 / bf16, times 3 in fp32).

    python tools/selfattention_time.py [--calls 50]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import torch_scatter_shim as shim  # noqa: E402
from ptgnn_b200.edgeplan import shared_num_graphs  # noqa: E402
from ptgnn_b200.reduceops import graph_plan  # noqa: E402
from ptgnn_b200.selfattention import native_selfatt, native_selfatt_backward  # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet
TC_FLOP_PER_S = 989e12          # H100 SXM data sheet, dense fp16 / bf16
G, PER, D, DK, DV, HEADS, INTER, L = 80, 2560, 128, 16, 16, 8, 512, 250
PRE = "_MultiHeadSelfAttentionMessagePassing__"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def shim_path(m, x, n2g):
    """The reference's forward on torch ops and the torch_scatter shim (host loop over the chunks, one device read per graph)."""
    x = x.float()
    t = getattr(m, PRE + "selfatt_head_transforms")(x).reshape(x.shape[0], HEADS, -1)
    keys, queries, values = t[:, :, :DK], t[:, :, DK:2 * DK], t[:, :, 2 * DK:]
    counts = shim.scatter_sum(torch.ones_like(n2g, dtype=torch.int64), index=n2g)
    outs, off = [], 0
    for c in counts:
        for s in range(0, c, L):
            idx = torch.arange(s, min(s + L, c), dtype=torch.int64, device=x.device) + off
            scores = torch.einsum("khd,vhd->khv", keys[idx], queries[idx]) / DK ** 0.5
            outs.append(torch.einsum("khv,vhd->khd", torch.softmax(scores, dim=-1), values[idx]))
        off += c
    o = torch.cat(outs, dim=0)
    y1 = getattr(m, PRE + "layer_norm1")(getattr(m, PRE + "summarization_layer")(o.reshape(o.shape[0], -1)) + x)
    hidden = torch.relu(getattr(m, PRE + "intermediate_layer")(y1))
    return getattr(m, PRE + "layer_norm2")(getattr(m, PRE + "output_layer")(hidden) + y1)


def time_calls(fn, calls):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    args = ap.parse_args()
    print(f"card: {card()}")
    torch.manual_seed(0)
    n = G * PER
    n2g = torch.repeat_interleave(torch.arange(G, device="cuda"), PER)
    m = P.MultiHeadSelfAttentionMessagePassing(D, DK, DV, D, INTER, HEADS, max_num_nodes=L).cuda().eval()
    plan = graph_plan(n2g, G)
    W = 2 * DK + DV
    pairs = sum(min(L, PER - s) ** 2 for s in range(0, PER, L)) * G * HEADS       # (i, j) pairs inside the chunks
    flop = 2 * pairs * (DK + DV)
    for dtype in (torch.float32, torch.bfloat16):
        es = 2 if dtype == torch.bfloat16 else 4
        x = (torch.randn(n, D, device="cuda") * 0.5).to(dtype)
        t = (torch.randn(n, HEADS * W, device="cuda") * 0.5).to(dtype)

        def native():
            with shared_num_graphs(G):
                return m(x, [], n2g, {}, {}, [])

        with torch.no_grad():
            t_nat = time_calls(native, args.calls)
            t_ref = time_calls(lambda: shim_path(m, x, n2g), max(args.calls // 10, 2))
            t_fwd = time_calls(lambda: native_selfatt(t, plan, HEADS, DK, DV, L), args.calls)
            diff = ((native().float() - shim_path(m, x, n2g)).abs().max()).item()
        hbm_ms = (n * HEADS * W + n * HEADS * DV) * es / HBM_BYTES_PER_S * 1e3
        tc_ms = flop * (3 if dtype == torch.float32 else 1) / TC_FLOP_PER_S * 1e3
        line = (f"{str(dtype).replace('torch.', '')}: N={n} G={G} heads={HEADS} dk=dv={DK} L={L}: native call {t_nat:.3f} ms, "
                f"shim call {t_ref:.3f} ms; forward kernel {t_fwd:.4f} ms (HBM floor {hbm_ms:.4f} ms for "
                f"{(n * HEADS * W + n * HEADS * DV) * es / 1e6:.0f} MB, tensor-core floor {tc_ms:.4f} ms for {flop / 1e9:.1f} GFLOP)")
        if dtype == torch.float32:
            o, lse = native_selfatt(t, plan, HEADS, DK, DV, L)
            d_o = torch.randn_like(o)
            t_bwd = time_calls(lambda: native_selfatt_backward(t, plan, HEADS, DK, DV, L, o, lse, d_o), args.calls)
            line += f", backward kernels {t_bwd:.3f} ms"
        print(line + f"; max |native - shim| {diff:.2e}")


if __name__ == "__main__":
    main()
