"""Times one GraphNorm call at four shapes, fp32 and bf16 states:

* native -- the layer on the GraphNorm kernels (DESIGN.md §3.9), graph count handed in, plan cached as in a container call;
* shim -- the reference's formula as it runs without the native class: two ``scatter_mean`` calls of ``torch_scatter_shim`` (no
  ``dim_size``, as the reference calls them), gathers and torch ops (bf16: on the up-cast states);
* native forward + backward (fp32): the layer under autograd, ``backward`` with a fixed ``dy``.

Call times come from CUDA events over many calls; kernel times from ``ptgnn_b200_kernel_timing_*`` (every GraphNorm kernel, the chunk
table and the backward's chunk-order sum run under "reduce").  HBM floors count what the kernels must move: the forward reads the
states twice and writes the output once; the backward as implemented reads x and dy twice each (chunk sums, then dx) and writes dx.

    python tools/graphnorm_time.py [--calls 200]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200 import torch_scatter_shim as shim  # noqa: E402
from ptgnn_b200.edgeplan import shared_num_graphs  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet
FWD_PASSES, BWD_PASSES = 3, 5  # [N, D] passes: forward 2 reads + 1 write; backward (x, dy) + (x, dy, dx)

SHAPES = (("config 2", 80, 2560, 128), ("varmisuse GGNN (config 3)", 40, 2000, 64), ("one graph", 1, 204800, 128),
          ("10,000 small graphs", 10000, 20, 128))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def shim_path(layer, x, n2g):
    """graphnorm.py:36-46 of the reference on the torch_scatter shim (fp32)."""
    x = x.float()
    mean = shim.scatter_mean(x, index=n2g, dim=0)
    shifted = x - layer.alpha * mean[n2g]
    sigma_2 = shim.scatter_mean(torch.pow(shifted, 2), index=n2g, dim=0) + 1e-10
    return layer.gamma * shifted / torch.sqrt(sigma_2[n2g]) + layer.bias


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


def kernel_ms(fn, calls):
    """Summed kernel time per call (all categories) and launches per call."""
    fn()
    torch.cuda.synchronize()
    N.read_kernel_timing()
    N.kernel_timing(True)
    for _ in range(calls):
        fn()
    N.kernel_timing(False)
    t = N.read_kernel_timing()
    return sum(ms for ms, _ in t.values()) / calls, sum(n for _, n in t.values()) // calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    args = ap.parse_args()
    print(f"card: {card()}")
    for name, G, per, D in SHAPES:
        Nn = G * per
        torch.manual_seed(0)
        n2g = torch.repeat_interleave(torch.arange(G, device="cuda"), per)
        n2g = n2g[torch.randperm(Nn, device="cuda")]
        layer = P.GraphNorm(D).cuda()
        with torch.no_grad():
            layer.gamma.uniform_(0.5, 1.5), layer.alpha.uniform_(0.0, 1.5), layer.bias.normal_(0.0, 0.3)
        for dtype in (torch.float32, torch.bfloat16):
            x = (torch.randn(Nn, D, device="cuda") * 2.0 + 1.0).to(dtype)
            es = 2 if dtype == torch.bfloat16 else 4
            with torch.no_grad(), shared_num_graphs(G):
                native = lambda: layer(x, [], n2g, {}, {}, [])  # noqa: E731
                t_nat = time_calls(native, args.calls)
                k_nat, launches = kernel_ms(native, 20)
                out_nat = native().float()
                cur = lambda: shim_path(layer, x, n2g)  # noqa: E731
                t_cur = time_calls(cur, max(args.calls // 10, 3))
                out_cur = cur()
            floor = FWD_PASSES * Nn * D * es / HBM_BYTES_PER_S * 1e3
            diff = ((out_nat - out_cur).abs().max() / out_cur.abs().max()).item()
            line = (f"{name} {str(dtype).replace('torch.', '')}: N={Nn} D={D} G={G}: native {t_nat:.4f} ms/call, shim {t_cur:.4f} ms/call "
                    f"({t_cur / t_nat:.1f}x); forward kernels {k_nat:.4f} ms ({launches} launches), HBM floor {floor:.4f} ms "
                    f"({k_nat / floor:.2f}x); max |native - shim| / max |shim| {diff:.2e}")
            if dtype == torch.float32:
                xg = x.clone().requires_grad_(True)
                dy = torch.randn(Nn, D, device="cuda")
                layer.train()
                with shared_num_graphs(G):
                    y = layer(xg, [], n2g, {}, {}, [])

                    def fwd_bwd():
                        layer(xg, [], n2g, {}, {}, []).backward(dy)

                    t_fb = time_calls(fwd_bwd, args.calls)
                    k_bwd, bl = kernel_ms(lambda: y.backward(dy, retain_graph=True), 20)
                layer.eval()
                bfloor = BWD_PASSES * Nn * D * 4 / HBM_BYTES_PER_S * 1e3
                line += (f"; forward + backward {t_fb:.4f} ms/call; backward kernels {k_bwd:.4f} ms ({bl} launches), HBM floor "
                         f"{bfloor:.4f} ms ({k_bwd / bfloor:.2f}x)")
            print(line, flush=True)


if __name__ == "__main__":
    main()
