"""Times PnaMessageAggregation at two shapes, fp32 and bf16 messages:

* native -- the module on the PNA kernel (DESIGN.md §3.10), plan of the targets cached as in repeated calls;
* shim -- the previous torch-op restatement of the reference's formula: five ``torch_scatter_shim`` scatters (degree, sum, max, min,
  std), the ``mean[targets]`` gather and the pointwise / ``cat`` passes (bf16: on the up-cast messages, as the reference does);
* native forward + backward of the module (fp32), and of an ``MlpMessagePassingLayer`` with the native PNA (fp32 states).

Call times come from CUDA events over many calls; kernel times from ``ptgnn_b200_kernel_timing_*`` (the PNA kernels run under
"reduce").  The HBM floor counts what the forward kernel must move: the messages read once, ``perm`` and ``row_ptr``, and the
[N, 15 D] fp32 output written once (at config 2 the output, ~1.57 GB, outweighs the ~0.57 GB of fp32 messages).  The backward's
floor: the messages and ``perm`` read once, ``d_out``, the mean and std blocks of the output and the arg ids read, ``d messages``
written.

    python tools/pna_time.py [--calls 50]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200 import torch_scatter_shim as ts  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet

SHAPES = (("config 2", 204_800, 1_105_920, 128), ("config 3", 80_000, 480_000, 128))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def shim_path(messages, targets, num_nodes, delta):
    """pna_aggregation.py:27-56 of the reference on the torch_scatter shim."""
    degree = ts.scatter(torch.ones_like(targets), index=targets, dim_size=num_nodes, reduce="sum")
    dtype = messages.dtype
    m = messages.to(torch.float32)
    total = ts.scatter(m, index=targets, dim=0, dim_size=num_nodes, reduce="sum")
    mean = total / (degree.unsqueeze(-1) + 1e-5)
    largest = ts.scatter(m, index=targets, dim=0, dim_size=num_nodes, reduce="max")
    smallest = ts.scatter(m, index=targets, dim=0, dim_size=num_nodes, reduce="min")
    spread = torch.relu(m.pow(2) - mean[targets].pow(2)) + 1e-10
    std = torch.sqrt(ts.scatter(spread, index=targets, dim=0, dim_size=num_nodes, reduce="sum"))
    stats = torch.cat([total, mean, largest, smallest, std], dim=-1).to(dtype)
    amplify = torch.log(degree.float() + 1).unsqueeze(-1) / delta
    return torch.cat([stats, stats * amplify, stats * (1 / (amplify + 1e-3))], dim=-1)


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
    ap.add_argument("--calls", type=int, default=50)
    args = ap.parse_args()
    print(f"card: {card()}")
    delta = 2.3
    for name, n, E, D in SHAPES:
        gen = torch.Generator(device="cuda").manual_seed(0)
        targets = torch.randint(0, n, (E,), device="cuda", generator=gen)
        agg = P.PnaMessageAggregation(delta=delta)
        for dtype in (torch.float32, torch.bfloat16):
            m = torch.randn(E, D, device="cuda", generator=gen).to(dtype)
            es = 2 if dtype == torch.bfloat16 else 4
            with torch.no_grad():
                native = lambda: agg(m, targets, n)  # noqa: E731
                t_nat = time_calls(native, args.calls)
                k_nat, launches = kernel_ms(native, 10)
                out_nat = native()
                cur = lambda: shim_path(m, targets, n, delta)  # noqa: E731
                t_cur = time_calls(cur, max(args.calls // 5, 3))
                out_cur = cur()
            floor = (E * D * es + E * 4 + (n + 1) * 4 + n * 15 * D * 4) / HBM_BYTES_PER_S * 1e3
            fin = torch.isfinite(out_cur)
            diff = ((out_nat - out_cur).abs()[fin].max() / out_cur.abs()[fin].max()).item()
            line = (f"{name} {str(dtype).replace('torch.', '')}: N={n} E={E} D={D}: native {t_nat:.4f} ms/call, shim {t_cur:.4f} ms/call "
                    f"({t_cur / t_nat:.1f}x); forward kernel {k_nat:.4f} ms ({launches} launches), HBM floor {floor:.4f} ms "
                    f"({k_nat / floor:.2f}x); max |native - shim| / max |shim| {diff:.2e}")
            if dtype == torch.float32:
                x = m.clone().requires_grad_(True)
                g = torch.randn(n, 15 * D, device="cuda", generator=gen)
                out = agg(x, targets, n)
                t_fb = time_calls(lambda: agg(x, targets, n).backward(g), args.calls)
                k_bwd, bl = kernel_ms(lambda: out.backward(g, retain_graph=True), 10)
                # messages read once (the second walk hits the caches), perm, d_out, the mean and std blocks of out, the arg ids,
                # d messages written once
                bfloor = (E * D * 4 + E * 4 + n * 15 * D * 4 + n * 2 * D * 4 + n * 2 * D * 4 + E * D * 4) / HBM_BYTES_PER_S * 1e3
                line += (f"; module forward + backward {t_fb:.4f} ms/call; backward kernel {k_bwd:.4f} ms ({bl} launches), "
                         f"HBM floor {bfloor:.4f} ms ({k_bwd / bfloor:.2f}x)")
            print(line, flush=True)
            del m
        # Mlp + PNA layer forward + backward (fp32 states, 3 edge types)
        H = 64
        src = torch.randint(0, n, (E,), device="cuda", generator=gen)
        cut = [0, E // 2, 5 * E // 6, E]
        adj = [(src[a:b], targets[a:b]) for a, b in zip(cut[:-1], cut[1:])]
        layer = P.MlpMessagePassingLayer(H, H, D, 3, P.PnaMessageAggregation(delta=delta)).cuda().train()
        h = torch.randn(n, H, device="cuda", generator=gen).requires_grad_(True)
        g = torch.randn(n, H, device="cuda", generator=gen)
        with torch.no_grad():
            t_f = time_calls(lambda: layer(h, adj), args.calls)
        t_fb = time_calls(lambda: layer(h, adj).backward(g), max(args.calls // 5, 3))
        print(f"{name} Mlp + PNA layer (H={H}, D={D}, 3 edge types, fp32): forward {t_f:.3f} ms/call, forward + backward {t_fb:.3f} ms/call",
              flush=True)


if __name__ == "__main__":
    main()
