"""Times the native CharUnitEmbedder (csrc/char_cnn.cu, DESIGN.md §3.13) against the reference's formulation on library ops, on the
same card in the same run.

Shapes: VarMisuse (B = 80,000 tokens of L = 15 characters, C = 101, the default CnnConfig(256, 3, 128, 3, 3)) at D = 63 and D = 127,
plus D = 128 and B = 204,800.  Per shape: the eval forward (native fp32, native bf16 under autocast, library ops with cuDNN TF32 off --
true fp32 -- and on, the library default), the training forward + backward (native fp32, library ops with TF32 off), and the peak
memory of each.  Calls alternate between the variants; times are CUDA events, median and 10th / 90th percentile.  Reported with
each: the algorithmic FLOPs (layers 2 and 3, 2 per multiply-add), the share of the tensor-core floor at the data-sheet rate (fp32
through the 3xFP16 split counts three products), and the kernel's per-token L2 weight bytes.  The card's name and power limit are
read in the same run.

    python tools/char_embedding_time.py [--calls 30] [--out /tmp/char_embedding_time.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ptgnn_b200.embeddings import CharUnitEmbedder, CnnConfig  # noqa: E402

DENSE_F16_FLOPS = 989e12         # H100 SXM data sheet, dense fp16 / bf16 tensor core
CFG = CnnConfig(256, 3, 128, 3, 3)
SHAPES = {"varmisuse_d63": (80_000, 63), "varmisuse_d127": (80_000, 127), "d128": (80_000, 128), "b204800_d127": (204_800, 127)}
C, L = 101, 15


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()


def library_forward(m, chars):
    """The reference's CharUnitEmbedder.forward (strelementrepresentationmodel.py:128-142) on library ops, with m's parameters."""
    w1, b1, w2, b2, w3 = m._params()
    x = F.one_hot(chars, C).transpose(1, 2).float()
    l2 = F.conv1d(F.relu(F.conv1d(x, w1, b1)), w2, b2)
    return F.conv1d(F.relu(l2), w3).max(dim=-1).values


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
    out = []
    for t in times:
        q = statistics.quantiles(t, n=10)
        out.append((statistics.median(t), q[0], q[-1]))
    return out


def peak_mb(f):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    f()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def flops(B, D):
    L1 = L - CFG.l1_window_size + 1
    L2, L3 = L1 - CFG.l2_window_size + 1, L1 - CFG.l2_window_size - CFG.lout_window_size + 2
    return 2.0 * B * (L2 * CFG.l2_filters * CFG.l1_filters * CFG.l2_window_size + L3 * D * CFG.l2_filters * CFG.lout_window_size)


def l2_weight_bytes_per_token(D, bf16):
    """Weight stages each tile copies from L2 (csrc/char_cnn.cu: 128 rows x 64 channels per stage, hi and lo' for fp32), per token."""
    copies = 1 if bf16 else 2
    dp = 64 if D <= 64 else (128 if D <= 128 else 256)
    w2 = CFG.l2_window_size * (CFG.l1_filters // 64) * CFG.l2_filters * 128 * copies
    w3 = CFG.lout_window_size * (CFG.l2_filters // 64) * dp * 128 * copies
    tokens = min(128 // (L - CFG.l1_window_size + 1), 16)
    return (w2 + w3) / tokens


def fmt(t):
    return f"{t[0]:8.3f} ms  [{t[1]:.3f}, {t[2]:.3f}]"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    result = {"card": card(), "shapes": {}}
    print("card (name, power limit, max SM clock):", result["card"])
    for name, (B, D) in SHAPES.items():
        torch.manual_seed(0)
        m = CharUnitEmbedder(C, D, CFG, 0.0).cuda().eval()
        chars = torch.randint(0, C, (B, L), device="cuda")
        fl = flops(B, D)

        def native():
            with torch.no_grad():
                m(chars)

        def native_bf16():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                m(chars)

        def lib(tf32):
            def f():
                torch.backends.cudnn.allow_tf32 = tf32
                with torch.no_grad():
                    library_forward(m, chars)
            return f

        def train_native():
            m.train()
            for p in m.parameters():
                p.grad = None
            m(chars).sum().backward()
            m.eval()

        def train_lib():
            torch.backends.cudnn.allow_tf32 = False
            for p in m.parameters():
                p.grad = None
            library_forward(m, chars).sum().backward()

        fwd = time_alternating([native, native_bf16, lib(False), lib(True)], args.calls)
        trn = time_alternating([train_native, train_lib], max(5, args.calls // 3))
        mem = {"native": peak_mb(native), "library": peak_mb(lib(False)), "train_native": peak_mb(train_native),
               "train_library": peak_mb(train_lib)}
        torch.backends.cudnn.allow_tf32 = True
        row = {"B": B, "D": D, "gflop": fl / 1e9,
               "eval_ms": {"native_fp32": fwd[0], "native_bf16": fwd[1], "library_fp32": fwd[2], "library_tf32": fwd[3]},
               "train_ms": {"native_fp32": trn[0], "library_fp32": trn[1]}, "peak_mb": mem,
               "floor_share": {"native_fp32": 3 * fl / DENSE_F16_FLOPS / (fwd[0][0] * 1e-3), "native_bf16": fl / DENSE_F16_FLOPS / (fwd[1][0] * 1e-3)},
               "l2_weight_bytes_per_token": {"fp32": l2_weight_bytes_per_token(D, False), "bf16": l2_weight_bytes_per_token(D, True)}}
        result["shapes"][name] = row
        print(f"\n{name}: B={B} D={D}  {fl / 1e9:.1f} GFLOP  L2 weight bytes/token fp32 {row['l2_weight_bytes_per_token']['fp32'] / 1e3:.1f} KB, "
              f"bf16 {row['l2_weight_bytes_per_token']['bf16'] / 1e3:.1f} KB")
        for k, v in row["eval_ms"].items():
            print(f"  eval  {k:13s} {fmt(v)}")
        for k, v in row["train_ms"].items():
            print(f"  train {k:13s} {fmt(v)}")
        print(f"  floor share fp32 {row['floor_share']['native_fp32']:.2f}, bf16 {row['floor_share']['native_bf16']:.2f};  peak MB "
              + ", ".join(f"{k} {v:.0f}" for k, v in mem.items()))
        del m, chars
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
