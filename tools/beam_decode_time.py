"""Times graph2seq's beam search (DESIGN.md §3.19) next to greedy decoding (§3.18), whole decodes timed with CUDA events.

    python tools/beam_decode_time.py [--iters 20] [--json OUT]

Shape: that of tools/greedy_decode_time.py -- 50 graphs, H = 128, E = 256, memories D = 128, V = 20,000, 8 steps, 0 to 59 memory rows
per graph, seeded parameters and inputs, eval mode.  Rows: ``decoding.greedy_decode`` and ``decoding.beam_decode`` with K in
{1, 2, 4, 8}, alternating, after a warm-up.  Per minibatch: milliseconds between an event recorded before the call and one recorded
after it returns (the call's host work included), the native launch count and whether K = 1 reproduced greedy's result.  The card's
name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200 import decoding  # noqa: E402
from greedy_decode_time import card, setup  # noqa: E402  (the same shape and inputs)

WIDTHS = (1, 2, 4, 8)


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    launches = N.launch_count()
    start.record()
    with torch.no_grad():
        out = fn()
    end.record()
    end.synchronize()
    return out, start.elapsed_time(end), N.launch_count() - launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    model, kw = setup()
    fns = {"greedy": lambda: decoding.greedy_decode(model, **kw)}
    for K in WIDTHS:
        fns[f"beam_{K}"] = lambda K=K: decoding.beam_decode(model, beam_width=K, **kw)
    for fn in fns.values():
        for _ in range(3):
            fn()
    times = {k: [] for k in fns}
    launches, outs = {}, {}
    for _ in range(args.iters):
        for name, fn in fns.items():
            outs[name], ms, launches[name] = timed(fn)
            times[name].append(ms)
    greedy = [(t, lp.tobytes()) for t, lp in outs["greedy"]]
    width_one = [(hs[0][0], hs[0][1].tobytes()) for hs in outs["beam_1"]]
    result = {"card": card(), "shape": "G=50 H=128 E=256 D=128 V=20000 steps=8", "memory_rows": kw["input_memories"].shape[0],
              "beam_1_equals_greedy": greedy == width_one}
    for name in fns:
        ts = sorted(times[name])
        result[name] = {"ms_median": statistics.median(ts), "ms_min": ts[0], "ms_max": ts[-1], "launches": launches[name]}
    print(json.dumps(result))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
