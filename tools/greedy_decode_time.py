"""Times graph2seq's greedy decoding (DESIGN.md §3.18): the native decode loop against a host loop with the reference method's structure.

    python tools/greedy_decode_time.py [--iters 20] [--json OUT]

Shape: graph2seq's decoder defaults (grucopydecoder.py:220-230): 50 graphs, H = 128, E = 256, memories D = 128, V = 20,000, 8 steps,
with 0 to 59 memory rows per graph and copied values that are partly in the vocabulary and partly not.  Seeded parameters and inputs.

* native: ``ptgnn_b200.decoding.greedy_decode``.
* host loop: written here from the contract (the reference's code is not used): per step, the decoder module's own
  ``_compute_logprobs`` for one step (this package's ``GruCopyingDecoder``, so the attention already runs on the native kernels), a
  ``[G, V]`` top-100, the top-100 and the ``[M]`` copy log-probabilities copied to the host, and the merge in Python dictionaries keyed
  by string, then a Python ``max``.
Both run the same module in eval mode on the same inputs, alternating, after a warm-up.  Per minibatch: milliseconds (wall time around
a synchronised call), native launches (``ptgnn_b200_launch_count``) and host synchronisations (torch's sync debug mode, counted as
warnings).  The card's name and power limit are read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200 import decoding  # noqa: E402
import greedy_decode_reference as GR  # noqa: E402  (the vocabulary and decoder-model stand-ins)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out.splitlines()[0] if out else torch.cuda.get_device_name()


def host_loop_decode(model, *, input_concrete_values, input_memories, input_memories_origin_idx, initial_states, neural_model):
    """The reference method's structure, from the contract: one-step _compute_logprobs, top-100 and copy log-probabilities to the
    host, a string-keyed dictionary merge and a Python max per graph."""
    vocab = model._GruCopyingDecoderModel__output_vocabulary
    G = initial_states.shape[0]
    h = initial_states
    ids = torch.full((G, 1), vocab.get_id_or_unk(model.START), dtype=torch.int64, device=input_memories.device)
    tokens, logprobs, done = [[] for _ in range(G)], [0.0] * G, [False] * G
    origin = input_memories_origin_idx.cpu().numpy()
    for _ in range(model.max_seq_len):
        copy_lp, target_lp, h_new = neural_model._compute_logprobs(h, input_memories, input_memories_origin_idx, ids)
        h = h_new.squeeze(0)
        top_lp, top_ids = torch.topk(target_lp.squeeze(1), min(100, target_lp.shape[-1]), dim=-1)
        top_lp, top_ids, copy_lp = top_lp.cpu().numpy(), top_ids.cpu().numpy(), copy_lp.squeeze(1).cpu().numpy()
        preds = [{vocab.get_name_for_id(int(i)): lp for i, lp in zip(top_ids[g], top_lp[g])} for g in range(G)]
        for g, value, lp in zip(origin, input_concrete_values, copy_lp):
            preds[g][value] = np.logaddexp(preds[g].get(value, -math.inf), lp)
        step = []
        for g in range(G):
            if done[g]:
                step.append(model.END)
                continue
            tok, lp = max(preds[g].items(), key=lambda kv: kv[1])
            if tok == model.END:
                done[g] = True
            else:
                tokens[g].append(tok)
            step.append(tok)
            logprobs[g] += lp
        ids = torch.tensor([[vocab.get_id_or_unk(t)] for t in step], device=input_memories.device)
    return list(zip(tokens, logprobs))


def setup(G=50, H=128, E=256, D=128, V=20000, T=8, seed=0):
    gen = torch.Generator().manual_seed(seed)
    vocab = GR.TokenVocab([GR.UNK, GR.START, GR.END] + [f"v{i}" for i in range(3, V)])
    torch.manual_seed(seed)
    module = P.GruCopyingDecoder(V, E, H, D, unk_id=0, dropout_rate=0.2).cuda().eval()
    counts = torch.randint(0, 60, (G,), generator=gen)
    origin = torch.repeat_interleave(torch.arange(G), counts)
    origin = origin[torch.randperm(origin.numel(), generator=gen)]
    values = [f"v{int(i)}" if i < V else f"ident{int(i) - V}" for i in torch.randint(3, V + 400, (origin.numel(),), generator=gen)]
    kw = dict(input_concrete_values=values, input_memories=torch.randn(origin.numel(), D, generator=gen).cuda(),
              input_memories_origin_idx=origin.cuda(), initial_states=torch.randn(G, H, generator=gen).cuda(), neural_model=module)
    return GR.DecoderModelStub(vocab, T), kw


def measure(fn, model, kw):
    torch.cuda.synchronize()
    launches = N.launch_count()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            t0 = time.perf_counter()
            with torch.no_grad():
                out = fn(model, **kw)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = sum(1 for w in caught if "synchroniz" in str(w.message).lower()) - 1        # the timing's own synchronize
    return out, ms, N.launch_count() - launches, syncs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    model, kw = setup()
    fns = {"native": decoding.greedy_decode, "host_loop": host_loop_decode}
    with torch.no_grad():
        for fn in fns.values():
            for _ in range(3):
                fn(model, **kw)
    times = {k: [] for k in fns}
    info = {}
    for _ in range(args.iters):
        for name, fn in fns.items():
            out, ms, launches, syncs = measure(fn, model, kw)
            times[name].append(ms)
            info[name] = {"launches": launches, "host_syncs": syncs, "tokens": [t for t, _ in out]}
    same = sum(a == b for a, b in zip(info["native"]["tokens"], info["host_loop"]["tokens"]))
    result = {"card": card(), "shape": "G=50 H=128 E=256 D=128 V=20000 steps=8", "memory_rows": kw["input_memories"].shape[0]}
    for name in fns:
        ts = sorted(times[name])
        result[name] = {"ms_median": statistics.median(ts), "ms_min": ts[0], "ms_max": ts[-1], "launches": info[name]["launches"],
                        "host_syncs": info[name]["host_syncs"]}
    result["graphs_with_equal_tokens"] = f"{same}/{len(info['native']['tokens'])}"
    print(json.dumps(result))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
