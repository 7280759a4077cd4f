"""Times the native classification heads (DESIGN.md §3.17) against the reference's torch formulation, with CUDA events.

    python tools/classification_heads_time.py [--iters 50] [--json OUT]

Shapes:
* Typilus (Graph2Class, config 2): N = 204,800 node states (the config-2 batch), H = 64 and 128, C = 101, S = 20,480 supernodes.  The
  supernode share (one node in ten) is an assumption, not a measured property of the Typilus data.
* PPI: H = 256, C = 121, at N = 3,000 (the reference's minibatch) and N = 204,800.
The torch formulation is the reference's head as written (graph2class.py:79-102, ppi.py:37-62): Linear on the gathered rows, argmax
accuracy and CrossEntropyLoss; Linear, sigmoid >= 0.5 counts, three ``float(x.cpu())`` metric reads and BCE-with-logits.  The native one
is ``ptgnn_b200.Graph2ClassModule`` / ``PPIClassification`` on a stub GNN that returns the same fp32 states.  Both time forward plus the
loss's backward into d h, d W and d b, and the forward alone, alternating three times.  The host synchronisations of one training step
of each are counted with torch's sync debug mode.  Prints the card name and power limit with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200.gnn import GnnOutput  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name()
    return out.splitlines()[0] if out else torch.cuda.get_device_name()


class StubGnn(nn.Module):
    def __init__(self, dim, output):
        super().__init__()
        self.output_node_state_dim = dim
        self.output = output

    def forward(self, **kwargs):
        return self.output


class TorchGraph2Class:
    """graph2class.py:79-102 on a fixed GNN output."""

    def __init__(self, h, idx, lin):
        self.h, self.idx, self.lin, self.acc = h, idx, lin, torch.zeros((), dtype=torch.int64, device=h.device)

    def __call__(self, target):
        logits = self.lin(self.h[self.idx])
        with torch.no_grad():
            self.acc += (torch.argmax(logits, dim=-1) == target).sum()
        return nn.functional.cross_entropy(logits, target)


class TorchPPI:
    """ppi.py:37-62 on a fixed GNN output."""

    def __init__(self, h, lin):
        self.h, self.lin, self.sums = h, lin, [0.0, 0.0, 0.0]

    def __call__(self, targets):
        logits = self.lin(self.h)
        with torch.no_grad():
            predictions = torch.sigmoid(logits) >= 0.5
            tp = (predictions & targets).sum().float()
            fp = (predictions & (~targets)).sum().float()
            fn = ((~predictions) & targets).sum().float()
            precision = tp / (tp + fp + 1e-10)
            recall = tp / (tp + fn + 1e-10)
            fscore = 2 * precision * recall / (precision + recall + 1e-10)
            n = int(predictions.shape[0])
            self.sums[0] += float(fscore.cpu()) * n
            self.sums[1] += float(precision.cpu()) * n
            self.sums[2] += float(recall.cpu()) * n
        return nn.functional.binary_cross_entropy_with_logits(logits, targets.float(), reduction="none").sum(dim=-1).mean()


def timed(fn, iters, backward):
    def step():
        loss = fn()
        if backward:
            loss.backward()

    for _ in range(5):
        step()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        step()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters * 1000.0


def host_syncs(fn):
    """Synchronising calls of one forward + backward, as torch's sync debug mode reports them."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn().backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("synchronizing" in str(w.message) for w in caught)


def compare(name, ref, nat, params, iters):
    out = {"forward_backward_us": {}, "forward_us": {}}
    for _ in range(3):
        for label, fn in (("torch", ref), ("native", nat)):
            for p in params:
                p.grad = None
            out["forward_backward_us"].setdefault(label, []).append(round(timed(fn, iters, True), 1))
            with torch.no_grad():
                out["forward_us"].setdefault(label, []).append(round(timed(fn, iters, False), 1))
    out["host_syncs_per_step"] = {"torch": host_syncs(ref), "native": host_syncs(nat)}
    print(name, json.dumps(out), flush=True)
    return out


def graph2class(H, iters, N=204_800, S=20_480, C=101):
    gen = torch.Generator().manual_seed(H)
    h = torch.randn(N, H, generator=gen).cuda().requires_grad_(True)
    idx = torch.randint(0, N, (S,), generator=gen).cuda()
    target = torch.randint(0, C, (S,), generator=gen).cuda()
    torch.manual_seed(1)
    m = P.Graph2ClassModule(StubGnn(H, GnnOutput(h, h, torch.zeros(N, dtype=torch.int64, device="cuda"), {"supernodes": idx},
                                                 {"supernodes": torch.zeros_like(idx)}, 1)), C).cuda()
    lin = m._Graph2ClassModule__node_to_class
    with torch.no_grad():
        lin.weight.mul_(0.05)
    ref = TorchGraph2Class(h, idx, lin)
    return compare(f"graph2class H={H}", lambda: ref(target), lambda: m({}, target, None), [h, lin.weight, lin.bias], iters)


def ppi(N, iters, H=256, C=121):
    gen = torch.Generator().manual_seed(N)
    h = torch.randn(N, H, generator=gen).cuda().requires_grad_(True)
    targets = (torch.rand(N, C, generator=gen) < 0.3).cuda()
    torch.manual_seed(2)
    m = P.PPIClassification(StubGnn(H, GnnOutput(h, h, torch.zeros(N, dtype=torch.int64, device="cuda"), {}, {}, 1)), C).cuda()
    lin = m._PPIClassification__output_representation_to_logits
    ref = TorchPPI(h, lin)
    return compare(f"ppi N={N}", lambda: ref(targets), lambda: m({}, targets), [h, lin.weight, lin.bias], iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "classification_heads_time.py measures on the GPU"
    result = {"card": card(),
              "graph2class": {f"N=204800 H={H} C=101 S=20480": graph2class(H, args.iters) for H in (64, 128)},
              "ppi": {f"N={N} H=256 C=121": ppi(N, args.iters) for N in (3000, 204_800)}}
    print(json.dumps(result))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
