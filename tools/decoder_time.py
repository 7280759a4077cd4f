"""Times the graph2seq decoder's ``_compute_logprobs`` at a synthetic graph2seq-like shape: G = 80 samples of 640 memory rows each
(a quarter of graph2seq's 2,560-node graphs taken as backbone), D = H = 128, E = 256, V = 20,000, L = 7 decoder steps.

* native -- ``ptgnn_b200.GruCopyingDecoder._compute_logprobs`` (DESIGN.md §3.11), forward under no_grad, and forward + backward;
* the two attention kernels alone: the copy kernel (``native_copy_attention``) and the attention-readout call it shares with the
  reducers (``native_attention_readout``, the 7 steps padded to 8 heads);
* shim -- the reference's ``_compute_logprobs`` (grucopydecoder.py:59-142) written with the same torch ops on the
  ``torch_scatter_shim`` (``scatter_log_softmax``, ``scatter_add``, ``scatter_logsumexp``), forward only: the shim has no autograd,
  so its backward is incomplete.  That is shown directly: after a backward of the reference's loss (grucopydecoder.py:144-212) through
  the shim restatement, the two attention weights' ``.grad`` and the memories' ``.grad`` stay None; through the native class they do not.

Times are CUDA events over many calls after a warm-up; peak memory is ``max_memory_allocated`` above what was allocated before the
call.  The card's name and power limit are read in the same run.

    python tools/decoder_time.py [--calls 50] [--out /tmp/decoder_time.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import torch_scatter_shim as ts  # noqa: E402
from ptgnn_b200.decoder import native_copy_attention  # noqa: E402
from ptgnn_b200.reduceops import graph_plan, native_attention_readout  # noqa: E402

G, PER, H, E, V, L = 80, 640, 128, 256, 20_000, 7


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def shim_compute_logprobs(m, initial_states, memories, origin, token_ids):
    """The reference's _compute_logprobs on the shim, with the native module's parameters (its dropout is 0 here)."""
    p = "_GruCopyingDecoder__"
    emb = getattr(m, p + "embedding_layer")
    output_states, state = getattr(m, p + "output_gru")(emb(token_ids), initial_states.unsqueeze(0))
    output_states = output_states.contiguous()
    std = getattr(m, p + "memories_to_standard_attention")(memories)
    cop = getattr(m, p + "memories_to_copy_attention")(memories)
    per_row = output_states[origin]
    std_scores = torch.einsum("ilh,ih->il", per_row, std)
    copy_scores = torch.einsum("ilh,ih->il", per_row, cop)
    std_lp = ts.scatter_log_softmax(std_scores, index=origin, dim=0, eps=0)
    ctx = ts.scatter_add(torch.einsum("il,ih->ilh", torch.exp(std_lp), std), index=origin, dim=0)
    target_scores = torch.einsum("blh,hd,vd->blv", torch.cat((ctx, output_states), dim=-1), getattr(m, p + "hidden_to_vocab"),
                                 emb.weight) + getattr(m, p + "vocab_bias")
    total_copy = ts.scatter_logsumexp(copy_scores, index=origin, dim=0, eps=0)
    norm = torch.logsumexp(torch.cat((target_scores, total_copy.unsqueeze(-1)), dim=-1), dim=-1)
    return copy_scores - norm[origin], target_scores - norm.unsqueeze(-1), state


def shim_loss(m, initial_states, memories, origin, target_token_ids, copyable_elements_idxs, copyable_elements_sample_idxs, target_lengths):
    """The reference's forward (grucopydecoder.py:144-212) on the shim restatement."""
    copy_lp, target_lp, _ = shim_compute_logprobs(m, initial_states, memories, origin, target_token_ids[:, :-1])
    B, T = target_token_ids.shape[0], target_token_ids.shape[1] - 1
    valid = ts.scatter_add(src=torch.ones_like(copyable_elements_sample_idxs), index=copyable_elements_sample_idxs, dim_size=B * T)
    mask = (valid.reshape(B, T) > 0) & (target_token_ids[:, 1:] == 0)
    gen = torch.gather(target_lp, index=target_token_ids[:, 1:].unsqueeze(-1), dim=-1).squeeze(-1)
    gen.masked_fill_(mask, float("-inf"))
    cp = ts.scatter_logsumexp(src=copy_lp.flatten()[copyable_elements_idxs], index=copyable_elements_sample_idxs, dim=0, dim_size=B * T,
                              eps=0).view(B, T)
    anyc = torch.logsumexp(torch.stack((gen, cp)), dim=0)
    keep = (torch.arange(T, device=target_lengths.device).unsqueeze(0) < target_lengths.unsqueeze(1)).float()
    return -((anyc * keep).sum(dim=-1) / keep.sum(dim=-1)).mean()


def measure(fn, calls):
    """(ms per call by CUDA events, peak MiB above the allocation before one call)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / calls, peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "decoder_time.py measures on a GPU"
    torch.manual_seed(0)
    # dropout 0 in training mode (the identity): cuDNN's GRU runs its backward only in training mode
    m = P.GruCopyingDecoder(V, E, H, H, unk_id=0, dropout_rate=0.0).cuda().train()
    gen = torch.Generator().manual_seed(1)
    origin = torch.repeat_interleave(torch.arange(G), PER).cuda()
    mem = torch.randn(G * PER, H, generator=gen).cuda()
    h0 = (torch.randn(G, H, generator=gen) * 0.5).cuda()
    tokens = torch.randint(0, V, (G, L), generator=gen).cuda()
    g_copy, g_target = torch.randn(G * PER, L, device="cuda"), torch.randn(G, L, V, device="cuda") * 1e-3

    def native_fwd():
        with torch.no_grad():
            return m._compute_logprobs(h0, mem, origin, tokens)

    memg = mem.clone().requires_grad_(True)

    def native_fwd_bwd():
        c, t, _ = m._compute_logprobs(h0, memg, origin, tokens)
        torch.autograd.backward([c, t], [g_copy, g_target])

    def shim_fwd():
        with torch.no_grad():
            return shim_compute_logprobs(m, h0, mem, origin, tokens)

    plan = graph_plan(origin, G)
    with torch.no_grad():
        o, _ = m._GruCopyingDecoder__output_gru(m._GruCopyingDecoder__embedding_layer(tokens), h0.unsqueeze(0))
        o = o.contiguous()
        q = torch.nn.functional.pad(o, (0, 0, 0, 1))
    rows = torch.randn(G * PER, H, device="cuda")

    # the outputs agree before anything is timed
    nat, shim = native_fwd(), shim_fwd()
    agree = {k: float(((a - b).abs() / b.abs().clamp(min=1)).max()) for k, a, b in zip(("copy", "target", "state"), nat, shim)}
    del nat, shim

    res = {"card": card(), "shape": dict(G=G, memories_per_sample=PER, M=G * PER, D=H, H=H, E=E, V=V, L=L), "calls": args.calls,
           "native_vs_shim_max_scaled_diff": agree}
    for name, fn in (("native_forward", native_fwd), ("native_forward_backward", native_fwd_bwd), ("shim_forward", shim_fwd),
                     ("copy_kernel", lambda: native_copy_attention(rows, plan, o)),
                     ("attention_readout_8_heads", lambda: native_attention_readout(rows, plan, q, 8))):
        ms, peak = measure(fn, args.calls)
        res[name] = {"ms": round(ms, 4), "peak_mib": round(peak, 1)}
        print(f"{name:28s} {ms:8.3f} ms   peak +{peak:8.1f} MiB", flush=True)

    # the shim's backward: the loss gives the attention weights and the memories no gradient through its reductions
    pick = torch.rand(G * PER, L, generator=gen) < 0.05
    row, step = torch.nonzero(pick, as_tuple=True)
    ce, ces = (row * L + step).cuda(), (origin.cpu()[row] * L + step).cuda()
    target = torch.cat([tokens, torch.randint(0, V, (G, 1), generator=gen).cuda()], dim=1)
    lengths = torch.randint(2, L + 2, (G,), generator=gen).cuda()
    m.zero_grad()
    memg.grad = None
    shim_loss(m, h0, memg, origin, target, ce, ces, lengths).backward()
    p = "_GruCopyingDecoder__memories_to_"
    res["shim_loss_backward_grad_is_none"] = {n: getattr(m, p + n).weight.grad is None for n in ("standard_attention", "copy_attention")}
    res["shim_loss_backward_grad_is_none"]["memories"] = memg.grad is None
    m.zero_grad()
    memg.grad = None
    m(input_memories=memg, input_memories_origin_idx=origin, initial_states=h0, target_token_ids=target, copyable_elements_idxs=ce,
      copyable_elements_sample_idxs=ces, target_lengths=lengths).backward()
    res["native_loss_backward_grad_is_none"] = {n: getattr(m, p + n).weight.grad is None for n in ("standard_attention", "copy_attention")}
    res["native_loss_backward_grad_is_none"]["memories"] = memg.grad is None
    res["one_MLH_fp32_tensor_mib"] = G * PER * L * H * 4 / 2 ** 20
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
