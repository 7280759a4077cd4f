"""graph2seq decoder on the GPU: the copy kernel against float64 with per-element bounds, the module against the reference's fixtures
and the float64 restatement (decoder_reference.py), gradients against torch.autograd through the restatement, training-mode dropout,
bf16 memories against the reference's autocast fixture, no host synchronisation in the attention pieces, peak memory at the timing
shape, refusals, and two SGD steps of a graph2seq-shaped model.  Every case runs twice and must be bit-identical.

Copy kernel bound (DESIGN.md §3.11 gives the order), u = 2^-24, gamma_k = k u / (1 - k u): a score is a per-lane fmaf chain over
H / 32 features and a five-level butterfly, |ds| <= eps = gamma_{H/32+5} sum_f |c_f o_f|.  lse follows the attention readout's bound
(test_gpu_attention_readout.py) without the weighted sum: with E the graph's largest eps and K = 4 + 5 (CHUNK - 1) + 4 + CHUNK + k +
ceil(max s - min s) for k chunks, |dlse| <= E + gamma_K + 4 u |log L| + u |lse|, 1 % slack."""
import math
import os

import numpy as np
import pytest
import torch

import attention_readout_reference as AR
import decoder_reference as DR
import global_exchange_reference as GX
from helpers import gated_oracle_args
from oracle import ptgnn_oracle as O

pytestmark = pytest.mark.gpu

CHUNK = 32
U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["decoder_h32_l1", "decoder_h32_l4", "decoder_h128_l4", "decoder_h128_l7"]
INPUTS = ("memories", "origin", "initial_states", "target_token_ids", "copyable_elements_idxs", "copyable_elements_sample_idxs",
          "target_lengths")
COUNTS = [1, 0, 31, 32, 33, 64, 65]           # memory rows per sample: a sample without memories (not the last), chunk edges


def gamma(k):
    return k * U / (1 - k * U)


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: torch.from_numpy(z[k]) if z[k].ndim else z[k].item() for k in z.files}


def scaled(a, b):
    return ((a.detach().double().cpu() - b.detach().double().cpu()).abs() / b.detach().double().cpu().abs().clamp(min=1)).max().item()


def grads_close(a, b, what):
    """The bar of test_gpu_backward.py: max error over max(1, max |ref|), and rel. L2, both <= 1e-4."""
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    s = (a - b).abs().max().item() / max(1.0, b.abs().max().item())
    rel = ((a - b).norm() / b.norm().clamp(min=1e-30)).item()
    assert s <= 1e-4 and rel <= 1e-4, f"{what}: scaled {s:.2e} rel L2 {rel:.2e}"


def module(V, E, H, D, seed=0, dropout=0.2):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    return P.GruCopyingDecoder(V, E, H, D, unk_id=0, dropout_rate=dropout).cuda()


def inputs(counts, H, L, D, V, gen):
    """Seeded decoder inputs with the rows of the samples shuffled (unsorted origin), copyable rows at some steps, UNK targets."""
    G = len(counts)
    origin = torch.repeat_interleave(torch.arange(G), torch.tensor(counts))
    origin = origin[torch.randperm(origin.numel(), generator=gen)]
    mem = torch.randn(origin.numel(), D, generator=gen)
    h0 = torch.randn(G, H, generator=gen) * 0.5
    tokens = torch.randint(0, V, (G, L + 1), generator=gen)
    ce, ces = [], []
    for g in range(G):
        rows = torch.nonzero(origin == g).flatten()
        for t in range(L):
            pick = rows[torch.rand(len(rows), generator=gen) < 0.2]
            ce += (pick * L + t).tolist()
            ces += [g * L + t] * len(pick)
    lengths = torch.randint(1, L + 2, (G,), generator=gen)
    return mem, origin, h0, tokens, torch.tensor(ce, dtype=torch.int64), torch.tensor(ces, dtype=torch.int64), lengths


def cuda_all(ts):
    return [t.cuda() for t in ts]


def native_loss_and_grads(m, ins):
    """The loss and its gradients.  cuDNN's GRU runs its backward only in training mode: a module in eval mode is trained here with
    dropout p = 0 (the identity, as eval mode)."""
    mem, origin, h0, tokens, ce, ces, lengths = cuda_all(ins)
    mem, h0 = mem.clone().requires_grad_(True), h0.clone().requires_grad_(True)
    dropout, eval_mode = m._GruCopyingDecoder__dropout, not m.training
    rate = dropout.p
    if eval_mode:
        m.train()
        dropout.p = 0.0
    m.zero_grad()
    try:
        loss = m(input_memories=mem, input_memories_origin_idx=origin, initial_states=h0, target_token_ids=tokens, copyable_elements_idxs=ce,
                 copyable_elements_sample_idxs=ces, target_lengths=lengths)
        loss.backward()
    finally:
        if eval_mode:
            m.eval()
            dropout.p = rate
    return loss.detach(), [mem.grad, h0.grad] + [p.grad for _, p in m.named_parameters()]


def restated_loss_and_grads(m, ins, masks=None):
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in m.named_parameters()}
    mem, origin, h0, tokens, ce, ces, lengths = ins
    mem, h0 = mem.double().requires_grad_(True), h0.double().requires_grad_(True)
    loss = DR.loss(sd, 0, mem, origin, h0, tokens, ce, ces, lengths, masks)
    loss.backward()
    return loss.detach(), [mem.grad, h0.grad] + [sd[n].grad for n, _ in m.named_parameters()]


def check_grads(m, got, ref, what):
    names = ["memories", "initial_states"] + [n for n, _ in m.named_parameters()]
    for n, a, b in zip(names, got, ref):
        grads_close(a, b, f"{what} d {n}")


# ---- the copy kernel ------------------------------------------------------------------------------------------------------------
def copy_ref(c64, origin, G, o64):
    """float64 (s [M, L], lse [G, L], bound_s, bound_lse)."""
    L, H = o64.shape[1], o64.shape[2]
    per_row = o64[origin]
    s = torch.einsum("ih,ilh->il", c64, per_row)
    eps = gamma(H // 32 + 5) * torch.einsum("ih,ilh->il", c64.abs(), per_row.abs())
    idx = origin[:, None].expand(-1, L)
    count = torch.bincount(origin, minlength=G).double()
    M = torch.full((G, L), -math.inf, dtype=torch.float64, device=c64.device).scatter_reduce(0, idx, s, "amax", include_self=True)
    Mn = torch.full((G, L), math.inf, dtype=torch.float64, device=c64.device).scatter_reduce(0, idx, s, "amin", include_self=True)
    has = (count > 0)[:, None]
    Ls = torch.zeros(G, L, dtype=torch.float64, device=c64.device).index_add(0, origin, torch.exp(s - M[origin]))
    lse = torch.where(has, M + torch.log(Ls), torch.full_like(M, -math.inf))
    E = torch.zeros(G, L, dtype=torch.float64, device=c64.device).scatter_reduce(0, idx, eps, "amax", include_self=True)
    K = 4 + 5 * (CHUNK - 1) + 4 + CHUNK + torch.ceil(count / CHUNK)[:, None] + torch.where(has, torch.ceil(M - Mn), torch.zeros_like(M))
    gK = K * U / (1 - K * U)
    logL = torch.where(has, torch.log(Ls), torch.zeros_like(Ls))
    bound_lse = (E + gK + 4 * U * logL.abs() + U * lse.abs().nan_to_num(0, 0, 0)) * 1.01
    return s, lse, eps * 1.01 + 1e-30, bound_lse


@pytest.mark.parametrize("L", [1, 2, 3, 5, 7, 8])
@pytest.mark.parametrize("H", [32, 64, 128, 256])
def test_copy_kernel_against_float64(H, L):
    from ptgnn_b200.decoder import native_copy_attention
    from ptgnn_b200.reduceops import graph_plan

    gen = torch.Generator().manual_seed(H * 10 + L)
    G = len(COUNTS)
    origin = torch.repeat_interleave(torch.arange(G), torch.tensor(COUNTS))
    origin = origin[torch.randperm(origin.numel(), generator=gen)].cuda()
    c = torch.randn(origin.numel(), H, generator=gen).cuda()
    o = (torch.randn(G, L, H, generator=gen) * (4.0 / H ** 0.5)).cuda()
    plan = graph_plan(origin, G)
    s1, lse1 = native_copy_attention(c, plan, o)
    s2, lse2 = native_copy_attention(c, plan, o)
    plan.validate()
    assert torch.equal(s1, s2) and torch.equal(lse1, lse2), "copy attention is not run-to-run bit-identical"
    s, lse, bs, bl = copy_ref(c.double(), origin, G, o.double())
    err = (s1.double() - s).abs()
    assert bool((err <= bs).all()), f"s error / bound {float((err / bs).max()):.3f}"
    fin = torch.isfinite(lse)
    assert bool((lse1[~fin] == -math.inf).all()) and int((~fin).sum()) == L, "the sample without memories gives lse = -inf"
    lerr = (lse1.double()[fin] - lse[fin]).abs()
    assert bool((lerr <= bl[fin]).all()), f"lse error / bound {float((lerr / bl[fin]).max()):.3f}"

    # backward: against the float64 formula at the bar of the gradient checks
    from ptgnn_b200.decoder import native_copy_attention_backward

    d_s = torch.randn(origin.numel(), L, generator=gen).cuda()
    d_lse = torch.randn(G, L, generator=gen).cuda()
    d_lse[~fin] = 0
    d_c1, d_o1 = native_copy_attention_backward(c, plan, o, lse1, d_s, d_lse)
    d_c2, d_o2 = native_copy_attention_backward(c, plan, o, lse1, d_s, d_lse)
    assert torch.equal(d_c1, d_c2) and torch.equal(d_o1, d_o2), "copy attention backward is not run-to-run bit-identical"
    c64, o64 = c.double().requires_grad_(True), o.double().requires_grad_(True)
    s64 = torch.einsum("ih,ilh->il", c64, o64[origin])
    lse64 = DR.segment_logsumexp(s64.cpu(), origin.cpu(), G).cuda()
    ((s64 * d_s.double()).sum() + (lse64[fin] * d_lse.double()[fin]).sum()).backward()
    grads_close(d_c1, c64.grad, f"H={H} L={L} d c")
    grads_close(d_o1, o64.grad, f"H={H} L={L} d o")
    assert bool((d_o1[COUNTS.index(0)] == 0).all()), "the sample without memories gets d o = 0"


# ---- the module -------------------------------------------------------------------------------------------------------------
def from_fixture(f):
    m = module(int(f["vocabulary"]), int(f["embedding"]), int(f["hidden"]), int(f["memories_dim"]))
    m.load_state_dict({k[4:]: v for k, v in f.items() if k.startswith("sd::")})
    return m


@pytest.mark.parametrize("name", NAMES)
def test_forward_matches_reference_fixtures_and_float64(name):
    f = load(name)
    m = from_fixture(f).eval()
    mem, origin, h0, tokens = (f[k] for k in INPUTS[:4])
    with torch.no_grad():
        runs = [m._compute_logprobs(h0.cuda(), mem.cuda(), origin.cuda(), tokens[:, :-1].cuda()) for _ in range(2)]
    assert all(torch.equal(a, b) for a, b in zip(*runs)), "forward is not run-to-run bit-identical"
    sd = {k: v.double().cpu() for k, v in m.state_dict().items()}
    with torch.no_grad():
        ref = DR.compute_logprobs(sd, h0.double(), mem.double(), origin, tokens[:, :-1])
    for got, r, key in zip(runs[0], ref, ("copy_logprobs", "target_logprobs", "gru_state")):
        assert scaled(got, f[key]) <= 1e-5, f"{name} {key} vs the reference: {scaled(got, f[key]):.2e}"
        assert scaled(got, r) <= 1e-5, f"{name} {key} vs float64: {scaled(got, r):.2e}"


@pytest.mark.parametrize("name", NAMES)
def test_gradients_match_reference_fixtures_and_float64(name):
    f = load(name)
    m = from_fixture(f).eval()
    ins = [f[k] for k in INPUTS]
    loss, got = native_loss_and_grads(m, ins)
    loss2, again = native_loss_and_grads(m, ins)
    assert torch.equal(loss, loss2) and all(torch.equal(a, b) for a, b in zip(got, again)), "gradients are not run-to-run bit-identical"
    assert abs(loss.item() - float(f["loss"])) <= 1e-5 * max(1.0, abs(float(f["loss"])))
    names = ["memories", "initial_states"] + [n for n, _ in m.named_parameters()]
    for n, g in zip(names, got):
        grads_close(g, f["grad::" + n], f"{name} d {n} vs the reference")
    ref_loss, ref = restated_loss_and_grads(m, ins)
    assert abs(loss.item() - ref_loss.item()) <= 1e-5 * max(1.0, abs(ref_loss.item()))
    check_grads(m, got, ref, f"{name} vs float64")


@pytest.mark.parametrize("L", [1, 2, 3, 5, 7, 8])
@pytest.mark.parametrize("H", [32, 64, 128, 256])
def test_module_structural_edges(H, L):
    """Memory counts 0 / 1 / 31 / 32 / 33 / 64 / 65 in an unsorted origin map, every step count the kernels take, every hidden size."""
    gen = torch.Generator().manual_seed(100 * H + L)
    D, E, V = 48, 32, 40
    m = module(V, E, H, D, seed=H + L).eval()
    ins = inputs(COUNTS, H, L, D, V, gen)
    mem, origin, h0, tokens = ins[:4]
    with torch.no_grad():
        got = m._compute_logprobs(h0.cuda(), mem.cuda(), origin.cuda(), tokens[:, :-1].cuda())
        ref = DR.compute_logprobs({k: v.double().cpu() for k, v in m.state_dict().items()}, h0.double(), mem.double(), origin,
                                  tokens[:, :-1])
    for a, b, key in zip(got, ref, ("copy_logprobs", "target_logprobs", "gru_state")):
        assert scaled(a, b) <= 1e-5, f"H={H} L={L} {key}: {scaled(a, b):.2e}"
    loss, grads = native_loss_and_grads(m, ins)
    ref_loss, ref_grads = restated_loss_and_grads(m, ins)
    assert abs(loss.item() - ref_loss.item()) <= 1e-5 * max(1.0, abs(ref_loss.item()))
    check_grads(m, grads, ref_grads, f"H={H} L={L}")


def test_training_mode_dropout_masks_reproduced_by_reseeding():
    import torch.nn.functional as F

    gen = torch.Generator().manual_seed(9)
    H, L, D, E, V, p = 64, 7, 48, 32, 40, 0.2
    m = module(V, E, H, D, seed=9, dropout=p).train()
    ins = inputs(COUNTS, H, L, D, V, gen)
    torch.manual_seed(123)
    loss, got = native_loss_and_grads(m, ins)
    # the four masks in the reference's order: token embeddings, copy representations, standard attention output, embedding weight
    torch.manual_seed(123)
    G, M = len(COUNTS), ins[0].shape[0]
    masks = [F.dropout(torch.ones(shape, device="cuda"), p, True).cpu().double() for shape in ((G, L, E), (M, H), (G, L, H), (V, E))]
    assert all(0 < int((mk == 0).sum()) < mk.numel() for mk in masks)
    ref_loss, ref = restated_loss_and_grads(m, ins, masks)
    assert abs(loss.item() - ref_loss.item()) <= 1e-5 * max(1.0, abs(ref_loss.item())), (loss.item(), ref_loss.item())
    check_grads(m, got, ref, "dropout 0.2")


def test_bf16_memories_vs_reference_autocast():
    """DESIGN §4 bf16 rule: rel. L2 <= 1e-2 against the reference's autocast output, and at least as close to the fp32 result as the
    reference's autocast path is."""
    f = load("decoder_h128_l7_bf16ac")
    m = from_fixture(f).eval()
    mem, origin, h0, tokens = (f[k] for k in INPUTS[:4])
    with torch.no_grad():
        runs = [m._compute_logprobs(h0.cuda(), mem.to(torch.bfloat16).cuda(), origin.cuda(), tokens[:, :-1].cuda()) for _ in range(2)]
    assert all(torch.equal(a, b) for a, b in zip(*runs)) and runs[0][0].dtype == torch.float32
    got = torch.cat([runs[0][0].flatten(), runs[0][1].flatten()]).cpu()
    ref_ac = torch.cat([f["copy_autocast"].flatten(), f["target_autocast"].flatten()])
    ref32 = torch.cat([f["copy_fp32_rounded_inputs"].flatten(), f["target_fp32_rounded_inputs"].flatten()])
    scale = ref32.abs().clamp(min=1)
    err_ours, err_ref = (got - ref32).abs(), (ref_ac - ref32).abs()
    frac_ours, frac_ref = (err_ours <= 1e-2 * scale).float().mean().item(), (err_ref <= 1e-2 * scale).float().mean().item()
    rel_ac = ((got - ref_ac).norm() / ref_ac.norm()).item()
    msg = f"rel L2 vs autocast {rel_ac:.2e}; mean err ours {err_ours.mean():.2e} / ref {err_ref.mean():.2e}; within 1e-2 {frac_ours:.4f} / {frac_ref:.4f}"
    assert rel_ac <= 1e-2 and err_ours.mean().item() <= 1.1 * err_ref.mean().item() and frac_ours >= frac_ref - 0.002, msg


def test_unsupported_shapes_raise():
    m = module(40, 32, 64, 48)
    origin = torch.zeros(10, dtype=torch.int64).cuda()
    mem, h0 = torch.randn(10, 48).cuda(), torch.randn(2, 64).cuda()
    origin[5:] = 1
    with torch.no_grad(), pytest.raises(NotImplementedError):
        m._compute_logprobs(h0, mem, origin, torch.zeros(2, 9, dtype=torch.int64).cuda())        # L = 9
    with pytest.raises(NotImplementedError):
        m._compute_logprobs(h0, mem.to(torch.bfloat16).requires_grad_(True), origin, torch.zeros(2, 7, dtype=torch.int64).cuda())
    odd = module(40, 32, 48, 48)
    with torch.no_grad(), pytest.raises(NotImplementedError):
        odd._compute_logprobs(torch.randn(2, 48).cuda(), mem, origin, torch.zeros(2, 7, dtype=torch.int64).cuda())   # H = 48


def test_attention_pieces_make_no_host_synchronisation():
    from ptgnn_b200 import autograd as AG
    from ptgnn_b200.decoder import native_copy_attention
    from ptgnn_b200.reduceops import graph_plan, native_attention_readout

    gen = torch.Generator().manual_seed(5)
    G, L, H = 80, 7, 128
    origin = torch.randint(0, G, (20_000,), generator=gen).cuda()
    a, c = torch.randn(20_000, H, device="cuda", requires_grad=True), torch.randn(20_000, H, device="cuda", requires_grad=True)
    o = torch.randn(G, L, H, device="cuda", requires_grad=True)

    def pieces(grad):
        plan = graph_plan(origin, G)
        q = torch.nn.functional.pad(o, (0, 0, 0, 1))
        if grad:
            ctx = AG.attention_readout_with_grad(plan, 8, a, q)[:, :L]
            s, lse = AG.copy_attention_with_grad(plan, c, o)
            plan.poll()
            (ctx.sum() + s.sum() + lse.sum()).backward()
        else:
            native_attention_readout(a.detach(), plan, q.detach(), 8)
            native_copy_attention(c.detach(), plan, o.detach())
            plan.poll()

    for grad in (False, True):
        pieces(grad)                                                  # warm: plan cache
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            pieces(grad)
        finally:
            torch.cuda.set_sync_debug_mode("default")


def test_peak_memory_at_timing_shape():
    """G = 80 samples of 640 memories, D = H = 128, E = 256, V = 20,000, L = 7: the forward's peak-memory rise stays below one
    [M, L, H] fp32 tensor (the reference's gathered decoder states alone are one, and its einsum / exp / scatter chain makes more)."""
    G, per, H, L, E, V = 80, 640, 128, 7, 256, 20_000
    m = module(V, E, H, H).eval()
    origin = torch.repeat_interleave(torch.arange(G), per).cuda()
    mem, h0 = torch.randn(G * per, H, device="cuda"), torch.randn(G, H, device="cuda")
    tokens = torch.randint(0, V, (G, L), device="cuda")
    with torch.no_grad():
        out = m._compute_logprobs(h0, mem, origin, tokens)
        del out
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = m._compute_logprobs(h0, mem, origin, tokens)
        torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    one = G * per * L * H * 4
    assert rise < one, f"peak rise {rise / 2**20:.1f} MiB >= one [M, L, H] fp32 tensor ({one / 2**20:.1f} MiB)"


def test_graph2seq_shaped_model_two_sgd_steps_match_cpu():
    """graph2seq (graph2seq.py): gated layers at H = 128, the native 8-head summary of the concatenated input and output states as the
    decoder's initial states, the output states of a subset of the nodes as its memories, and the native decoder's loss; two SGD
    steps against the same steps in float64 on the CPU.  Both attention weights receive gradients."""
    import ptgnn_b200 as P

    N, Hn, T, G, L, E, V = 2000, 128, 2, 8, 7, 64, 100
    gen = torch.Generator().manual_seed(71)
    adj = [(torch.randint(0, N, (c,), generator=gen), torch.randint(0, N, (c,), generator=gen)) for c in (2 * N, N)]
    n2g = torch.sort(torch.randint(0, G, (N,), generator=gen)).values
    backbone = torch.sort(torch.randperm(N, generator=gen)[:500]).values
    origin = n2g[backbone]
    h0 = torch.randn(N, Hn, generator=gen) * 0.5
    tokens = torch.randint(0, V, (G, L + 1), generator=gen)
    ce, ces = [], []
    for g in range(G):
        rows = torch.nonzero(origin == g).flatten()
        for t in range(L):
            pick = rows[torch.rand(len(rows), generator=gen) < 0.05]
            ce += (pick * L + t).tolist()
            ces += [g * L + t] * len(pick)
    ce, ces = torch.tensor(ce, dtype=torch.int64), torch.tensor(ces, dtype=torch.int64)
    lengths = torch.randint(2, L + 2, (G,), generator=gen)
    torch.manual_seed(72)
    layers = [P.GatedMessagePassingLayer(Hn, Hn, T, "sum").cuda(), P.GatedMessagePassingLayer(Hn, Hn, T, "sum").cuda()]
    reducer = P.MultiheadSelfAttentionVarSizedElementReduce(2 * Hn, 2 * Hn, Hn, 8, P.SimpleVarSizedElementReduce("max")).cuda()
    decoder = P.GruCopyingDecoder(V, E, Hn, Hn, unk_id=0, dropout_rate=0.0).cuda().train()      # cuDNN's GRU backward: training mode
    modules = layers + [reducer, decoder]
    params = [p for mod in modules for p in mod.parameters()]
    ref_params = [p.detach().cpu().double().clone().requires_grad_(True) for p in params]
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    opt = torch.optim.SGD(params, lr=0.05)
    for step in range(2):
        opt.zero_grad()
        h = h0.cuda()
        for layer in layers:
            h = layer(h, adj_d)
        summary = reducer(P.ElementsToSummaryRepresentationInput(torch.cat((h0.cuda(), h), dim=-1), n2g.cuda(), G))
        loss = decoder(input_memories=h[backbone.cuda()], input_memories_origin_idx=origin.cuda(), initial_states=summary,
                       target_token_ids=tokens.cuda(), copyable_elements_idxs=ce.cuda(), copyable_elements_sample_idxs=ces.cuda(),
                       target_lengths=lengths.cuda())
        loss.backward()
        if step == 0:
            named = dict(decoder.named_parameters())
            for n in ("_GruCopyingDecoder__memories_to_standard_attention.weight", "_GruCopyingDecoder__memories_to_copy_attention.weight"):
                assert named[n].grad is not None and float(named[n].grad.abs().sum()) > 0, f"{n} receives no gradient"
        opt.step()

    def run_cpu():
        it = iter(ref_params)
        h = h0.double()
        for layer in layers:
            names = {n: next(it) for n, _ in layer.named_parameters()}
            h = O.gated_layer_forward(h, adj, [torch.empty(s.shape[0], 0, dtype=torch.float64) for s, _ in adj], aggregation_fn="sum",
                                      **gated_oracle_args(names))
        rp = {n: next(it) for n, _ in reducer.named_parameters()}
        p = "_MultiheadSelfAttentionVarSizedElementReduce__"
        x = torch.cat((h0.double(), h), dim=-1)
        summary = AR.multihead_self_attention_forward(x, n2g, G, GX.graph_readout(x, n2g, G, "max"), rp[p + "key_layer.weight"], 8,
                                                      rp[p + "output_layer.weight"])
        dp = {n: next(it) for n, _ in decoder.named_parameters()}
        return DR.loss(dp, 0, h[backbone], origin, summary, tokens, ce, ces, lengths)

    ref_opt = torch.optim.SGD(ref_params, lr=0.05)
    for _ in range(2):
        ref_opt.zero_grad()
        run_cpu().backward()
        ref_opt.step()
    for p, r in zip(params, ref_params):
        grads_close(p, r, "parameters after two SGD steps")
