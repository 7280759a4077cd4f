"""MlpMessagePassingLayer training with bf16 node states: the gathered bf16 weight-gradient kernel (csrc/wgrad.cu) element by element
against float64, the layer's gradients against float64 autograd of its restatement on the bf16-rounded inputs, determinism, a short
training run against fp32, and the refusals outside the supported configurations."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

GRAD_SCALES = (1.0, 2.0 ** -17, 2.0 ** -27, 2.0 ** -37, 2.0 ** 17)     # tests/test_gpu_backward_edges.py: what training produces


def _graph(counts, num_nodes, seed):
    gen = torch.Generator().manual_seed(seed)
    return [(torch.randint(0, num_nodes, (n,), generator=gen).cuda(), torch.randint(0, num_nodes, (n,), generator=gen).cuda()) for n in counts]


def _chunk_edges(E, D, C):
    """The kernel's split-K chunk length (csrc/wgrad.cu chunk_edges_for)."""
    tiles = math.ceil(D / 64) * math.ceil(C / 64)
    chunks = math.ceil(132 * 8 / tiles)
    return max(4 * 64, math.ceil(math.ceil(max(E, 1) / chunks) / 64) * 64)


# ---- the weight-gradient kernel ----------------------------------------------------------------------------------------
WGRAD_CASES = [   # (H, D, per-type edge counts): ragged counts with 0, 1, around the 64-edge stage and the chunk length
    (64, 64, [0, 1, 63, 65, 255, 256, 257, 1000]),
    (128, 128, [1, 0, 511, 512, 513, 3000]),
    (96, 80, [7, 300, 0, 129]),
    (256, 128, [2000, 1, 0]),
    (128, 128, [60_000, 41_001, 0, 3]),          # chunks longer than the minimum
]


@pytest.mark.parametrize("H,D,counts", WGRAD_CASES)
@pytest.mark.parametrize("use_target", [False, True])
@pytest.mark.parametrize("by_target", [True, False])
def test_weight_grad_kernel_per_element(H, D, counts, use_target, by_target):
    """got[t, i, j] against ref = sum_e g_e,i x_e,j in float64, x_e the bf16 states and g_e the gradient rows, bf16 values times a power
    of two here so that the operands the kernel sees are exact.  Bound: c 2^-8 sum_e |g_e,i| |x_e,j| with c = 0 for these exact
    operands (the bf16 rounding of an fp32 g_e s contributes 2^-9 |g| |x| per product, c = 1 with a factor 2 of margin; the layer
    tests cover it), plus the fp32 accumulation: products of bf16 values are exact in fp32, each of the n_e / 16 MMA steps and each of
    the n_chunks partial additions rounds once (at most 2^-24 of the running sum, 2^-23 if the tensor core truncates), with 16 more
    steps and a factor 2 of margin: 4 (n_e / 16 + n_chunks + 16) 2^-24 sum |g| |x|.  A mutant without the first chunk of a type must
    break the bound: the split-K partials are all needed."""
    from ptgnn_b200 import autograd as AG
    from ptgnn_b200.edgeplan import plan_for

    num_nodes = 3000
    adj = _graph(counts, num_nodes, seed=H + D + len(counts))
    plan = plan_for(adj, num_nodes)
    gen = torch.Generator().manual_seed(7)
    h = torch.randn(num_nodes, H, generator=gen).to(torch.bfloat16).cuda()
    rows = num_nodes if by_target else plan.num_edges
    g = torch.randn(rows, D, generator=gen).to(torch.bfloat16).float().cuda() * 2.0 ** -25      # gradient magnitudes of a mean loss
    g[::7] *= 2.0 ** 10
    scale, inv = AG._pow2_scale(g)
    got = AG._weight_grad_bf16(plan, (g * scale).to(torch.bfloat16), plan.tgt32 if by_target else None, inv, h, use_target).cpu().double()
    C = (2 if use_target else 1) * H
    L = _chunk_edges(plan.num_edges, D, C)
    hd, gd = h.double().cpu(), g.double().cpu()
    checked = 0
    for t, (src, tgt) in enumerate(adj):
        x = hd[src.cpu()] if not use_target else torch.cat([hd[src.cpu()], hd[tgt.cpu()]], dim=1)
        ge = gd[tgt.cpu()] if by_target else gd[plan.type_off[t]:plan.type_off[t + 1]]
        ref = ge.t() @ x
        mag = ge.abs().t() @ x.abs()
        n = x.shape[0]
        bound = 4 * (n / 16 + math.ceil(n / L) + 16) * 2.0 ** -24 * mag + 1e-45
        err = (got[t] - ref).abs()
        assert bool((err <= bound).all()), f"type {t} ({n} edges): worst err/bound {float((err / bound).max()):.3g}"
        if n == 0:
            assert bool((got[t] == 0).all())
        if n > L:      # the mutant without the first chunk
            mutant = ge[L:].t() @ x[L:]
            assert not bool(((mutant - ref).abs() <= bound).all()), f"type {t}: dropping a chunk passes the bound"
        checked += n
    assert checked == plan.num_edges


def test_weight_grad_kernel_is_deterministic():
    from ptgnn_b200 import autograd as AG
    from ptgnn_b200.edgeplan import plan_for

    adj = _graph([50_000, 20_001, 0, 999], 20_000, seed=3)
    plan = plan_for(adj, 20_000)
    h = torch.randn(20_000, 128, device="cuda").to(torch.bfloat16)
    g = torch.randn(20_000, 128, device="cuda").to(torch.bfloat16)
    one = torch.ones((), device="cuda")
    a = AG._weight_grad_bf16(plan, g, plan.tgt32, one, h, True)
    b = AG._weight_grad_bf16(plan, g, plan.tgt32, one, h, True)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- the layer -----------------------------------------------------------------------------------------------------------
def _layer(H, D, T, reduce, use_target, seed=0):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    layer = P.MlpMessagePassingLayer(H, H, D, T, reduce, use_target_state_as_message_input=use_target).cuda().train()
    with torch.no_grad():      # a LayerNorm that is not the identity
        for p in layer.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.1)
    return layer


def _reference(layer, h64, adj, reduce, use_target, G):
    """float64 autograd of mlpmessagepassing.py:68-117 (default message MLP, no dropout) on h64 as the bf16 forward evaluates it: edge
    weights rounded to bf16, messages rounded to bf16 (straight through for the gradient), so that max / min pick the same winners.
    Returns d h and the parameter grads."""
    import torch.nn.functional as F

    params = {n: p.detach().double().cpu().requires_grad_(True) for n, p in layer.named_parameters()}
    names = list(params)
    w_names = [n for n in names if "edge_message_transformation_layers" in n]
    ln_w, ln_b, d_w, d_b = [params[n] for n in names if "state_update" in n]
    x = h64.clone().requires_grad_(True)
    msgs, tgts = [], []
    for (src, tgt), wn in zip(adj, w_names):
        inp = x[src.cpu()] if not use_target else torch.cat([x[src.cpu()], x[tgt.cpu()]], dim=1)
        m = inp @ (params[wn] + (params[wn].to(torch.bfloat16).double() - params[wn]).detach()).t()
        msgs.append(m + (m.to(torch.bfloat16).double() - m).detach())
        tgts.append(tgt.cpu())
    m, tg = torch.cat(msgs), torch.cat(tgts)
    n, D = x.shape[0], m.shape[1]
    if reduce in ("sum", "mean"):
        agg = torch.zeros(n, D, dtype=torch.float64).index_add(0, tg, m)
        if reduce == "mean":
            agg = agg / torch.bincount(tg, minlength=n).clamp(min=1)[:, None]
    else:
        # torch_scatter's rule, which the kernels follow: the first of tied messages wins and takes the whole gradient
        E, idx = m.shape[0], tg[:, None].expand(-1, D)
        best = torch.full((n, D), -math.inf if reduce == "max" else math.inf, dtype=torch.float64)
        best = best.scatter_reduce(0, idx, m.detach(), reduce="amax" if reduce == "max" else "amin", include_self=True)
        cand = torch.where(m.detach() == best[tg], torch.arange(E)[:, None].expand(-1, D), E)
        arg = torch.full((n, D), E).scatter_reduce(0, idx, cand, reduce="amin", include_self=True)
        agg = torch.cat([m, torch.zeros(1, D, dtype=torch.float64)]).gather(0, arg)
    y = torch.tanh(F.linear(F.layer_norm(F.gelu(agg), (D,), ln_w, ln_b, 1e-5), d_w, d_b))
    grads = torch.autograd.grad(y, [x] + [params[k] for k in names], G.double().cpu())
    return grads[0], dict(zip(names, grads[1:]))


def _check(got, ref, s, what):
    """SURVEY.md §8c's bf16 criterion on the gradients divided by max |ref| (the criterion is written for values of order one, and the
    gradient scale s cancels): rel L2 <= 1e-2, 99.9 % within 1e-2 max(1, |ref|)."""
    norm = ref.double().abs().max().clamp(min=1e-300)
    got, ref = got.detach().double().cpu() / norm, ref.double() / norm
    rel_l2 = float((got - ref).norm() / ref.norm().clamp(min=1e-300))
    within = float((((got - ref).abs() / ref.abs().clamp(min=1.0)) <= 1e-2).double().mean())
    assert rel_l2 <= 1e-2 and within >= 0.999, f"{what}: rel L2 {rel_l2:.3e}, within {within:.5f}"
    return rel_l2


LAYER_CASES = [      # (H, D): fused forward and transposed aggregation / fused forward, three-kernel transposed / three-kernel forward
    (128, 128), (64, 128), (128, 64),
]


@pytest.mark.parametrize("H,D", LAYER_CASES)
@pytest.mark.parametrize("reduce", ["sum", "mean", "max", "min"])
@pytest.mark.parametrize("use_target", [True, False])
def test_layer_gradients_against_float64(H, D, reduce, use_target):
    from ptgnn_b200.messagepassing import _use_fused
    from ptgnn_b200 import _native as N

    num_nodes = 2000
    adj = _graph([4000, 0, 1, 2500, 777], num_nodes, seed=H * 3 + D)
    layer = _layer(H, D, len(adj), reduce, use_target)
    assert _use_fused(N.lib(), True, H, D) == (D == 128)
    h = torch.randn(num_nodes, H, device="cuda").to(torch.bfloat16)
    G1 = torch.randn(num_nodes, H, device="cuda")
    ref_h = ref_p = None
    for s in GRAD_SCALES if (H, D) == (128, 128) else (1.0,):
        x = h.clone().requires_grad_(True)
        layer.zero_grad(set_to_none=True)
        out = layer(x, adj)
        assert out.dtype == torch.bfloat16
        out.backward(G1.to(torch.bfloat16) * s)          # s a power of two: exact in bf16
        assert x.grad.dtype == torch.bfloat16
        if ref_h is None:
            ref_h, ref_p = _reference(layer, h.double().cpu(), adj, reduce, use_target, G1.to(torch.bfloat16))
        _check(x.grad, ref_h * s, s, f"d h (s={s})")
        for name, p in layer.named_parameters():
            assert p.grad.dtype == torch.float32
            _check(p.grad, ref_p[name] * s, s, f"d {name} (s={s})")


@pytest.mark.parametrize("reduce", ["max", "min"])
@pytest.mark.parametrize("H,D", [(128, 128), (64, 64)])
def test_max_min_recompute_matches_the_forward_bit_for_bit(reduce, H, D):
    """The backward re-computes max / min from the bf16 messages of the three-kernel path; the forward's aggregate (fused kernel or
    three-kernel path) must be the same bits, or the tail would be differentiated at another point."""
    from ptgnn_b200 import _native as N
    from ptgnn_b200 import composed as C
    from ptgnn_b200.edgeplan import plan_for

    num_nodes = 5000
    adj = _graph([30_000, 0, 7, 12_345], num_nodes, seed=11)
    plan = plan_for(adj, num_nodes)
    torch.manual_seed(1)
    W = [torch.randn(D, 2 * H, device="cuda") / math.sqrt(2 * H) for _ in adj]
    h = torch.randn(num_nodes, H, device="cuda").to(torch.bfloat16)
    msg = C.edge_messages(plan, h, h, W, True)
    agg, _arg = C.segment_reduce(msg, plan, N.REDUCE[reduce], return_arg=True)
    forward = C.aggregate(plan, h, W, N.REDUCE[reduce], True)
    assert torch.equal(agg.view(torch.int32), forward.view(torch.int32))


def test_layer_backward_is_deterministic():
    adj = _graph([20_000, 5_000, 3], 4000, seed=5)
    for reduce in ("sum", "max"):
        layer = _layer(128, 128, len(adj), reduce, True)
        h = torch.randn(4000, 128, device="cuda").to(torch.bfloat16)
        G = torch.randn(4000, 128, device="cuda").to(torch.bfloat16)
        grads = []
        for _ in range(2):
            x = h.clone().requires_grad_(True)
            layer.zero_grad(set_to_none=True)
            layer(x, adj).backward(G)
            grads.append([x.grad.clone()] + [p.grad.clone() for p in layer.parameters()])
        for a, b in zip(*grads):
            assert torch.equal(a, b)


def test_container_trains_in_bf16_like_fp32():
    """Three Mlp layers as the Typilus factory builds them (max aggregation, output dropout 0.1, H = D = 64) in a GraphNeuralNetwork,
    trained for 300 Adam steps to regress fixed targets from fixed inputs, from the same seed in bf16 and fp32.  Band: every bf16 loss
    within 0.1 x the first fp32 loss of the fp32 loss at the same step, and both curves fall below half their start."""
    import ptgnn_b200 as P
    from ptgnn_b200.synthetic import block_diagonal_batch

    b = block_diagonal_batch(8, 250, 8 * 600, (0.5, 0.3, 0.2), seed=3)
    raw = [(s.cuda(), t.cuda()) for s, t in b.adjacency_lists]
    gen = torch.Generator().manual_seed(0)
    h0 = torch.randn(b.num_nodes, 64, generator=gen).cuda()
    target = torch.tanh(torch.randn(b.num_nodes, 64, generator=gen)).cuda()
    curves = {}
    for dtype in (torch.float32, torch.bfloat16):
        torch.manual_seed(0)
        T = 2 * len(raw) + 1
        layers = [P.MlpMessagePassingLayer(64, 64, 64, T, "max", dropout_rate=0.1) for _ in range(3)]
        gnn = P.GraphNeuralNetwork(layers, torch.nn.Identity(), True, True).cuda().train()
        opt = torch.optim.Adam(gnn.parameters(), lr=1e-3)
        adj = gnn.expand_adjacency(raw, b.num_nodes, "cuda")
        losses = []
        for _ in range(300):
            opt.zero_grad(set_to_none=True)
            out = gnn.gnn(h0.to(dtype), adj, None, None, {}, {})
            out = out[-1] if isinstance(out, (list, tuple)) else out
            loss = torch.nn.functional.mse_loss(out.float(), target)
            loss.backward()
            opt.step()
            losses.append(float(loss))
        curves[dtype] = losses
    f32, bf = curves[torch.float32], curves[torch.bfloat16]
    print("\nstep  fp32 loss  bf16 loss")
    for i in list(range(0, 300, 25)) + [299]:
        print(f"{i:4d}  {f32[i]:.5f}    {bf[i]:.5f}")
    band = 0.1 * f32[0]
    worst = max(abs(a - c) for a, c in zip(f32, bf))
    assert worst <= band, f"bf16 loss leaves the band: max |bf16 - fp32| = {worst:.4f} > {band:.4f}"
    assert f32[-1] < 0.5 * f32[0] and bf[-1] < 0.5 * bf[0]


# ---- refusals ------------------------------------------------------------------------------------------------------------
def test_out_of_scope_bf16_training_refuses_before_any_launch():
    import ptgnn_b200 as P
    from ptgnn_b200 import _native as N

    adj = _graph([100, 50], 64, seed=1)
    h = torch.randn(64, 128, device="cuda").to(torch.bfloat16).requires_grad_(True)
    h32 = torch.randn(64, 32, device="cuda").to(torch.bfloat16).requires_grad_(True)
    cases = [
        (P.MlpMessagePassingLayer(128, 128, 128, 2, "sum", mlp_hidden_layers=1).cuda(), h),
        (P.MlpMessagePassingLayer(128, 128, 128, 2, P.PnaMessageAggregation()).cuda(), h),
        (P.MlpMessagePassingLayer(32, 32, 32, 2, "sum").cuda(), h32),
        (P.GatedMessagePassingLayer(128, 128, 2, "sum").cuda(), h),
    ]
    torch.cuda.synchronize()
    for layer, x in cases:
        launches = N.launch_count()
        with pytest.raises(NotImplementedError):
            layer(x, adj)
        assert N.launch_count() == launches
    gsrc = torch.randn(64, 128, device="cuda").to(torch.bfloat16)
    launches = N.launch_count()
    with pytest.raises(NotImplementedError):      # sharded
        P.MlpMessagePassingLayer(128, 128, 128, 2, "sum").cuda()(h, adj, gather_states=gsrc)
    assert N.launch_count() == launches
