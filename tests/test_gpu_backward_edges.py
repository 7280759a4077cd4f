"""The fp32 layer backward passes at the gradient magnitudes training produces, against float64 (``backward_reference``).

Stage tests call the native steps of ``ptgnn_b200/autograd.py`` directly and check every element: the gather-split bit for bit,
the GRU gate derivatives, the split-fp16 weight-gradient GEMMs and the transposed aggregation within their derived bounds.  Layer
tests scale the upstream gradient by s (a mean loss over 204,800 x 128 outputs gives 3.8e-8 per element) and compare d node_states
and every parameter gradient with float64 autograd of the layer's restatement, on a bar that does not depend on magnitude:
max|err| / max|ref| and the relative L2 error under TAU, and err(s) / s no worse than twice err(1)."""
import functools
import math

import pytest
import torch

import backward_reference as BR
import egc_reference as E
import fused_reference as FR
import unfused_reference as UR

pytestmark = pytest.mark.gpu

GRAD_SCALES = (1.0, 2.0 ** -17, 2.0 ** -27, 2.0 ** -37, 2.0 ** 17)
TAU = 5e-5          # ~5x the largest max|err| / max|ref| measured at s = 1 on an H100 (1.1e-5, the 100k-edge gated case)
WORST = {}          # family -> largest error / bound ratio (stages) or max|err| / max|ref| at s = 1 (layers); printed with -s


def _record(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)


def _lib():
    from ptgnn_b200 import _native as N

    return N


# ---- gather_split ------------------------------------------------------------------------------------------------------
def _split_values(rows, cols, seed):
    gen = torch.Generator().manual_seed(seed)
    mag = torch.exp(torch.empty(rows, cols).uniform_(math.log(1e-30), math.log(6e4), generator=gen))
    sign = torch.where(torch.rand(rows, cols, generator=gen) < 0.5, -1.0, 1.0)
    x = (sign * mag).float()
    flat = x.view(-1)
    k = min(flat.numel(), 16)
    flat[:k] = torch.tensor([0.0, -0.0, 6e4, -6e4, 6.1e-5, 5.9e-8, -3e-8, 2.0 ** -24, 2.0 ** -25, 1e-30, 65519.0, 65520.0, 1.0, -1.0,
                             2049.0, 1e-7])[:k]
    return x


def _bits(t):
    return t.contiguous().view(torch.int16).cpu()


@pytest.mark.parametrize("cols", [8, 64, 128, 136, 384, 36, 100])
@pytest.mark.parametrize("indexed", [False, True])
def test_gather_split_bit_exact(cols, indexed):
    from ptgnn_b200 import autograd as AG

    N = _lib()
    rows = 300
    x = _split_values(rows, cols, seed=cols).cuda()
    idx = None
    if indexed:
        g = torch.Generator().manual_seed(1)
        idx = torch.cat([torch.randint(0, rows, (400,), generator=g), torch.tensor([0, 0, rows - 1, rows - 1])]).to(torch.int32).cuda()
    # the backward's own entry point (its scale from the device, the torch split for cols % 8 != 0)
    hi, lo, inv = AG._split16(x, index=idx)
    scale = 1.0 / float(inv)
    assert scale == BR.pow2_scale(x.cpu())
    e_hi, e_lo = BR.gather_split(x, idx, scale)
    assert torch.equal(_bits(hi), _bits(e_hi)) and torch.equal(_bits(lo), _bits(e_lo))
    if cols % 8:
        return
    # the native pass with no scale and with device scalars (2^3 sends 6e4 past fp16's range: hi = inf, lo = -inf)
    for s in (None, 2.0 ** -6, 2.0 ** 3):
        n_out = rows if idx is None else idx.shape[0]
        hi = torch.empty(n_out, cols, dtype=torch.float16, device="cuda")
        lo = torch.empty_like(hi)
        sd = None if s is None else torch.tensor(s, dtype=torch.float32, device="cuda")
        rc = N.lib().ptgnn_b200_gather_split_f16(N.ptr(x), N.ptr(idx), n_out, cols, N.ptr(sd), N.ptr(hi), N.ptr(lo), N.current_stream(x.device))
        N.check(rc, "ptgnn_b200_gather_split_f16")
        e_hi, e_lo = BR.gather_split(x, idx, s)
        assert torch.equal(_bits(hi), _bits(e_hi)) and torch.equal(_bits(lo), _bits(e_lo)), f"scale {s}"


def test_gather_split_empty_and_past_the_grid_stride_cap():
    from ptgnn_b200 import autograd as AG

    hi, lo, inv = AG._split16(torch.empty(0, 128, device="cuda"))
    assert hi.shape == (0, 128) and lo.shape == (0, 128)
    x = _split_values(70_000, 128, seed=3).cuda()        # 70,000 * 16 float8 groups > 132 * 16 blocks * 256 threads
    idx = torch.randint(0, 70_000, (70_000,), generator=torch.Generator().manual_seed(2)).to(torch.int32).cuda()
    for index in (None, idx):
        hi, lo, inv = AG._split16(x, index=index)
        e_hi, e_lo = BR.gather_split(x, index, 1.0 / float(inv))
        assert torch.equal(_bits(hi), _bits(e_hi)) and torch.equal(_bits(lo), _bits(e_lo))


# ---- gru_gate_grads ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [4, 36, 64, 128, 256])
@pytest.mark.parametrize("rows", [1, 63, 64, 65, 20_000])
def test_gru_gate_grads_per_element(H, rows):
    N = _lib()
    gen = torch.Generator().manual_seed(H * 7 + rows)
    row_scale = torch.tensor([0.3, 3.0, 15.0])[torch.randint(0, 3, (rows, 1), generator=gen)]
    gi = (torch.randn(rows, 3 * H, generator=gen) * row_scale).clamp(-15, 15)
    gh = (torch.randn(rows, 3 * H, generator=gen) * row_scale).clamp(-15, 15)     # gate pre-activations up to +-30
    h = torch.randn(rows, H, generator=gen)
    g1 = torch.randn(rows, H, generator=gen)
    d = [t.cuda() for t in (gi, gh, h)]
    for gs in (1.0, 2.0 ** -30, 2.0 ** 20):
        g = (g1 * gs).cuda()
        d_gi, d_gh, d_h = torch.empty_like(d[0]), torch.empty_like(d[1]), torch.empty_like(d[2])
        rc = N.lib().ptgnn_b200_gru_gate_grads_f32(N.ptr(d[0]), N.ptr(d[1]), N.ptr(d[2]), N.ptr(g), rows, H, N.ptr(d_gi), N.ptr(d_gh),
                                                  N.ptr(d_h), N.current_stream(g.device))
        N.check(rc, "ptgnn_b200_gru_gate_grads_f32")
        ref = BR.gru_gate_grads(gi, gh, h, g)
        for name, got in (("d_gi", d_gi), ("d_gh", d_gh), ("d_h", d_h)):
            _record("gru_gate_grads", FR.check_bound(got, *ref[name], f"H={H} rows={rows} g*{gs}: {name}"))


# ---- split GEMMs and the transposed aggregation, through _aggregation_backward -----------------------------------------------
@functools.lru_cache(maxsize=2)
def _stage_graph(kind):
    if kind == "unfused":
        adj, _ = UR.structured_graph(6000, big=8000)
        return adj, 6000
    return FR.structured_graph(64, 4, 300)


@pytest.mark.parametrize("kind,H,D", [("unfused", 64, 128), ("fused", 128, 128), ("fused", 128, 64)])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("gs", [1.0, 2.0 ** -27, 2.0 ** 17])
def test_split_gemm_and_transposed_aggregation(kind, H, D, reduce, gs):
    from ptgnn_b200 import autograd as AG
    from ptgnn_b200.edgeplan import EdgePlan

    adj, n = _stage_graph(kind)
    gen = torch.Generator().manual_seed(H + D)
    h = torch.randn(n, H, generator=gen)
    W = [torch.randn(D, H, generator=gen) / math.sqrt(H) for _ in adj]
    d_agg = torch.randn(n, D, generator=gen) * gs
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    plan = EdgePlan(adj_d, n)
    hd, Wd, gd = h.cuda(), [w.cuda() for w in W], d_agg.cuda()
    d_W, d_h = AG._aggregation_backward(plan, adj_d, hd, Wd, gd, reduce, None, torch.zeros_like(hd))
    x = gd
    if reduce == "mean":
        x = gd / (plan.row_ptr[1:] - plan.row_ptr[:-1]).clamp(min=1).to(torch.float32)[:, None]
    x = x.cpu()
    fused = kind == "fused"
    assert fused == (H == 128 and D in (64, 128))
    ref, bnd = BR.transposed_aggregate(x, adj, W, n, fused)
    _record(f"transposed aggregation ({kind})", FR.check_bound(d_h, ref, bnd, f"d h_src, {kind} {H}x{D} {reduce} g*{gs}"))
    sa, sb = BR.pow2_scale(x), BR.pow2_scale(h)
    for t, ((s, tg), got) in enumerate(zip(adj, d_W)):
        r, b = BR.mm_t_split(x[tg], h[s], sa, sb)
        _record("split gemm", FR.check_bound(got, r, b, f"dW_{t}, {kind} {H}x{D} {reduce} g*{gs}"))


# ---- layer gradients at gradient scales --------------------------------------------------------------------------------
def _graph(n, counts, seed, tie_free=False, empty_tail=0):
    gen = torch.Generator().manual_seed(seed)
    adj = [(torch.randint(0, n, (c,), generator=gen), torch.randint(0, n - empty_tail, (c,), generator=gen)) for c in counts]
    if tie_free:
        adj = [(s, t) if s.numel() == 0 else BR.dedup([(s, t)])[0] for s, t in adj]
    return adj


def _tie_free_states(n, H, seed, reduce, adj, message_fn):
    """Random states on which no winning message of max / min is within 5e-6 of its runner-up (the kernels' messages carry ~1e-6 of
    rounding, and a swapped winner moves a gradient row)."""
    gen = torch.Generator().manual_seed(seed)
    tgt = torch.cat([t for _s, t in adj])
    for _ in range(60):
        h = torch.randn(n, H, generator=gen)
        if reduce not in ("max", "min") or BR.tie_gap(message_fn(h.double()), tgt, n, reduce) > 5e-6:
            return h
    pytest.fail("could not draw states without near-ties")


def _check_layer(family, layer, h0, adj, forward64, scales=GRAD_SCALES, determinism=True):
    """Native d node_states and parameter gradients at every gradient scale against float64 autograd of the restatement."""
    n = h0.shape[0]
    p64 = BR.leaves64(layer)
    h64 = h0.double().requires_grad_(True)
    out64 = forward64(h64, p64)
    probe = torch.randn(out64.shape, generator=torch.Generator().manual_seed(99))
    names = ["node_states"] + list(p64)
    ref = torch.autograd.grad(out64, [h64] + list(p64.values()), probe.double(), allow_unused=True)
    ref = [torch.zeros_like(l) if r is None else r for r, l in zip(ref, [h64] + list(p64.values()))]
    layer = layer.cuda().train()
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]

    def run(gs):
        layer.zero_grad()
        x = h0.cuda().requires_grad_(True)
        layer(x, adj_d).backward(probe.cuda() * gs)
        grads = [x.grad] + [p.grad for _k, p in layer.named_parameters()]
        return [torch.zeros_like(p) if g is None else g.detach().clone() for g, p in zip(grads, [x] + list(layer.parameters()))]

    err1 = None
    for gs in scales:
        got = run(gs)
        errs = []
        for name, a, r in zip(names, got, ref):
            r_max, rel, e = BR.check_scaled(a, r * gs, f"{family} g*{gs:.3g}: d {name}")
            assert r_max <= TAU and rel <= TAU, f"{family} g*{gs:.3g}: d {name}: max|err|/max|ref| {r_max:.3e}, rel L2 {rel:.3e}"
            errs.append(e / gs)
            _record(f"{family} (every s)", max(r_max, rel))
            if gs == 1.0:
                _record(family, max(r_max, rel))
        if gs == 1.0:
            err1 = errs
            if determinism:
                again = run(gs)
                for name, a, b in zip(names, got, again):
                    assert torch.equal(a, b), f"{family}: d {name} differs between two backward passes"
        else:
            for name, e, e1, r in zip(names, errs, err1, ref):
                amax = float(r.abs().max()) if r.numel() else 0.0
                assert e <= 2 * e1 + 2.0 ** -40 * amax, f"{family} g*{gs:.3g}: d {name}: err/s {e:.3e} vs 2 err(1) {2 * e1:.3e}"


REDUCES = ["sum", "mean", "max", "min"]


@pytest.mark.parametrize("H,D", [(128, 128), (64, 128), (128, 64), (32, 68)])
@pytest.mark.parametrize("reduce", REDUCES)
def test_gated_layer_gradients_at_gradient_scales(H, D, reduce):
    import ptgnn_b200 as P

    torch.manual_seed(H + D)
    small = reduce in ("max", "min")
    n = 200 if small else 1500
    counts = [500, 0, 150, 40] if small else [5000, 0, 1500, 300]
    adj = _graph(n, counts, seed=H * D, tie_free=small, empty_tail=0 if small else 20)
    layer = P.GatedMessagePassingLayer(H, D, len(counts), reduce)
    W = [m.weight.detach().double() for m in layer.modules() if isinstance(m, torch.nn.Linear)]
    h0 = _tie_free_states(n, H, H + D, reduce, adj, lambda h: BR.messages64(h, adj, W, False))
    _check_layer(f"gated {H}x{D}", layer, h0, adj, lambda h, p: BR.gated_forward64(h, adj, p, reduce)[0])


@pytest.mark.parametrize("reduce,use_target,H,D,ln,dense,act", [
    ("sum", True, 128, 128, True, True, "gelu"), ("mean", False, 128, 64, False, True, None), ("max", True, 64, 128, True, False, "gelu"),
    ("min", False, 128, 128, False, False, None), ("sum", False, 128, 128, False, False, "tanh"), ("mean", True, 128, 128, True, True, "relu"),
    ("max", False, 36, 68, False, False, None)])
def test_mlp_layer_gradients_at_gradient_scales(reduce, use_target, H, D, ln, dense, act):
    import ptgnn_b200 as P

    torch.manual_seed(D + H)
    small = reduce in ("max", "min")
    n = 200 if small else 1500
    counts = [500, 0, 150, 40] if small else [5000, 0, 1500, 300]
    adj = _graph(n, counts, seed=D * 3 + H, tie_free=small, empty_tail=0 if small else 20)
    acts = {None: None, "gelu": torch.nn.GELU(), "tanh": torch.nn.Tanh(), "relu": torch.nn.ReLU()}
    layer = P.MlpMessagePassingLayer(H, H, D, len(counts), reduce, message_activation=acts[act], use_target_state_as_message_input=use_target,
                                     use_layer_norm=ln, use_dense_layer=dense)
    W = [m.single_linear.weight.detach().double() for m in layer.modules() if isinstance(m, P.MLP)]
    h0 = _tie_free_states(n, H, D + H, reduce, adj, lambda h: BR.messages64(h, adj, W, use_target))
    _check_layer(f"mlp {H}x{D}", layer, h0, adj, lambda h, p: BR.mlp_forward64(layer, h, adj, p, reduce, use_target)[0])


@pytest.mark.parametrize("reduce", REDUCES)
def test_egc_layer_gradients_at_gradient_scales(reduce):
    import ptgnn_b200 as P

    torch.manual_seed(17)
    small = reduce in ("max", "min")
    n = 150 if small else 1500
    counts = [350, 0, 100, 30] if small else [5000, 0, 1500, 300]
    adj = _graph(n, counts, seed=5, tie_free=small, empty_tail=0 if small else 20)
    layer = P.EGCMessagePassingLayer(128, 128, len(counts), reduce)
    W, cw, cb = (lambda w, a, b: ([x.double() for x in w], a.double(), b.double()))(*E.params_of(layer.state_dict(), len(counts)))
    h0 = _tie_free_states(n, 128, 3, reduce, adj, lambda h: BR.messages64(h, adj, W, False))
    pre = "_EGCMessagePassingLayer__"

    def fwd(h, p):
        return E.forward_torch(h, adj, [p[f"{pre}bases.{t}.weight"] for t in range(len(counts))], p[pre + "weight_coeffs.weight"],
                               p[pre + "weight_coeffs.bias"], reduce, 8, 4)

    _check_layer("egc 128", layer, h0, adj, fwd)


@pytest.mark.parametrize("case", ["no_edges", "large_sum"])
def test_gated_layer_gradients_edge_sizes(case):
    import ptgnn_b200 as P

    torch.manual_seed(23)
    if case == "no_edges":
        n, counts = 100, [0, 0]
    else:
        n, counts = 24_000, [60_000, 0, 30_000, 10_000]          # N > 20,000, E = 100k: several waves of every kernel
    adj = _graph(n, counts, seed=8)
    layer = P.GatedMessagePassingLayer(128, 128, len(counts), "sum")
    h0 = torch.randn(n, 128, generator=torch.Generator().manual_seed(4))
    _check_layer(f"gated 128x128 {case}", layer, h0, adj, lambda h, p: BR.gated_forward64(h, adj, p, "sum")[0])


# ---- range cases -------------------------------------------------------------------------------------------------------
def test_gradients_beyond_fp16_range_and_a_second_backward():
    """d_agg > 65504 (a sum loss under a 2^17 loss scale): finite, within the bar, and the transposed plans' range status stays clear
    (a second backward on the same adjacency raises nothing)."""
    import ptgnn_b200 as P
    from ptgnn_b200.edgeplan import plan_for

    torch.manual_seed(29)
    n, counts = 1500, [5000, 0, 1500, 300]
    adj = _graph(n, counts, seed=9)
    layer = P.MlpMessagePassingLayer(128, 128, 128, len(counts), "sum", message_activation=None, use_layer_norm=False, use_dense_layer=False)
    h0 = torch.randn(n, 128, generator=torch.Generator().manual_seed(6))
    gs = 2.0 ** 17
    probe = torch.randn(n, 128, generator=torch.Generator().manual_seed(99))
    assert float(probe.abs().max()) * gs > 65504              # d_agg = the upstream gradient: beyond fp16's range
    _check_layer("mlp 128x128 beyond fp16", layer, h0, adj, lambda h, p: BR.mlp_forward64(layer, h, adj, p, "sum", True)[0],
                 scales=(1.0, gs), determinism=False)
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    for _ in range(2):
        x = h0.cuda().requires_grad_(True)
        layer(x, adj_d).backward(probe.cuda() * gs)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(x.grad).all())
        plan_for([(t, s) for s, t in adj_d], n).poll()
        plan_for([(t, t) for _s, t in adj_d], n).poll()


@pytest.mark.parametrize("kind", ["gated", "mlp"])
def test_tf32_mode_gradients_with_large_states(kind, monkeypatch):
    """PTGNN_B200_FP32_MODE=tf32 is the documented mode for states beyond fp16's range: its backward splits them with a scale."""
    import ptgnn_b200 as P

    monkeypatch.setenv("PTGNN_B200_FP32_MODE", "tf32")
    torch.manual_seed(31)
    n, counts = 800, [3000, 0, 900, 200]
    adj = _graph(n, counts, seed=10)
    gen = torch.Generator().manual_seed(7)
    h0 = (torch.where(torch.rand(n, 128, generator=gen) < 0.5, -1.0, 1.0) * 10.0 ** (5 + torch.rand(n, 128, generator=gen))).float()
    if kind == "gated":
        layer = P.GatedMessagePassingLayer(128, 128, len(counts), "sum")
        gru = layer._GatedMessagePassingLayer__state_update
        with torch.no_grad():       # gate pre-activations of O(1) from states of 1e6: fp32 cannot resolve that cancellation with O(1) weights
            gru.weight_ih.mul_(1e-6)
            gru.weight_hh.mul_(1e-6)
        fwd = lambda h, p: BR.gated_forward64(h, adj, p, "sum")[0]        # noqa: E731
    else:
        layer = P.MlpMessagePassingLayer(128, 128, 128, len(counts), "sum")
        fwd = lambda h, p: BR.mlp_forward64(layer, h, adj, p, "sum", True)[0]      # noqa: E731
    _check_layer(f"{kind} tf32 large states", layer, h0, adj, fwd, scales=(1.0, 2.0 ** -27))


def test_zz_report_worst():
    """Prints the largest error / bound ratio of each stage family and the largest max|err| / max|ref| of each layer family at s = 1
    (run with -s)."""
    if not WORST:
        pytest.skip("no bound-checked case ran in this session")
    for k in sorted(WORST):
        print(f"worst {k:>40}: {WORST[k]:.3e}")
