"""GPU: the native PNA kernel (DESIGN.md §3.10) against the float32 restatement of its operation order (tests/pna_reference.py), its
gradients against torch.autograd, and ``MlpMessagePassingLayer`` with the native ``PnaMessageAggregation`` under autograd and
training-mode dropout."""
import pytest
import torch
import torch.nn.functional as F

import pna_reference as R
from test_oracle_pna import FORWARD, load

pytestmark = pytest.mark.gpu


def plan_of(targets: torch.Tensor, n: int):
    from ptgnn_b200.edgeplan import EdgePlan

    t = targets.cuda()
    return EdgePlan([(t, t)], n)


def run(messages: torch.Tensor, targets: torch.Tensor, n: int, delta: float, plan=None):
    """The forward entry point with NaN-prefilled outputs and -1-prefilled arg ids: (out, arg_max, arg_min) on the CPU."""
    from ptgnn_b200 import _native as N

    plan = plan or plan_of(targets, n)
    m = messages.cuda().contiguous()
    D = m.shape[1]
    out = torch.full((n, 15 * D), float("nan"), device="cuda")
    args = torch.full((2, n, D), -1, dtype=torch.int32, device="cuda")
    rc = N.lib().ptgnn_b200_pna_forward(int(m.dtype == torch.bfloat16), N.ptr(m), m.shape[0], D, N.ptr(plan.row_ptr),
                                        N.ptr(plan.perm) if m.shape[0] else None, n, float(delta), N.ptr(out), N.ptr(args[0]),
                                        N.ptr(args[1]), N.current_stream(m.device))
    N.check(rc, "ptgnn_b200_pna_forward")
    return out.cpu(), args[0].cpu().long(), args[1].cpu().long()


def check_forward(messages, targets, n, delta, what):
    got, amx, amn = run(messages, targets, n, delta)
    ref, rmx, rmn = R.emulate_forward(messages, targets, n, delta)
    D = messages.shape[1]
    nan_g, nan_r = torch.isnan(got), torch.isnan(ref)
    assert torch.equal(nan_g[:, :5 * D], nan_r[:, :5 * D]), f"{what}: NaN pattern of S"
    assert torch.equal(torch.nan_to_num(got[:, :5 * D]), torch.nan_to_num(ref[:, :5 * D])), f"{what}: S not bit-identical"
    err = (got.double() - ref.double()).abs()
    ok = (err <= R.scaled_bound(torch.nan_to_num(ref), D)) | nan_r | (err == 0)
    assert bool(ok[:, 5 * D:].all()), f"{what}: scaled blocks outside the bound (worst {(err / ref.double().abs())[~ok].max():.3e})"
    assert torch.equal(amx, rmx) and torch.equal(amn, rmn), f"{what}: winning edge ids"


@pytest.mark.parametrize("name", FORWARD)
def test_kernel_matches_the_restatement_at_the_fixtures(name):
    f = load(name)
    check_forward(f["messages"], f["targets"], f["n"], f["delta"], name)


def degree_case(counts, D, dtype, seed, delta=2.3):
    gen = torch.Generator().manual_seed(seed)
    t = torch.cat([torch.full((c,), v, dtype=torch.int64) for v, c in enumerate(counts)])
    t = t[torch.randperm(t.numel(), generator=gen)]
    m = (torch.randn(t.numel(), D, generator=gen) * 1.3 + 0.2).to(dtype)
    return m, t, len(counts), delta


DEGREES = [0, 1, 2, 15, 16, 17, 31, 32, 33]


@pytest.mark.parametrize("D,dtype", [(4, torch.float32), (36, torch.float32), (64, torch.float32), (128, torch.float32),
                                     (384, torch.float32), (512, torch.float32), (64, torch.bfloat16), (256, torch.bfloat16),
                                     (512, torch.bfloat16)])
def test_kernel_at_degree_edges_and_widths(D, dtype):
    # every degree around the load batches, runs of empty targets, a target count that is not a multiple of the rows per warp (4)
    counts = DEGREES * 3 + [0] * 7 + DEGREES[::-1] + [0, 0, 5]
    assert len(counts) % 4 != 0
    check_forward(*degree_case(counts, D, dtype, D), f"D={D} {dtype}")


def test_kernel_on_a_hub_of_200000_edges():
    m, t, n, delta = degree_case([200_000], 128, torch.float32, 3, delta=1.0)
    check_forward(m, t, n, delta, "hub")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_kernel_at_config_3_size(dtype):
    gen = torch.Generator().manual_seed(11)
    n, E, D = 80_000, 480_000, 128
    t = torch.randint(0, n, (E,), generator=gen)
    m = torch.randn(E, D, generator=gen).to(dtype)
    check_forward(m, t, n, 2.3, f"config 3 {dtype}")


def test_runs_are_bit_identical_forward_and_backward():
    from ptgnn_b200.aggregation import native_pna, native_pna_backward

    gen = torch.Generator().manual_seed(12)
    n, E, D = 20_000, 120_000, 128
    t = torch.randint(0, n, (E,), generator=gen).cuda()
    m = torch.randn(E, D, generator=gen).cuda()
    g = torch.randn(n, 15 * D, generator=gen).cuda()
    plan = plan_of(t, n)
    a = native_pna(m, plan, 2.3, want_arg=True)
    b = native_pna(m, plan, 2.3, want_arg=True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    da = native_pna_backward(m, plan, 2.3, *a, g)
    db = native_pna_backward(m, plan, 2.3, *b, g)
    assert torch.equal(da, db)


def close(got, ref, tol, what):
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    scaled = ((got - ref).abs().max() / ref.abs().max().clamp(min=1e-30)).item()
    rel = ((got - ref).norm() / ref.norm().clamp(min=1e-30)).item()
    assert scaled <= tol and rel <= tol, f"{what}: scaled max {scaled:.3e}, relative L2 {rel:.3e}"


def test_backward_kernel_matches_the_formula():
    from ptgnn_b200.aggregation import native_pna, native_pna_backward

    m, t, n, delta = degree_case(DEGREES * 4 + [300, 0, 1], 64, torch.float32, 5)
    plan = plan_of(t, n)
    out, amx, amn = native_pna(m.cuda(), plan, delta, want_arg=True)
    g = torch.randn(n, 15 * 64, generator=torch.Generator().manual_seed(6))
    got = native_pna_backward(m.cuda(), plan, delta, out, amx, amn, g.cuda()).cpu()
    ref = R.emulate_backward(m, t, n, delta, out.cpu(), amx.cpu().long(), amn.cpu().long(), g)
    close(got, ref, 1e-5, "backward kernel vs its formula")
    dropped = R.emulate_backward(m, t, n, delta, out.cpu(), amx.cpu().long(), amn.cpu().long(), g, drop_mean_term=True)
    assert ((got - dropped).abs().max() / got.abs().max()).item() > 1e-3


@pytest.mark.parametrize("name", ["pna_grad_d8"])
def test_module_gradient_matches_the_reference_fixture(name):
    import ptgnn_b200 as P

    f = load(name)
    z = f["z"]
    x = f["messages"].cuda().requires_grad_(True)
    out = P.PnaMessageAggregation(delta=f["delta"])(x, f["targets"].cuda(), f["n"])
    out.backward(torch.from_numpy(z["d_out"]).cuda())
    close(x.grad, torch.from_numpy(z["d_messages"]), 1e-4, name)


@pytest.mark.parametrize("seed", [1, 2])
def test_module_gradient_matches_autograd(seed):
    import ptgnn_b200 as P

    m, t, n, delta = degree_case(DEGREES * 5 + [0, 0, 700, 1, 1], 32, torch.float32, 20 + seed)
    g = torch.randn(n, 15 * 32, generator=torch.Generator().manual_seed(seed))
    x = m.cuda().requires_grad_(True)
    out = P.PnaMessageAggregation(delta=delta)(x, t.cuda(), n)
    out.backward(g.cuda())
    xr = m.clone().requires_grad_(True)
    ref = R.layer_forward(xr, t, n, delta)
    ref.backward(g)
    close(out, ref, 1e-5, "module forward")
    close(x.grad, xr.grad, 1e-4, "module gradient vs float32 autograd")
    # float64 on the (target, column) pairs none of whose messages is within 1e-3 of the relu's mask boundary (this excludes every
    # one-message target, whose fp32 std cancels: m^2 - (m / 1.00001)^2)
    x64 = m.double().requires_grad_(True)
    R.layer_forward(x64, t, n, delta).backward(g.double())
    mean = R.layer_forward(m.double(), t, n, delta)[:, 32:64]
    near = ((m.double() ** 2 - mean[t] ** 2).abs() <= 1e-3 * (m.double() ** 2)).double()
    good = torch.zeros(n, 32, dtype=torch.float64).index_add_(0, t, near)[t] == 0
    assert good.float().mean() > 0.5
    close(x.grad[good.cuda()], x64.grad[good], 1e-4, "module gradient vs float64 autograd")


def test_module_refuses_what_it_cannot_do():
    import ptgnn_b200 as P

    t = torch.zeros(8, dtype=torch.int64, device="cuda")
    agg = P.PnaMessageAggregation()
    with pytest.raises(NotImplementedError):
        agg(torch.randn(8, 6, device="cuda"), t, 2)                      # D not a multiple of 4
    with pytest.raises(NotImplementedError):
        agg(torch.randn(8, 516, device="cuda"), t, 2)
    with pytest.raises(NotImplementedError):
        agg(torch.randn(8, 8, device="cuda", dtype=torch.bfloat16).requires_grad_(True), t, 2)
    with pytest.raises(ValueError):
        agg(torch.randn(7, 8, device="cuda"), t, 2)
    out = agg(torch.randn(8, 8, device="cuda", dtype=torch.bfloat16), t, 2)
    assert out.dtype == torch.float32 and out.shape == (2, 120)


def test_module_call_makes_no_host_synchronisation():
    import ptgnn_b200 as P

    m, t, n, delta = degree_case(DEGREES * 2, 64, torch.float32, 7)
    m, t = m.cuda(), t.cuda()
    agg = P.PnaMessageAggregation(delta=delta)
    agg(m, t, n)            # builds and caches the plan
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        agg(m, t, n)
        agg(m.requires_grad_(True), t, n).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")


# ---- MlpMessagePassingLayer + PNA -------------------------------------------------------------------------------------------------
def mlp_pna_reference(layer, h, adj, use_target, delta):
    """mlpmessagepassing.py:82-117 with PNA on the CPU: messages per type, the float32 restatement, GELU, LayerNorm, dense, Tanh.
    The messages take the values of the native message kernel (their gradient flows through the CPU product): the std of a
    one-message target, sqrt(relu(m^2 - (m / 1.00001)^2) + 1e-10), turns a relative difference of 1e-7 in m into 5e-3 in the std."""
    from ptgnn_b200 import composed as C
    from ptgnn_b200.edgeplan import plan_for

    p = "_MlpMessagePassingLayer__"
    params = dict(layer.named_parameters())
    leaves = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in params.items()}
    msgs = []
    for i, (s, t) in enumerate(adj):
        w = leaves[f"{p}edge_message_transformation_layers.{i}._MLP__mlp_modules.1.weight"]
        msgs.append(F.linear(torch.cat([h[s], h[t]], -1) if use_target else h[s], w))
    msg = torch.cat(msgs)
    with torch.no_grad():
        hd = h.detach().cuda()
        native = C.edge_messages(plan_for([(s.cuda(), t.cuda()) for s, t in adj], h.shape[0]), hd, hd if use_target else None,
                                 [params[f"{p}edge_message_transformation_layers.{i}._MLP__mlp_modules.1.weight"].detach()
                                  for i in range(len(adj))], use_target).cpu()
    msg = (msg - msg.detach()) + native                 # the native values exactly, the CPU product's gradient
    targets = torch.cat([t for _, t in adj])
    agg = R.layer_forward(msg, targets, h.shape[0], delta)
    x = F.layer_norm(F.gelu(agg), (agg.shape[1],), leaves[p + "state_update.0.weight"], leaves[p + "state_update.0.bias"])
    out = torch.tanh(F.linear(x, leaves[p + "state_update.1.weight"], leaves[p + "state_update.1.bias"]))
    return out, leaves


@pytest.mark.parametrize("use_target", [True, False])
def test_mlp_layer_with_pna_trains(use_target):
    import ptgnn_b200 as P
    from helpers import random_adjacency

    gen = torch.Generator().manual_seed(31)
    torch.manual_seed(4)
    n, H, D, counts = 500, 64, 32, [1500, 0, 600]
    adj = random_adjacency(gen, n, counts)
    h = torch.randn(n, H, generator=gen)
    layer = P.MlpMessagePassingLayer(H, 48, D, len(counts), P.PnaMessageAggregation(delta=2.0),
                                     use_target_state_as_message_input=use_target).cuda().train()
    g = torch.randn(n, 48, generator=gen)
    hg = h.cuda().requires_grad_(True)
    out = layer(hg, [(s.cuda(), t.cuda()) for s, t in adj])
    out.backward(g.cuda())
    hr = h.clone().requires_grad_(True)
    ref, leaves = mlp_pna_reference(layer, hr, adj, use_target, 2.0)
    ref.backward(g)
    close(out, ref, 1e-4, "mlp + PNA forward")
    close(hg.grad, hr.grad, 1e-4, "d node_states")
    for name, p in layer.named_parameters():
        close(p.grad, leaves[name].grad, 1e-4, f"d {name}")


def test_mlp_layer_with_pna_training_dropout():
    import ptgnn_b200 as P
    from helpers import random_adjacency

    gen = torch.Generator().manual_seed(32)
    torch.manual_seed(5)
    n, H, D = 400, 32, 16
    adj = [(s.cuda(), t.cuda()) for s, t in random_adjacency(gen, n, [1200])]
    h = torch.randn(n, H, generator=gen).cuda()
    layer = P.MlpMessagePassingLayer(H, 32, D, 1, P.PnaMessageAggregation(), dropout_rate=0.5).cuda()
    with torch.no_grad():
        plain = layer.eval()(h, adj)
        layer.train()
        dropped = layer(h, adj)                  # no gradients: the composed path, dropout on the result
    hg = h.clone().requires_grad_(True)
    trained = layer(hg, adj)                     # gradients: _MlpLayerFunction, dropout outside it
    trained.sum().backward()
    for out in (dropped, trained):
        zero = out == 0
        assert 0.4 < zero.float().mean().item() < 0.6
        assert torch.allclose(out[~zero], 2.0 * plain[~zero], rtol=1e-6, atol=1e-7)
    kept = (trained != 0).float()
    hr = h.clone().requires_grad_(True)
    (layer.eval()(hr, adj) * 2.0 * kept).sum().backward()
    close(hg.grad, hr.grad, 1e-5, "d node_states through the dropout mask")


def test_mlp_layer_with_pna_eval_matches_the_module():
    """The layer's PNA on its own plan equals the module called on the concatenated targets (as the reference passes them)."""
    import ptgnn_b200 as P
    from ptgnn_b200 import composed as C
    from helpers import random_adjacency

    gen = torch.Generator().manual_seed(33)
    torch.manual_seed(6)
    n, H, D = 300, 32, 16
    adj = [(s.cuda(), t.cuda()) for s, t in random_adjacency(gen, n, [700, 300])]
    h = torch.randn(n, H, generator=gen).cuda()
    agg_fn = P.PnaMessageAggregation(delta=1.5)
    layer = P.MlpMessagePassingLayer(H, 24, D, 2, agg_fn, message_activation=None, use_layer_norm=False, use_dense_layer=False).cuda().eval()
    with torch.no_grad():
        got = layer(h, adj)
        plan = P.plan_for(adj, n)
        ws = [m.single_linear.weight for m in layer._MlpMessagePassingLayer__edge_message_transformation_layers]
        msg = C.edge_messages(plan, h, h, ws, True)
        ref = agg_fn(msg, torch.cat([t for _, t in adj]), n)
    assert torch.equal(got, ref)
