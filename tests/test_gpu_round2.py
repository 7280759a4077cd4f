"""Round-2 parity cases (VERDICT r1 "What's weak" 1-2): the reference's OWN bf16 (autocast) outputs, the full 8-layer config-2
chain, the VarMisuse-shaped config 3 with the reference's default Mlp-max stack, a slice of the config-5 sweep, a Typilus-GGNN
stack with a residual layer between gated layers, inference_mode, two devices in one process."""
import pytest
import torch

from helpers import GOLDEN_DIR, assert_close, gated_oracle_args, golden_adjacency, golden_state_dict, load_golden, unchained  # noqa: F401
from oracle import ptgnn_oracle as O

pytestmark = pytest.mark.gpu


class _Embed(torch.nn.Module):
    def forward(self, x):
        return x


def _dev(adj):
    return [(s.cuda(), t.cuda()) for s, t in adj]


def _mlp_oracle_layer(layer, agg="max"):
    sd = {k: v.clone().cpu() for k, v in layer.state_dict().items()}
    p = "_MlpMessagePassingLayer__"
    T = sum(1 for k in sd if k.startswith(p + "edge_message_transformation_layers.") and k.endswith("_MLP__mlp_modules.1.weight"))
    return dict(kind="mlp", aggregation_fn=agg,
                edge_mlp_weights=[[sd[f"{p}edge_message_transformation_layers.{t}._MLP__mlp_modules.1.weight"]] for t in range(T)],
                ln_weight=sd[p + "state_update.0.weight"], ln_bias=sd[p + "state_update.0.bias"],
                dense_weight=sd[p + "state_update.1.weight"], dense_bias=sd[p + "state_update.1.bias"])


# ---- 1. bf16: pinned to the reference's own autocast path -----------------------------------------------------------------
# Fixtures: tests/golden/*_bf16ac.npz (generate_golden.py::main_round2): the reference layer under torch.autocast("cpu", bfloat16)
# and in fp32, same bf16-rounded inputs.  Measured reference-vs-reference gap (autocast vs fp32), committed with the generator's
# log: max 1.8e-2 .. 2.2e-2, mean 1.6e-3 .. 2.5e-3, fraction within 1e-2 * max(1, |ref|): gated sum 0.9979, gated max 0.9990,
# mlp sum 0.9962, mlp max 0.9854 -- the reference's own bf16 path does not meet a flat 1e-2 / 99.9 % bar against fp32.
# Bar used here: the kernels must be (a) within rel. L2 1e-2 of the reference's autocast output, and (b) AT LEAST AS CLOSE to
# the fp32 result as the reference's autocast path is (mean error <= 1.1 x, fraction within 1e-2 >= the reference's - 0.002).
@pytest.mark.parametrize("name", ["gated_sum_bf16ac", "gated_max_bf16ac", "mlp_sum_bf16ac", "mlp_max_bf16ac"])
def test_bf16_vs_reference_autocast(name):
    import ptgnn_b200 as P

    g = load_golden(name)
    adj, sd = golden_adjacency(g), golden_state_dict(g)
    H, agg = g["h"].shape[1], str(g["agg"])
    if name.startswith("gated"):
        layer = P.GatedMessagePassingLayer(H, H, len(adj), agg)
    else:
        layer = P.MlpMessagePassingLayer(H, H, H, len(adj), agg)
    layer.load_state_dict(sd)
    layer = layer.cuda().eval()
    hb = torch.from_numpy(g["h"]).to(torch.bfloat16)
    with torch.no_grad():
        got = layer(hb.cuda(), _dev(adj)).float().cpu()
    ref_ac, ref32 = torch.from_numpy(g["out_autocast"]), torch.from_numpy(g["out_fp32_rounded_inputs"])
    scale = ref32.abs().clamp(min=1)
    err_ours, err_ref = (got - ref32).abs(), (ref_ac - ref32).abs()
    frac_ours, frac_ref = (err_ours <= 1e-2 * scale).float().mean().item(), (err_ref <= 1e-2 * scale).float().mean().item()
    rel_ac = ((got - ref_ac).norm() / ref_ac.norm()).item()
    msg = (f"{name}: rel L2 vs autocast {rel_ac:.2e}; mean |err| vs fp32 ours {err_ours.mean():.2e} / reference autocast "
           f"{err_ref.mean():.2e}; within 1e-2 ours {frac_ours:.4f} / reference {frac_ref:.4f}")
    print(msg)
    assert rel_ac <= 1e-2, msg
    assert err_ours.mean().item() <= 1.1 * err_ref.mean().item(), msg
    assert frac_ours >= frac_ref - 0.002, msg


# ---- 2. residual layer between gated layers (typilus/train.py:39-65), pinned to the reference container's output --------------
def test_residual_stack_vs_reference_golden():
    import ptgnn_b200 as P

    g = load_golden("gnn_residual")
    raw = golden_adjacency(g)
    H, T = g["h"].shape[1], 2 * len(raw) + 1
    shared, last = P.GatedMessagePassingLayer(H, H, T, "max"), P.GatedMessagePassingLayer(2 * H, H, T, "max")
    shared.load_state_dict(golden_state_dict(g, "shared::"))
    last.load_state_dict(golden_state_dict(g, "last::"))
    r1 = P.ConcatResidualLayer(H)
    gnn = P.GraphNeuralNetwork([r1.pass_through_dummy_layer(), shared, shared, shared, r1, last], _Embed(), True, True).cuda().eval()
    assert gnn.input_node_state_dim == H and gnn.output_node_state_dim == 2 * H
    n = g["h"].shape[0]
    with torch.no_grad():
        out = gnn(node_data={"x": torch.from_numpy(g["h"]).cuda()}, adjacency_lists=_dev(raw), edge_feature_data=[],
                  node_to_graph_idx=torch.zeros(n, dtype=torch.int64).cuda(), reference_node_ids={}, reference_node_graph_idx={},
                  num_graphs=2)
    assert_close(out.output_node_representations, torch.from_numpy(g["out"]), tol=2e-5, what="residual stack (4 chained layers)")


# ---- 3. config 2: the full 8-layer chain the bench times ---------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_config2_eight_layer_chain(dtype):
    """N = 204,800, E = 1,105,920, T = 17, H = 128, 8 GatedMessagePassingLayers.  Every layer is checked on the ORACLE's input
    states (teacher forcing: 1e-5 per layer, all 8 layers), and the free-running 8-layer chain against the oracle's final states."""
    import ptgnn_b200 as P
    from ptgnn_b200.synthetic import graph2class_batch

    b = graph2class_batch()
    torch.manual_seed(0)
    layers = [P.GatedMessagePassingLayer(128, 128, 17, "sum") for _ in range(8)]
    gnn = P.GraphNeuralNetwork(layers, _Embed(), True, True).cuda().eval()
    h = torch.randn(b.num_nodes, 128, generator=torch.Generator().manual_seed(11))
    adj = O.expand_adjacency(b.adjacency_lists, b.num_nodes, True, True)
    specs = [dict(kind="gated", aggregation_fn="sum", **gated_oracle_args({k: v.cpu() for k, v in l.state_dict().items()})) for l in layers]
    states = O.gnn_forward(h, adj, specs)              # [h0, h1, ..., h8] on the CPU
    adj_d = gnn.expand_adjacency(_dev(b.adjacency_lists), b.num_nodes, "cuda")
    plan = P.plan_for(adj_d, b.num_nodes)
    cast = (lambda t: t.to(torch.bfloat16)) if dtype == "bf16" else (lambda t: t)
    with torch.no_grad(), P.edgeplan.shared_plan(plan):
        worst = 0.0
        for i, layer in enumerate(layers):
            got = layer(cast(states[i]).cuda(), adj_d).float().cpu()
            if dtype == "f32":
                err = ((got - states[i + 1]).abs() / states[i + 1].abs().clamp(min=1)).max().item()
                worst = max(worst, err)
                assert err <= 1e-5, f"layer {i}: max scaled error {err:.3e}"
            else:
                rel = ((got - states[i + 1]).norm() / states[i + 1].norm()).item()
                assert rel <= 1e-2, f"layer {i}: bf16 rel L2 {rel:.3e}"
        free = gnn.gnn(cast(h).cuda(), adj_d, None, b.node_to_graph_idx.cuda(), {}, {}).float().cpu()
    plan.validate()
    if dtype == "f32":
        chain = ((free - states[-1]).abs() / states[-1].abs().clamp(min=1)).max().item()
        print(f"config 2 fp32: worst per-layer error {worst:.2e}, free-running 8-layer chain {chain:.2e}")
        assert chain <= 5e-5, f"8-layer chain: {chain:.3e}"
    else:
        rel = ((free - states[-1]).norm() / states[-1].norm()).item()
        print(f"config 2 bf16: free-running 8-layer chain rel L2 {rel:.2e}")
        assert rel <= 3e-2


# ---- 4. config 3: VarMisuse-shaped batch, the implementation's default Mlp-max stack (varmisuse/train.py:43-74) -----------------
def test_config3_varmisuse_mlp_max_stack():
    """N = 80,000, E = 480,000, T = 23, H = 128, aggregation max: 8 MlpMessagePassingLayers in the concat-residual pattern --
    6 x (H -> H, D = H) and 2 x (2H -> H, D = 2H).  Each layer is checked on the oracle's input (LayerNorm can amplify upstream
    rounding by 1/sqrt(eps), so chains are checked layer by layer); the residual joins run through the container."""
    import ptgnn_b200 as P
    from ptgnn_b200.synthetic import varmisuse_batch

    b = varmisuse_batch()
    H, T = 128, 23
    torch.manual_seed(3)
    mk = lambda: P.MlpMessagePassingLayer(H, H, H, T, "max")                     # noqa: E731
    mk2 = lambda: P.MlpMessagePassingLayer(2 * H, H, 2 * H, T, "max")            # noqa: E731
    r1, r2 = P.ConcatResidualLayer(H), P.ConcatResidualLayer(H)
    stack = [r1.pass_through_dummy_layer(), mk(), mk(), mk(), r1, mk2(), r2.pass_through_dummy_layer(), mk(), mk(), mk(), r2, mk2()]
    gnn = P.GraphNeuralNetwork(stack, _Embed(), True, True).cuda().eval()
    assert b.layer_level_edges() == 480000 and b.num_nodes == 80000
    h = torch.randn(b.num_nodes, H, generator=torch.Generator().manual_seed(5))
    adj = O.expand_adjacency(b.adjacency_lists, b.num_nodes, True, True)
    feats = [torch.empty(a[0].shape[0], 0) for a in adj]
    adj_d = gnn.expand_adjacency(_dev(b.adjacency_lists), b.num_nodes, "cuda")
    plan = P.plan_for(adj_d, b.num_nodes)
    cur, tap = h, None
    with torch.no_grad(), P.edgeplan.shared_plan(plan):
        for i, layer in enumerate(stack):
            if isinstance(layer, P.MlpMessagePassingLayer):
                spec = _mlp_oracle_layer(layer)
                spec.pop("kind")
                agg = spec.pop("aggregation_fn")
                ref = O.mlp_layer_forward(cur, adj, feats, spec.pop("edge_mlp_weights"), agg, **spec)
                got = layer(cur.cuda(), adj_d).cpu()
                assert_close(got, ref, what=f"config 3 layer {i} ({layer.input_state_dimension} -> {layer.output_state_dimension})")
                cur = ref
            elif isinstance(layer, P.ConcatResidualLayer):
                cur = torch.cat((tap, cur), dim=-1)
            else:
                tap = cur
        out = gnn.gnn(h.cuda(), adj_d, None, b.node_to_graph_idx.cuda(), {}, {})
    plan.validate()
    assert out.shape == (b.num_nodes, H) and torch.isfinite(out).all()


# ---- 5. a slice of the config-5 sweep (single random graph, not block diagonal) -------------------------------------------------
@pytest.mark.parametrize("E,T,H,agg", [(100000, 1, 128, "sum"), (100000, 16, 128, "max"), (100000, 4, 64, "sum"),
                                       (100000, 4, 256, "max"), (1000000, 16, 128, "sum")])
def test_config5_sweep_slice(E, T, H, agg):
    import ptgnn_b200 as P
    from ptgnn_b200.synthetic import single_random_graph

    b = single_random_graph(E // 5, E, T, seed=2000 + T + H)
    torch.manual_seed(E % 97 + T)
    layer = P.GatedMessagePassingLayer(H, H, T, agg).cuda().eval()
    h = torch.randn(b.num_nodes, H, generator=torch.Generator().manual_seed(1))
    ref = O.gated_layer_forward(h, b.adjacency_lists, [torch.empty(a[0].shape[0], 0) for a in b.adjacency_lists], aggregation_fn=agg,
                                **gated_oracle_args({k: v.cpu() for k, v in layer.state_dict().items()}))
    with torch.no_grad():
        got = layer(h.cuda(), _dev(b.adjacency_lists))
    assert_close(got, ref, what=f"sweep E={E} T={T} H={H} {agg}")


# ---- 6. torch.inference_mode (ADVICE r1: version counters do not exist there) ---------------------------------------------------
def test_inference_mode_layer_and_container():
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(3)
    torch.manual_seed(3)
    n, H = 600, 64
    raw = [(torch.randint(0, n, (1500,), generator=gen), torch.randint(0, n, (1500,), generator=gen))]
    h = torch.randn(n, H, generator=gen)
    layer = P.GatedMessagePassingLayer(H, H, 3, "sum")
    gnn = P.GraphNeuralNetwork([layer, layer], _Embed(), True, True).cuda().eval()
    adj = O.expand_adjacency(raw, n, True, True)
    spec = dict(kind="gated", aggregation_fn="sum", **gated_oracle_args({k: v.cpu() for k, v in layer.state_dict().items()}))
    ref = O.gnn_forward(h, adj, [spec, spec])[-1]
    with torch.inference_mode():
        adj_d = [(s.cuda(), t.cuda()) for s, t in raw]          # inference tensors: no version counter
        out = gnn(node_data={"x": h.cuda()}, adjacency_lists=adj_d, edge_feature_data=[],
                  node_to_graph_idx=torch.zeros(n, dtype=torch.int64).cuda(), reference_node_ids={}, reference_node_graph_idx={}, num_graphs=1)
        single = layer(h.cuda(), gnn.expand_adjacency(adj_d, n, "cuda"))
    assert_close(out.output_node_representations, ref, tol=2e-5, what="inference_mode container")
    assert single.shape == (n, H)


# ---- 7. two devices in ONE process (ADVICE r1: per-device kernel attributes) ------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_two_devices_in_one_process(monkeypatch):
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(8)
    torch.manual_seed(8)
    n, H = 3000, 128
    adj = [(torch.randint(0, n, (9000,), generator=gen), torch.randint(0, n, (9000,), generator=gen))]
    h = torch.randn(n, H, generator=gen)
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        for mode in ("", "tf32"):                                 # the fused path, then the round-1 path
            monkeypatch.setenv("PTGNN_B200_FP32_MODE", mode)
            torch.manual_seed(8)
            layer = P.GatedMessagePassingLayer(H, H, 1, "sum").to(dev).eval()
            with torch.no_grad():
                outs.append(layer(h.to(dev), [(s.to(dev), t.to(dev)) for s, t in adj]).cpu())
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3])


# ---- 8. CUDA-graph capture of the layer loop -------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_captured_layer_loop_matches_eager_and_follows_its_buffers(dtype):
    import ptgnn_b200 as P

    gen = torch.Generator().manual_seed(21)
    torch.manual_seed(21)
    n, H = 5000, 128
    raw = [(torch.randint(0, n, (7000,), generator=gen), torch.randint(0, n, (7000,), generator=gen)),
           (torch.randint(0, n, (3000,), generator=gen), torch.randint(0, n, (3000,), generator=gen))]
    layers = [P.GatedMessagePassingLayer(H, H, 5, "sum"), P.GatedMessagePassingLayer(H, H, 5, "max")]
    gnn = P.GraphNeuralNetwork(layers, _Embed(), True, True).cuda().eval()
    h_buf = torch.randn(n, H, generator=gen).to(dtype).cuda()
    adj_buf = gnn.expand_adjacency(_dev(raw), n, "cuda")
    graphed = gnn.capture(h_buf, adj_buf)
    with torch.no_grad():
        eager = gnn.gnn(h_buf, adj_buf, None, None, {}, {})
    assert torch.equal(graphed.replay(), eager)
    # new minibatch of the same shape: refill the static buffers in place (states AND edges), replay
    h2 = torch.randn(n, H, generator=gen).to(dtype).cuda()
    raw2 = [(torch.randint(0, n, (7000,), generator=gen).cuda(), torch.randint(0, n, (7000,), generator=gen).cuda()),
            (torch.randint(0, n, (3000,), generator=gen).cuda(), torch.randint(0, n, (3000,), generator=gen).cuda())]
    h_buf.copy_(h2)
    for (bs, bt), (s, t) in zip(adj_buf[:2], raw2):
        bs.copy_(s); bt.copy_(t)       # the backward-edge entries of adj_buf alias these tensors
    out2 = graphed.replay().clone()
    P.clear_plan_cache()
    with torch.no_grad():
        eager2 = gnn.gnn(h2, gnn.expand_adjacency(raw2, n, "cuda"), None, None, {}, {})
    assert torch.equal(out2, eager2)


# ---- 9. packed states handed from layer to layer (edgeplan.state_chain) ------------------------------------------------------------
def test_state_chain_is_bit_identical_and_skips_the_packing_passes():
    """Inside a container's layer loop the GRU kernel of layer i also writes the fp16 (hi | lo') form of its output and layer i + 1
    skips its packing pass: results bit-identical to the unchained run, L - 1 fewer launches; a tensor that is not the previous
    layer's output (here: a residual sum) falls back to packing; a stand-alone layer call never chains."""
    import ptgnn_b200 as P
    from ptgnn_b200 import _native as N
    from helpers import random_adjacency

    gen = torch.Generator().manual_seed(5)
    torch.manual_seed(5)
    n, counts, L = 5000, [9000, 4000, 0, 700], 4
    adj = _dev(random_adjacency(gen, n, counts))
    layers = [P.GatedMessagePassingLayer(128, 128, len(counts), "sum") for _ in range(L)]
    gnn = P.GraphNeuralNetwork(layers, _Embed(), False, False).cuda().eval()
    h = torch.randn(n, 128, generator=gen).cuda()
    with torch.no_grad():
        gnn.gnn(h, adj, None, None, {}, {})                      # plan + weight caches
        l0 = N.launch_count()
        chained = gnn.gnn(h, adj, None, None, {}, {})
        l1 = N.launch_count()
        with unchained():
            plain = gnn.gnn(h, adj, None, None, {}, {})
        l2 = N.launch_count()
        assert torch.equal(chained, plain)
        assert (l2 - l1) - (l1 - l0) == L - 1, f"chained {l1 - l0} launches, unchained {l2 - l1}"
        # every layer's own output is the same with and without the hand-off (all states)
        a = gnn.gnn(h, adj, None, None, {}, {}, return_all_states=True)
        with unchained():
            b = gnn.gnn(h, adj, None, None, {}, {}, return_all_states=True)
        assert torch.equal(a, b)
        # a layer that gets a different tensor than the previous layer's output must not use the stale packed copy
        join = P.MeanResidualLayer(128)
        res = P.GraphNeuralNetwork([join.pass_through_dummy_layer(), layers[0], join, layers[1]], _Embed(), False, False).cuda().eval()
        got = res.gnn(h, adj, None, None, {}, {})
        h1 = layers[0](h, adj)
        want = layers[1](torch.stack((h, h1), dim=-1).mean(dim=-1), adj)
        assert torch.equal(got, want)
        # ... and an in-place edit of the handed-over tensor invalidates the packed copy (version counter)
        with P.edgeplan.shared_plan(P.plan_for(adj, n)), P.edgeplan.state_chain() as chain:
            chain.want_output = True
            mid = layers[0](h, adj)
            assert chain.lookup(mid) is not None
            mid.mul_(0.5)
            assert chain.lookup(mid) is None
            assert torch.equal(layers[1](mid, adj), layers[1](mid.clone(), adj))
        # overflow in a chained state is still reported
        big = h.clone(); big[7, 3] = 1e30
        plan = P.plan_for(adj, n)
        with pytest.raises(FloatingPointError):
            gnn.gnn(big, adj, None, None, {}, {})
            plan.validate()
