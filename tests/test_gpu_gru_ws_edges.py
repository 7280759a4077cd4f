"""The weights-stationary GRU kernel (csrc/gru_ws.cu) element by element against float64 with a derived bound per element
(``unfused_reference.gru`` in mode '3xfp16' / 'bf16', ``unfused_reference.gru_table``), in both of its instances.

* Layer instance: the node update of ``GatedMessagePassingLayer(H, 128, 3, agg)`` on the fused path (fp32 H 64 / 128, bf16 H 64 /
  128 / 256).  Chain of bounds: ``fused_reference.messages`` -> ``aggregate`` -> GRU.  The row counts give a single partial tile
  (1, 63), exact tiles (64), one row past a tile (65, 129), fewer tiles than CTAs per hidden-unit block (1,000), a tile count the
  CTAs do not divide, and enough tiles that the operand ring wraps many times.
* State-only instance (TABLE): ``GruGlobalStateUpdate.table_update`` given exact fp32 summaries, over every ring depth the kernel
  takes (fp32 down to 3 slots at H = 448, bf16 down to 2 at H = 1024), with summaries from 0 to |g| ~ 30 (saturated gates, where
  the h-side carries the output).  Chain: ``dense`` (the fp32 input-side table) -> ``gru_table``.
* The packed fp16 (hi | lo') output both instances write under ``edgeplan.state_chain``: the split of their own fp32 output.
* The whole ``GruGlobalStateUpdate``: native readout -> table -> GRU.  Chain: ``global_exchange_reference.readout_bound`` ->
  ``dense`` -> ``gru_table``.

Every case runs twice and must be bit-identical.  The float64 GEMMs run on the device."""
import pytest
import torch

import fused_reference as FR
import global_exchange_reference as GX
import unfused_reference as R
from helpers import gated_oracle_args, random_adjacency, split_f16

pytestmark = pytest.mark.gpu

T = 3
D = 128
WORST = {}          # family -> largest error / bound ratio seen (printed with -s)
N_ROWS = (1, 63, 64, 65, 127, 129, 1000, 64 * (33 * 3 + 5) + 17, 40_000)


def _check(got, ref, bound, family, what):
    """check_bound on the device; the CPU version reports the elements outside their bound."""
    got = got.detach().double().to(ref.device)
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} != {tuple(ref.shape)}"
    err = (got - ref).abs()
    if not bool((err <= bound).all()):
        FR.check_bound(got.cpu(), ref.cpu(), bound.cpu(), what)
    pos = bound > 0
    ratio = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    return ratio


def _twice(fn):
    with torch.no_grad():
        a, b = fn(), fn()
    assert torch.equal(a, b), "output is not run-to-run bit-identical"
    return a


def _packed_split(out: torch.Tensor) -> torch.Tensor:
    """The fp16 (hi | lo') rows of fp32 rows, with round-to-nearest conversions: hi = fl16(x), lo' = fl16(2^11 (x - hi))."""
    return torch.cat(split_f16(out), 1)


# ---- layer instance ------------------------------------------------------------------------------------------------------
LAYER_ROWS = [("sum", N) for N in N_ROWS] + [(agg, N) for agg in ("mean", "max", "min") for N in (63, 64 * 104 + 17, 40_000)]


def _gated(H, agg, seed):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    layer = P.GatedMessagePassingLayer(H, D, T, agg).cuda().eval()
    return layer, gated_oracle_args({k: v.clone().cpu() for k, v in layer.state_dict().items()})


def _graph(N, seed):
    gen = torch.Generator().manual_seed(seed)
    adj = random_adjacency(gen, N, [max(1, 2 * N), max(1, N), max(1, N // 2)])
    return adj, [(s.cuda(), t.cuda()) for s, t in adj], gen


def _layer_case(H, agg, N, bf16):
    seed = N + H + len(agg) + 100 * bf16
    adj, adj_d, gen = _graph(N, seed)
    h = torch.randn(N, H, generator=gen) * 0.5
    h = h.to(torch.bfloat16) if bf16 else h
    layer, args = _gated(H, agg, seed)
    got = _twice(lambda: layer(h.cuda(), adj_d))
    tgt, m, err = FR.messages(h, adj, args["edge_weights"], False, bf16)
    x, ex, _ = FR.aggregate(tgt, m, err, N, agg, bf16)
    if not bf16:
        assert float(x.abs().max()) < 65504          # the fp16 (hi | lo') aggregate holds it
    ref, bound = R.gru(x.cuda(), ex.cuda(), h.cuda(), *(args[k] for k in ("gru_w_ih", "gru_w_hh", "gru_b_ih", "gru_b_hh")),
                       mode="bf16" if bf16 else "3xfp16")
    family = f"layer {'bf16' if bf16 else 'fp32'}"
    _check(got, ref, bound, family, f"{family} H={H} {agg} N={N}")


@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("agg,N", LAYER_ROWS)
def test_layer_gru_fp32(agg, N, H):
    _layer_case(H, agg, N, False)


@pytest.mark.parametrize("H", [64, 128, 256])
@pytest.mark.parametrize("agg,N", LAYER_ROWS)
def test_layer_gru_bf16(agg, N, H):
    _layer_case(H, agg, N, True)


# ---- state-only instance -------------------------------------------------------------------------------------------------
def num_slots(bf16: bool, H: int) -> int:
    """Geometry<NPROD>::num_slots(H, 0) of csrc/gru_ws.cu: the operand ring takes the shared memory the resident weights leave."""
    npart, max_slots = (1, 12) if bf16 else (2, 7)
    fixed = 1024 + (H // 64) * npart * 96 * 128 + H * 16 + 256
    return min((232448 - fixed) // (npart * 64 * 128), max_slots)


TABLE_H = {False: {64: 7, 192: 7, 256: 7, 320: 6, 384: 4, 448: 3}, True: {64: 12, 192: 12, 512: 12, 960: 3, 1024: 2}}


def test_table_shapes_and_ring_depths():
    from ptgnn_b200 import _native as N

    lib = N.lib()
    for bf16, depths in TABLE_H.items():
        for H, slots in depths.items():
            assert num_slots(bf16, H) == slots, (bf16, H)
            assert lib.ptgnn_b200_global_gru_supported(int(bf16), H) == 1, (bf16, H)
    assert num_slots(False, 512) < 2 and lib.ptgnn_b200_global_gru_supported(0, 512) == 0
    assert num_slots(True, 1088) < 2 and lib.ptgnn_b200_global_gru_supported(1, 1088) == 0


def _table_rows(H):
    """{1, 63, 65, a tile count the CTAs per hidden-unit block do not divide, many tiles}."""
    groups = 132 // (H // 32)
    tiles = 3 * groups + groups // 2 + 1
    assert tiles % groups != 0
    return (1, 63, 65, 64 * tiles - 5, 40_000 if H <= 448 else 12_000)


def _n2g(layout, N, gen):
    if layout == "one_graph":
        return torch.zeros(N, dtype=torch.int64), 1
    if layout == "node_per_graph":
        return torch.arange(N), N
    ids = torch.tensor([0, 2, 3, 5, 6, 9])[torch.randint(0, 6, (N,), generator=gen)]     # unsorted; 1, 4, 7, 8 and 10-11 empty
    ids[0] = 9
    return ids, 12


def _summaries(G, S, gen):
    g = torch.randn(G, S, generator=gen) * 4
    g[::5] *= 8                                       # |g| up to ~30: saturated gates
    g = g.clamp(-30.0, 30.0)
    g[1::7] = 0
    return g


def _global_layer(H, seed, kind="sum"):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    reducer = P.WeightedSumVarSizedElementReduce(H) if kind == "weighted" else P.SimpleVarSizedElementReduce(kind)
    layer = P.GruGlobalStateUpdate(reducer, H, H).cuda().eval()
    sd = {k: v.detach().cpu() for k, v in layer.state_dict().items()}
    p = "_GruGlobalStateUpdate__gru_cell."
    w = sd.get("_AbstractGlobalGraphExchange__global_graph_representation_module._WeightedSumVarSizedElementReduce__weights_layer.weight")
    return layer, w, [sd[p + k] for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]


def _table_ref(g64, e_g, n2g, h, p, bf16):
    S, H = g64.shape[1], h.shape[1]
    gi, e_gi = R.dense(g64.cuda(), None if e_g is None else e_g.cuda(), p[0], p[2], None, R.fp32_dense_mode(S, 3 * H))
    idx = n2g.cuda()
    return R.gru_table(gi[idx], e_gi[idx], h.cuda(), p[1], p[3], "bf16" if bf16 else "3xfp16")


TABLE_CASES = [(bf16, H, layout) for bf16 in (False, True) for H in TABLE_H[bf16]
               for layout in ("one_graph", "node_per_graph", "unsorted_empty")]


@pytest.mark.parametrize("bf16,H,layout", TABLE_CASES, ids=[f"{'bf16' if b else 'fp32'}-H{H}-{l}" for b, H, l in TABLE_CASES])
def test_table_gru(bf16, H, layout):
    from ptgnn_b200.reduceops import graph_plan

    layer, _, p = _global_layer(H, H + 7 * bf16)
    family = f"table {'bf16' if bf16 else 'fp32'} ({num_slots(bf16, H)} slots)"
    for N in _table_rows(H):
        gen = torch.Generator().manual_seed(N + H + len(layout))
        n2g, G = _n2g(layout, N, gen)
        g = _summaries(G, H, gen)
        h = torch.randn(N, H, generator=gen) * 0.5
        h = h.to(torch.bfloat16) if bf16 else h
        hd, gd, n2g_d = h.cuda(), g.cuda(), n2g.cuda()
        got = _twice(lambda: layer.table_update(hd, gd, graph_plan(n2g_d, G)))
        ref, bound = _table_ref(g.double(), None, n2g, h, p, bf16)
        _check(got, ref, bound, family, f"{family} H={H} {layout} N={N}")


# ---- packed output -------------------------------------------------------------------------------------------------------
def _packed_run(fn):
    from ptgnn_b200 import edgeplan

    with torch.no_grad(), edgeplan.state_chain() as chain:
        chain.want_output = True
        out = fn()
        packed = chain.lookup(out)
    assert packed is not None, "no packed output was handed on"
    N, H = out.shape
    return out, packed[:N * 2 * H * 2].view(torch.float16).reshape(N, 2 * H)


@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("N", [63, 65, 129, 64 * (33 * 3 + 5) + 17])
def test_layer_packed_output_is_the_split_of_the_output(N, H):
    adj, adj_d, gen = _graph(N, 300 + N + H)
    h = (torch.randn(N, H, generator=gen) * 0.5).cuda()
    layer, _ = _gated(H, "sum", N + H)
    out, packed = _packed_run(lambda: layer(h, adj_d))
    assert torch.equal(out, _twice(lambda: layer(h, adj_d))), "chained and plain outputs differ"
    want = _packed_split(out.cpu())
    assert torch.equal(packed.cpu().view(torch.int16), want.view(torch.int16)), "packed rows differ from the split of the output"


@pytest.mark.parametrize("H", [64, 192, 448])
@pytest.mark.parametrize("N", [63, 65, 64 * 37 + 9])
def test_table_packed_output_is_the_split_of_the_output(N, H):
    from ptgnn_b200.reduceops import graph_plan

    gen = torch.Generator().manual_seed(N * 5 + H)
    n2g, G = _n2g("unsorted_empty", N, gen)
    g, h = _summaries(G, H, gen).cuda(), (torch.randn(N, H, generator=gen) * 0.5).cuda()
    layer, _, _ = _global_layer(H, N + H)
    n2g_d = n2g.cuda()
    out, packed = _packed_run(lambda: layer.table_update(h, g, graph_plan(n2g_d, G)))
    assert torch.equal(out, _twice(lambda: layer.table_update(h, g, graph_plan(n2g_d, G)))), "chained and plain outputs differ"
    want = _packed_split(out.cpu())
    assert torch.equal(packed.cpu().view(torch.int16), want.view(torch.int16)), "packed rows differ from the split of the output"


# ---- the whole GruGlobalStateUpdate: readout -> table -> GRU ---------------------------------------------------------------
def _global_case(H, N, bf16):
    gen = torch.Generator().manual_seed(N * 3 + H + bf16)
    G = max(1, (N + 499) // 500)
    n2g = torch.randint(0, G, (N,), generator=gen)
    G = int(n2g.max()) + 1
    h = torch.randn(N, H, generator=gen) * 0.5
    h = h.to(torch.bfloat16) if bf16 else h
    layer, w, p = _global_layer(H, N + H + 1, "weighted")
    hd, n2g_d = h.cuda(), n2g.cuda()
    got = _twice(lambda: layer(hd, [], n2g_d, {}, {}, []))
    g64, e_g, _ = GX.readout_bound(h.double(), n2g, G, "weighted", w.double())
    ref, bound = _table_ref(g64, e_g, n2g, h, p, bf16)
    family = f"global layer {'bf16' if bf16 else 'fp32'}"
    _check(got, ref, bound, family, f"{family} H={H} N={N}")


@pytest.mark.parametrize("H", [64, 128, 256])
@pytest.mark.parametrize("N", N_ROWS)
def test_global_layer_fp32(N, H):
    _global_case(H, N, False)


@pytest.mark.parametrize("H", [64, 128, 256])
@pytest.mark.parametrize("N", [1, 65, 1000, 40_000])
def test_global_layer_bf16(N, H):
    _global_case(H, N, True)


def test_zz_report_worst():
    """Prints the largest error / bound ratio per family (run with -s)."""
    if not WORST:
        pytest.skip("no bound-checked case ran in this session")
    for k in sorted(WORST):
        print(f"worst error/bound {k:>28}: {WORST[k]:.3f}")
    assert all(v <= 1.0 for v in WORST.values())
