"""The unfused layer kernels at their tile edges, element by element against a float64 reference with a derived error bound
per element (tests/unfused_reference.py): the 3xTF32 message, GRU and dense pipelines, their bf16 versions, the FFMA
kernels and both segmented reduces.

Operators run through their stand-alone entry points (``composed.edge_messages / segment_reduce / grucell / linear``,
``scatter``) so that any (H, D, N) can be reached; the bf16 kernels and the reduce epilogue through layers at shapes the
fused kernel does not take (or the fused path where it does), fp32 layers at H = D = 128 with PTGNN_B200_FP32_MODE=tf32.  The
shape alone picks the tensor-core or the FFMA kernels (``unfused_reference.fp32_*_mode``); the FFMA cases use shapes that fit
no tensor-core tile.  Graphs come from ``unfused_reference.structured_graph``: per-type edge counts at the 128-edge tile
boundary between large types, >= 3 waves of tiles, a hub, runs of empty rows placed against the streaming reduce's 16-row warp blocks, N = 0 / +-1 (mod 16) and (mod 128).  Before each call a block of
memory is filled with NaN and freed, so that the caching allocator hands NaN back and an element no kernel wrote shows.
Every case runs twice and must be bit-identical (no float atomics on these paths)."""
import functools
import math

import pytest
import torch

import fused_reference as FR
import unfused_reference as R
from helpers import gated_oracle_args

pytestmark = pytest.mark.gpu
NODES = (12800, 12801, 12799, 12816)
ACTS = {None: None, "gelu": torch.nn.GELU, "tanh": torch.nn.Tanh, "relu": torch.nn.ReLU}
AGGS = ("sum", "mean", "max", "min")
WORST = {}          # kernel family -> largest error / bound ratio seen (printed with -s)
NAN_BITS = 0x7FC07FC0   # NaN as one fp32 word and as both of its bf16 halves


def _with_nodes(cases):
    """Appends a node count to each case, cycling through NODES by case index: every table of four or more cases runs at
    N = 0, 1 and -1 (mod 16 and mod 128); shorter tables start with N = 0 and N = 1."""
    out = [tuple(c) + (NODES[i % len(NODES)],) for i, c in enumerate(cases)]
    assert {n % 128 for *_, n in out} >= ({0, 1, 127} if len(out) >= 4 else {0, 1})
    return out


@functools.lru_cache(maxsize=4)
def _graph(N):
    adj, _ = R.structured_graph(N)
    return adj, [(s.cuda(), t.cuda()) for s, t in adj]


def _poison(nbytes):
    """Leave a NaN-filled block of at least nbytes in the caching allocator (best effort: later allocations are carved
    from it)."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    t = torch.full((nbytes // 4 + (1 << 20),), NAN_BITS, dtype=torch.int32, device="cuda")
    del t


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else (torch.int64 if t.element_size() == 8 else torch.int32))


def _twice(fn, nbytes):
    """fn() twice, each after poisoning nbytes: both results must be bit-identical; returns the first."""
    outs = []
    for _ in range(2):
        _poison(nbytes)
        with torch.no_grad():
            r = fn()
        torch.cuda.synchronize()
        outs.append(r if isinstance(r, tuple) else (r,))
    for a, b in zip(*outs):
        assert torch.equal(_bits(a), _bits(b)), "not run-to-run bit-identical"
    return outs[0] if len(outs[0]) > 1 else outs[0][0]


def _check(got, ref, bound, family, what):
    ratio = FR.check_bound(got.float() if got.dtype == torch.bfloat16 else got, ref.cpu(), bound.cpu(), what)
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    return ratio


def _weights(T, D, K, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(D, K, generator=g) / math.sqrt(K) for _ in range(T)]


def _states(N, H, seed, scale=1.0):
    return torch.randn(N, H, generator=torch.Generator().manual_seed(seed)) * scale


# ---- fp32 messages ---------------------------------------------------------------------------------------------------
MSG = _with_nodes([(32, 16, False), (36, 48, True), (44, 112, True), (100, 144, True), (128, 240, False), (132, 272, True),
                   (256, 512, False), (36, 512, False)])


def _fp32_messages_case(H, D, ut, N, seed):
    import ptgnn_b200 as P
    from ptgnn_b200 import composed as C

    adj, adj_d = _graph(N)
    h = _states(N, H, seed)
    w = _weights(len(adj), D, 2 * H if ut else H, seed)
    plan = P.EdgePlan(adj_d, N)
    hd, wd = h.cuda(), [x.cuda() for x in w]
    got = _twice(lambda: C.edge_messages(plan, hd, hd if ut else None, wd, ut), plan.num_edges * D * 4 * 2)
    _, m, err = R.fp32_messages(h, adj, w, ut, device="cuda")
    _check(got.cpu(), m, err, f"fp32 messages ({R.fp32_message_mode(H, D)})", f"messages H={H} D={D} ut={ut} N={N}")


@pytest.mark.parametrize("H,D,ut,N", MSG, ids=[f"H{h}-D{d}-{'tgt' if u else 'src'}-N{n}" for h, d, u, n in MSG])
def test_fp32_messages(H, D, ut, N):
    _fp32_messages_case(H, D, ut, N, H + D)


# the FFMA message kernel: D % 16 != 0, 4- vs 8-wide tiles (D <= 64 vs > 64), K tails of the 32-wide k-chunk
FFMA_MSG = _with_nodes([(36, 20, True), (44, 36, False), (100, 68, True), (4, 100, False), (132, 260, False)])


@pytest.mark.parametrize("H,D,ut,N", FFMA_MSG)
def test_ffma_messages(H, D, ut, N):
    _fp32_messages_case(H, D, ut, N, H + D)


# ---- fp32 segmented reduce: per-row kernel (D <= 64, or with args) and streaming kernel (D > 64) ------------------------
REDUCE_D = (4, 32, 36, 64, 68, 128, 132, 256, 260, 512)


def _reduce_inputs(D, N):
    adj, _ = _graph(N)
    tgt = torch.cat([t for _, t in adj])
    g = torch.Generator().manual_seed(D)
    m = torch.randn(tgt.shape[0], D, generator=g)
    m[:, ::2] = torch.round(m[:, ::2] * 2) / 2                      # even columns: few distinct values, many exact ties
    return tgt, m


# every D at every node count (one per reduction), every reduction at every node count
REDUCE = [(agg, D, NODES[(i + j) % len(NODES)]) for j, agg in enumerate(AGGS) for i, D in enumerate(REDUCE_D)]


@pytest.mark.parametrize("reduce,D,N", REDUCE, ids=[f"{a}-D{d}-N{n}" for a, d, n in REDUCE])
def test_fp32_reduce_exact(reduce, D, N):
    import ptgnn_b200 as P
    from ptgnn_b200 import _native as NA
    from ptgnn_b200 import composed as C

    _, adj_d = _graph(N)
    tgt, m = _reduce_inputs(D, N)
    ref, ref_arg = R.reduce_exact(tgt, m, N, reduce)
    plan = P.EdgePlan(adj_d, N)
    md = m.cuda()
    code = NA.REDUCE[reduce]
    nbytes = N * D * 12
    got = _twice(lambda: C.segment_reduce(md, plan, code), nbytes)
    assert torch.equal(got.cpu(), ref), f"{reduce} D={D}: not bit-exact"
    if reduce in ("max", "min"):
        val, arg = _twice(lambda: C.segment_reduce(md, plan, code, return_arg=True), nbytes)
        assert torch.equal(val.cpu(), ref) and torch.equal(arg.cpu(), ref_arg), f"{reduce} D={D} with args"
    # torch_scatter drop-in: unsorted index, one edge type -> its own plan and the perm path
    idx = tgt.cuda()
    if reduce in ("max", "min"):
        fn = P.scatter_max if reduce == "max" else P.scatter_min
        val, arg = _twice(lambda: fn(md, idx, dim=0, dim_size=N), nbytes)
        assert torch.equal(val.cpu(), ref) and torch.equal(arg.cpu(), ref_arg), f"scatter_{reduce} D={D}"
    else:
        out = _twice(lambda: P.scatter(md, idx, dim=0, dim_size=N, reduce=reduce), nbytes)
        assert torch.equal(out.cpu(), ref), f"scatter {reduce} D={D}: not bit-exact"


# ---- layers: shared helpers ------------------------------------------------------------------------------------------
def _mlp(H, D, Hout, T, agg, ut, act=None, ln=False, dense=False, dense_act=None, seed=0):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    layer = P.MlpMessagePassingLayer(H, Hout if dense else D, D, T, agg, message_activation=ACTS[act]() if act else None,
                                     use_layer_norm=ln, use_dense_layer=dense, use_target_state_as_message_input=ut,
                                     dense_activation=ACTS[dense_act]() if dense_act else None).cuda().eval()
    p = "_MlpMessagePassingLayer__"
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():                                           # LayerNorm scales away from 1, biases away from 0
        for name, t in layer.named_parameters():
            if t.dim() == 1:
                lo, hi = (0.5, 1.5) if ln and name == f"{p}state_update.0.weight" else (-0.5, 0.5)
                t.uniform_(lo, hi, generator=g)
    sd = {k: v.detach().cpu() for k, v in layer.state_dict().items()}
    w = [sd[f"{p}edge_message_transformation_layers.{t}._MLP__mlp_modules.1.weight"] for t in range(T)]
    extra = {}
    i = 0
    if ln:
        extra["ln"] = (sd[f"{p}state_update.0.weight"], sd[f"{p}state_update.0.bias"])
        i = 1
    if dense:
        extra["dense"] = (sd[f"{p}state_update.{i}.weight"], sd[f"{p}state_update.{i}.bias"])
    return layer, w, extra


def _layer_run(layer, h, adj_d, nbytes):
    return _twice(lambda: layer(h.cuda(), adj_d), nbytes).cpu()


def _msg_bytes(N, E, D, bf16):
    return (E + 2 * N) * D * (2 if bf16 else 4) + (64 << 20)


# ---- reduce epilogue (activation + LayerNorm) on both fp32 reduce kernels ---------------------------------------------
EPI = _with_nodes([(16, None, "sum"), (32, "gelu", "mean"), (48, "tanh", "max"), (64, "relu", "min"), (96, "gelu", "sum"),
                   (132, "tanh", "mean"), (260, "relu", "max")])


@pytest.mark.parametrize("D,act,agg,N", EPI, ids=[f"D{d}-{a}-{g}-N{n}" for d, a, g, n in EPI])
def test_fp32_reduce_epilogue_layer_norm(D, act, agg, N):
    adj, adj_d = _graph(N)
    H, ut = 64, D % 32 == 0
    layer, w, extra = _mlp(H, D, D, len(adj), agg, ut, act=act, ln=True, seed=D)
    h = _states(N, H, D)
    got = _layer_run(layer, h, adj_d, _msg_bytes(N, 60_000, D, False))
    tgt, m, err = R.fp32_messages(h, adj, w, ut, device="cuda")
    _, bnd, pre = FR.aggregate(tgt, m, err, N, agg, False)
    x, bx = FR.activation_bound(pre, bnd, act)
    y, by = R.layer_norm(x, bx, *extra["ln"], 1e-5)
    _check(got, y, by, f"fp32 reduce+LayerNorm ({R.fp32_message_mode(H, D)})", f"LayerNorm D={D} act={act} {agg}")


# ---- bf16 messages + bf16 streaming reduce ---------------------------------------------------------------------------
BF16_MSG = _with_nodes([(64, 64, "sum"), (64, 80, "mean"), (128, 112, "sum"), (96, 128, "max"), (128, 144, "min"),
                        (64, 176, "sum"), (128, 240, "mean"), (64, 256, "max")])


@pytest.mark.parametrize("H,D,agg,N", BF16_MSG, ids=[f"H{h}-D{d}-{a}-N{n}" for h, d, a, n in BF16_MSG])
def test_bf16_messages_and_reduce(H, D, agg, N):
    adj, adj_d = _graph(N)
    ut = D % 32 == 16
    layer, w, _ = _mlp(H, D, D, len(adj), agg, ut, seed=D + 1)
    h = _states(N, H, D + 1).to(torch.bfloat16)
    got = _layer_run(layer, h, adj_d, _msg_bytes(N, 60_000, D, True))
    ref, bound, _ = FR.aggregate(*FR.messages(h, adj, w, ut, True), N, agg, True)
    _check(got, ref, bound, "bf16 messages+reduce", f"bf16 D={D} H={H} {agg}")


# ---- bf16 reduce epilogue: activation + LayerNorm in fp32 on the fp32 aggregate, one rounding to bf16 ------------------
BF16_EPI = _with_nodes([(64, 112, "gelu", "sum"), (128, 176, "tanh", "max"), (64, 256, "relu", "mean"), (128, 64, None, "min")])


@pytest.mark.parametrize("H,D,act,agg,N", BF16_EPI, ids=[f"H{h}-D{d}-{a}-{g}-N{n}" for h, d, a, g, n in BF16_EPI])
def test_bf16_reduce_epilogue_layer_norm(H, D, act, agg, N):
    adj, adj_d = _graph(N)
    ut = D % 32 == 0
    layer, w, extra = _mlp(H, D, D, len(adj), agg, ut, act=act, ln=True, seed=D + 3)
    h = _states(N, H, D + 3).to(torch.bfloat16)
    got = _layer_run(layer, h, adj_d, _msg_bytes(N, 60_000, D, True))
    _, bnd, pre = FR.aggregate(*FR.messages(h, adj, w, ut, True), N, agg, True, round_bf16=False)
    x, bx = FR.activation_bound(pre, bnd, act)
    ref, bound = R.round_bf16(*R.layer_norm(x, bx, *extra["ln"], 1e-5))
    _check(got, ref, bound, "bf16 reduce+LayerNorm", f"bf16 LayerNorm H={H} D={D} act={act} {agg}")


# ---- fp32 GRU ----------------------------------------------------------------------------------------------------------
MULTI_WAVE = 3 * R.SM_COUNT * R.TILE_M + 1                      # H = 32: 3 waves of row tiles + a 1-row tile
GRU = [(32, 36, MULTI_WAVE), (64, 32, 1), (96, 100, 127), (160, 200, 128), (256, 36, 129), (512, 100, 1000), (32, 200, 129)]


def _fp32_gru_case(H, D, N, seed):
    from ptgnn_b200 import composed as C

    torch.manual_seed(seed)
    cell = torch.nn.GRUCell(D, H)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        cell.bias_ih.uniform_(-0.5, 0.5, generator=g)
        cell.bias_hh.uniform_(-0.5, 0.5, generator=g)
    p = [t.detach().clone() for t in (cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh)]
    cell = cell.cuda()
    x, h = _states(N, D, seed, 2.0), _states(N, H, seed + 1)
    xd, hd = x.cuda(), h.cuda()
    got = _twice(lambda: C.grucell(xd, hd, cell), N * H * 4 * 4 + (64 << 20))
    mode = R.fp32_gru_mode(H, D)
    ref, bound = R.gru(xd.double(), None, hd, *p, mode=mode)
    _check(got.cpu(), ref, bound, f"fp32 GRU ({mode})", f"GRU H={H} D={D} N={N}")


@pytest.mark.parametrize("H,D,N", GRU)
def test_fp32_gru(H, D, N):
    _fp32_gru_case(H, D, N, H + D + N)


@pytest.mark.parametrize("H,D,N", [(32, 20, 129), (64, 28, 127), (96, 12, 12800)])   # D < 32: the FFMA GRU
def test_ffma_gru(H, D, N):
    _fp32_gru_case(H, D, N, H + D)


# ---- bf16 GRU (gated layer, unfused) ---------------------------------------------------------------------------------
BF16_GRU = _with_nodes([(64, 112, "sum"), (96, 176, "max"), (160, 240, "mean"), (256, 80, "min")])


@pytest.mark.parametrize("H,D,agg,N", BF16_GRU, ids=[f"H{h}-D{d}-{a}-N{n}" for h, d, a, n in BF16_GRU])
def test_bf16_gated_layer(H, D, agg, N):
    import ptgnn_b200 as P

    adj, adj_d = _graph(N)
    torch.manual_seed(H)
    layer = P.GatedMessagePassingLayer(H, D, len(adj), agg).cuda().eval()
    with torch.no_grad():
        for b in (layer.state_dict(keep_vars=True)[f"_GatedMessagePassingLayer__state_update.bias_{k}"] for k in ("ih", "hh")):
            b.uniform_(-0.5, 0.5)
    args = gated_oracle_args({k: v.detach().cpu() for k, v in layer.state_dict().items()})
    h = _states(N, H, H, 0.5).to(torch.bfloat16)
    got = _layer_run(layer, h, adj_d, _msg_bytes(N, 60_000, max(D, 4 * H), True))
    agg_ref, agg_bnd, _ = FR.aggregate(*FR.messages(h, adj, args["edge_weights"], False, True), N, agg, True)
    ref, bound = R.gru(agg_ref.cuda(), agg_bnd.cuda(), h.cuda(), args["gru_w_ih"], args["gru_w_hh"], args["gru_b_ih"],
                       args["gru_b_hh"], mode="bf16")
    _check(got, ref, bound, "bf16 GRU layer", f"bf16 gated H={H} D={D} {agg}")


# ---- fp32 dense ------------------------------------------------------------------------------------------------------
DENSE = _with_nodes([(36, 16, True, None), (100, 48, False, "gelu"), (68, 112, True, "tanh"), (132, 144, True, "relu"),
                     (260, 272, False, None), (36, 4, True, "gelu"), (100, 20, False, "relu"), (68, 36, True, "tanh")])


def _fp32_dense_case(D, Hout, bias, act, N, seed):
    from ptgnn_b200 import composed as C

    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, D, generator=g)
    W = torch.randn(Hout, D, generator=g) / math.sqrt(D)
    b = torch.randn(Hout, generator=g) if bias else None
    xd, Wd, bd = x.cuda(), W.cuda(), None if b is None else b.cuda()
    mod = ACTS[act]() if act else None
    got = _twice(lambda: C.linear(xd, Wd, bd, mod), N * (Hout + 4) * 4 + (64 << 20))
    mode = R.fp32_dense_mode(D, Hout)
    ref, bound = R.dense(xd.double(), None, W, b, act, mode)
    _check(got.cpu(), ref, bound, f"fp32 dense ({mode})", f"dense D={D} Hout={Hout} bias={bias} act={act}")


@pytest.mark.parametrize("D,Hout,bias,act,N", DENSE)
def test_fp32_dense(D, Hout, bias, act, N):
    _fp32_dense_case(D, Hout, bias, act, N, D + Hout)


@pytest.mark.parametrize("D,Hout,N", _with_nodes([(20, 68), (36, 100), (4, 36), (100, 4)]))
def test_ffma_dense(D, Hout, N):
    _fp32_dense_case(D, Hout, True, "gelu", N, D + Hout + 1)


# ---- bf16 dense (Mlp layer with a dense layer at D = 128: fused aggregation at H = 64, unfused at H = 96) -------------------
BF16_DENSE = _with_nodes([(64, True, "sum"), (112, True, "max"), (112, False, "sum"), (176, False, "max"), (240, True, "max"),
                          (240, False, "sum"), (304, True, "sum"), (304, False, "max")])


@pytest.mark.parametrize("Hout,fused,agg,N", BF16_DENSE,
                         ids=[f"Hout{h}-{'fused' if f else 'unfused'}-{a}-N{n}" for h, f, a, n in BF16_DENSE])
def test_bf16_dense(Hout, fused, agg, N):
    adj, adj_d = _graph(N)
    H, D = 64 if fused else 96, 128
    layer, w, extra = _mlp(H, D, Hout, len(adj), agg, True, dense=True, dense_act="tanh", seed=Hout)
    h = _states(N, H, Hout).to(torch.bfloat16)
    got = _layer_run(layer, h, adj_d, _msg_bytes(N, 60_000, max(D, Hout), True))
    y, by, _ = FR.aggregate(*FR.messages(h, adj, w, True, True), N, agg, True)
    ref, bound = R.dense(y.cuda(), by.cuda(), *extra["dense"], "tanh", "bf16")
    _check(got, ref, bound, "bf16 dense", f"bf16 dense Hout={Hout} fused={fused} {agg}")


# ---- fp32 layers on the structured graph: bounds composed from the operator bounds --------------------------------------
# H = D = 128 (the fused kernel's shape) on the 3xTF32 kernels under PTGNN_B200_FP32_MODE=tf32; D = 20: FFMA messages and GRU
GATED = _with_nodes([(128, 128, True, agg) for agg in AGGS] + [(64, 20, False, "sum")])


@pytest.mark.parametrize("H,D,tf32,agg,N", GATED, ids=[f"H{h}-D{d}{'-tf32' if t else ''}-{a}-N{n}" for h, d, t, a, n in GATED])
def test_fp32_layers_gated(monkeypatch, H, D, tf32, agg, N):
    import ptgnn_b200 as P

    if tf32:
        monkeypatch.setenv("PTGNN_B200_FP32_MODE", "tf32")
    adj, adj_d = _graph(N)
    torch.manual_seed(7)
    layer = P.GatedMessagePassingLayer(H, D, len(adj), agg).cuda().eval()
    args = gated_oracle_args({k: v.detach().cpu() for k, v in layer.state_dict().items()})
    h = _states(N, H, 7, 0.5)
    got = _layer_run(layer, h, adj_d, _msg_bytes(N, 60_000, 4 * H, False))
    tgt, m, err = R.fp32_messages(h, adj, args["edge_weights"], False, device="cuda")
    _, bnd, pre = FR.aggregate(tgt, m, err, N, agg, False)
    ref, bound = R.gru(pre.cuda(), bnd.cuda(), h.cuda(), args["gru_w_ih"], args["gru_w_hh"], args["gru_b_ih"], args["gru_b_hh"],
                       mode=R.fp32_gru_mode(H, D))
    _check(got, ref, bound, f"fp32 gated layer ({R.fp32_message_mode(H, D)})", f"gated H={H} D={D} tf32={tf32} {agg}")


# the last case: FFMA messages (D % 16 != 0) and FFMA dense (Hout % 16 != 0)
@pytest.mark.parametrize("H,D,Hout,agg,N", _with_nodes([(64, 112, 144, "mean"), (36, 128, 48, "min"), (64, 64, 112, "max"),
                                                        (36, 36, 100, "sum")]))
def test_fp32_layers_mlp(H, D, Hout, agg, N):
    adj, adj_d = _graph(N)
    layer, w, extra = _mlp(H, D, Hout, len(adj), agg, True, act="gelu", ln=True, dense=True, dense_act="tanh", seed=H + D)
    h = _states(N, H, H + D)
    got = _layer_run(layer, h, adj_d, _msg_bytes(N, 60_000, max(D, Hout), False))
    tgt, m, err = R.fp32_messages(h, adj, w, True, device="cuda")
    _, bnd, pre = FR.aggregate(tgt, m, err, N, agg, False)
    x, bx = FR.activation_bound(pre, bnd, "gelu")
    y, by = R.layer_norm(x, bx, *extra["ln"], 1e-5)
    ref, bound = R.dense(y.cuda(), by.cuda(), *extra["dense"], "tanh", R.fp32_dense_mode(D, Hout))
    _check(got, ref, bound, f"fp32 Mlp layer ({R.fp32_message_mode(H, D)})", f"Mlp H={H} D={D} Hout={Hout} {agg}")


def test_zz_report_worst_ratios():
    """Prints the largest error / bound ratio per kernel family (run with -s)."""
    if not WORST:
        pytest.skip("no bound-checked case ran in this session")
    for k in sorted(WORST):
        print(f"worst error/bound {k:>32}: {WORST[k]:.3f}")
    assert all(v <= 1.0 for v in WORST.values())
