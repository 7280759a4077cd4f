"""The fused aggregation kernel (csrc/fused_mp.cu) at its structural edges, element by element against a float64 reference with
a derived error bound per element (tests/fused_reference.py).

Graphs come from ``fused_reference.structured_graph`` (every MMA width, sub-group sizes 16k and 16k +- 1, lower/upper splits
at 0, n and off the 16-column batches, segments across batches and sub-groups, empty blocks, a partial last block), run at
explicit block sizes through ``EdgePlan(block_targets=B)``: B = 8 with 2,500 blocks (about 19 per CTA) and B = 24 / 88
(half a block is not a multiple of 8).  The layer is an ``MlpMessagePassingLayer`` without LayerNorm or dense layer, so its
output is the kernel's aggregate (through the activation, where one is set).  Every case runs twice and must be
bit-identical."""
import functools

import pytest
import torch

import fused_reference as R
import unfused_reference as UR
from helpers import gated_oracle_args

pytestmark = pytest.mark.gpu

AGGS = ("sum", "mean", "max", "min")
ACTS = {None: None, "gelu": torch.nn.GELU, "tanh": torch.nn.Tanh, "relu": torch.nn.ReLU}
T_DEFAULT = 6
BLOCKS = {8: 2500, 24: 800, 88: 400}
WORST = {}          # instance family -> largest error / bound ratio seen (printed with -s)


@functools.lru_cache(maxsize=4)
def _graph(B, T=T_DEFAULT, num_blocks=None):
    adj, N = R.structured_graph(B, T, num_blocks or BLOCKS[B])
    return adj, [(s.cuda(), t.cuda()) for s, t in adj], N


def _states(N, K, bf16, scale, seed, positive=False):
    h = torch.randn(N, K, generator=torch.Generator().manual_seed(seed))
    if positive:
        h = h.abs()
    h = h * scale                                # a power of two: the fp32 values keep their full mantissa
    return h.to(torch.bfloat16) if bf16 else h


def _mlp(K, T, agg, ut, act=None, ln=False, seed=0, negative_weights=False):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    layer = P.MlpMessagePassingLayer(K, 128, 128, T, agg, message_activation=ACTS[act]() if act else None, use_layer_norm=ln,
                                     use_dense_layer=False, use_target_state_as_message_input=ut).cuda().eval()
    if negative_weights:
        with torch.no_grad():
            for p in layer.parameters():
                if p.dim() == 2:
                    p.copy_(-p.abs())
    p = "_MlpMessagePassingLayer__"
    sd = layer.state_dict()
    w = [sd[f"{p}edge_message_transformation_layers.{t}._MLP__mlp_modules.1.weight"].cpu() for t in range(T)]
    return layer, w


def _run(layer, h, adj_d, N, B):
    """The layer's output on an explicit block size, twice: returns the first output after checking the second is identical."""
    import ptgnn_b200 as P

    outs = []
    for _ in range(2):
        plan = P.EdgePlan(adj_d, N, block_targets=B)
        with torch.no_grad(), P.edgeplan.shared_plan(plan):
            outs.append(layer(h.cuda(), adj_d))
        plan.validate()                          # no index or fp16-range flag
        assert plan.block_targets == B
    assert torch.equal(outs[0], outs[1]), "fused aggregate is not run-to-run bit-identical"
    return outs[0].float().cpu()


@functools.lru_cache(maxsize=2)
def _messages(bf16, K, ut, B, scale, seed):
    adj, _, N = _graph(B)
    h = _states(N, K, bf16, scale, seed)
    _, w = _mlp(K, T_DEFAULT, "sum", ut, seed=seed)
    return h, R.messages(h, adj, w, ut, bf16)


def _check(got, ref, bound, family, what):
    ratio = R.check_bound(got, ref, bound, what)
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    return ratio


# ---- all 40 instances: {fp32 K 64 / 128, bf16 K 64 / 128 / 256} x use_target x reduction, at two block sizes --------------
INSTANCES = [(bf16, K, ut, agg) for bf16, Ks in ((False, (64, 128)), (True, (64, 128, 256))) for K in Ks for ut in (False, True)
             for agg in AGGS]


@pytest.mark.parametrize("bf16,K,ut,agg", INSTANCES,
                         ids=[f"{'bf16' if b else 'fp32'}-K{K}-{'tgt' if u else 'src'}-{a}" for b, K, u, a in INSTANCES])
def test_fused_aggregate_instance(bf16, K, ut, agg):
    family = f"{'bf16' if bf16 else 'fp32'} {agg}"
    for B, scale in ((8, 1.0), (88 if ut else 24, 2.0 ** -12 if K != 128 else 2.0 ** 8)):
        adj, adj_d, N = _graph(B)
        seed = K + 2 * ut + B
        h, (tgt, m, err) = _messages(bf16, K, ut, B, scale, seed)
        layer, _ = _mlp(K, T_DEFAULT, agg, ut, seed=seed)
        got = _run(layer, h, adj_d, N, B)
        ref, bound, _ = R.aggregate(tgt, m, err, N, agg, bf16)
        _check(got, ref, bound, family, f"{family} K={K} use_target={ut} B={B} scale={scale}")


# ---- more blocks per CTA at the largest block: 2+ waves, and a block count of 132 k + 1 --------------------------------------
@pytest.mark.parametrize("bf16,agg,explicit", [(False, "mean", False), (False, "min", True), (True, "sum", True), (True, "max", False)])
def test_fused_aggregate_block176_waves(bf16, agg, explicit):
    import ptgnn_b200 as P

    num_blocks = 2 * 132 + 1 if explicit else 256
    adj, adj_d, N = _graph(176, 4, num_blocks)
    assert N > 23_232
    if not explicit:
        assert int(P._native.lib().ptgnn_b200_block_plan_block_targets(N)) == 176
    h = _states(N, 128, bf16, 1.0, 7)
    layer, w = _mlp(128, 4, agg, True, seed=7)
    got = _run(layer, h, adj_d, N, 176)
    ref, bound, _ = R.aggregate(*R.messages(h, adj, w, True, bf16), N, agg, bf16)
    _check(got, ref, bound, f"{'bf16' if bf16 else 'fp32'} {agg}", f"B=176 blocks={num_blocks} {agg}")


# ---- T = 128 edge types (PTGNN_MAX_EDGE_TYPES) ---------------------------------------------------------------------------------
@pytest.mark.parametrize("bf16,agg", [(False, "sum"), (True, "max")])
def test_fused_aggregate_128_types(bf16, agg):
    adj, adj_d, N = _graph(8, 128, 400)
    h = _states(N, 64, bf16, 1.0, 12)
    layer, w = _mlp(64, 128, agg, False, seed=12)
    got = _run(layer, h, adj_d, N, 8)
    ref, bound, _ = R.aggregate(*R.messages(h, adj, w, False, bf16), N, agg, bf16)
    _check(got, ref, bound, f"{'bf16' if bf16 else 'fp32'} {agg}", f"T=128 {agg}")


# ---- inputs at the edges of the ranges -----------------------------------------------------------------------------------
@pytest.mark.parametrize("bf16,agg", [(False, "max"), (False, "min"), (True, "max"), (True, "min")])
def test_fused_aggregate_negative_messages(bf16, agg):
    """Every message negative: max must not mistake a real value for the identity, min must reach below it."""
    adj, adj_d, N = _graph(8)
    h = _states(N, 128, bf16, 1.0, 21, positive=True)
    layer, w = _mlp(128, T_DEFAULT, agg, False, seed=21, negative_weights=True)
    tgt, m, err = R.messages(h, adj, w, False, bf16)
    assert float(m.max()) < 0
    got = _run(layer, h, adj_d, N, 8)
    ref, bound, _ = R.aggregate(tgt, m, err, N, agg, bf16)
    _check(got, ref, bound, f"{'bf16' if bf16 else 'fp32'} {agg}", f"negative messages {agg}")


@pytest.mark.parametrize("agg", ["sum", "max"])
def test_fused_aggregate_near_fp16_limit(agg):
    """fp32 states up to ~ +-60,000 (below 65,504): the 3xFP16 split holds them and no status flag is raised."""
    adj, adj_d, N = _graph(24)
    h = (_states(N, 128, False, 2.0 ** 14, 31)).clamp(-60_000.0, 60_000.0)
    assert float(h.abs().max()) >= 50_000
    layer, w = _mlp(128, T_DEFAULT, agg, True, seed=31)
    got = _run(layer, h, adj_d, N, 24)
    ref, bound, _ = R.aggregate(*R.messages(h, adj, w, True, False), N, agg, False)
    _check(got, ref, bound, f"fp32 {agg}", f"|h| <= 60000 {agg}")


# ---- epilogues ---------------------------------------------------------------------------------------------------------------
EPI = [(bf16, act, agg) for bf16 in (False, True) for act, agg in (("gelu", "sum"), ("tanh", "max"), ("relu", "mean"))]


@pytest.mark.parametrize("bf16,act,agg", EPI, ids=[f"{'bf16' if b else 'fp32'}-{a}-{g}" for b, a, g in EPI])
def test_fused_activation_epilogue(bf16, act, agg):
    """The activation without LayerNorm (write_out_block's split-row path with act != NONE), bound-checked."""
    adj, adj_d, N = _graph(8)
    h = _states(N, 128, bf16, 1.0, 41)
    layer, w = _mlp(128, T_DEFAULT, agg, True, act=act, seed=41)
    got = _run(layer, h, adj_d, N, 8)
    ref, bound, _ = R.aggregate(*R.messages(h, adj, w, True, bf16), N, agg, bf16, act=act)
    _check(got, ref, bound, f"{'bf16' if bf16 else 'fp32'} {act}", f"{act} epilogue {agg}")


LN = [(bf16, act, agg) for bf16 in (False, True) for act, agg in ((None, "sum"), ("gelu", "max"), ("gelu", "mean"))]


@pytest.mark.parametrize("bf16,act,agg", LN, ids=[f"{'bf16' if b else 'fp32'}-{a}-{g}" for b, a, g in LN])
def test_fused_layernorm_epilogue(bf16, act, agg):
    """LayerNorm (whole-row write-out) with and without an activation, and after a mean: the aggregate's bound carried through the
    activation and LayerNorm (unfused_reference.layer_norm), then the bf16 rounding."""
    adj, adj_d, N = _graph(24)
    h = _states(N, 128, bf16, 1.0, 51)
    layer, w = _mlp(128, T_DEFAULT, agg, True, act=act, ln=True, seed=51)
    with torch.no_grad():
        for p in layer.parameters():
            if p.dim() == 1:
                p.uniform_(0.5, 1.5, generator=torch.Generator(device="cuda").manual_seed(p.numel()))
    sd = {k: v.double().cpu() for k, v in layer.state_dict().items()}
    ln_w, ln_b = sd["_MlpMessagePassingLayer__state_update.0.weight"], sd["_MlpMessagePassingLayer__state_update.0.bias"]
    got = _run(layer, h, adj_d, N, 24)
    y, by, _ = R.aggregate(*R.messages(h, adj, w, True, bf16), N, agg, bf16, act=act, round_bf16=False)
    ref, bound = UR.layer_norm(y, by, ln_w, ln_b, 1e-5)
    if bf16:
        ref, bound = UR.round_bf16(ref, bound)
    _check(got, ref, bound, f"{'bf16' if bf16 else 'fp32'} LayerNorm", f"LayerNorm act={act} {agg}")


# ---- the gated layer on the same graphs: aggregate (fp32: out_mode 2) -> weights-stationary GRU, bound through the GRU --------
@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("agg", AGGS)
def test_fused_gated_structured(agg, bf16):
    import ptgnn_b200 as P

    adj, adj_d, N = _graph(8)
    h = _states(N, 128, bf16, 0.5, 61)
    torch.manual_seed(61)
    layer = P.GatedMessagePassingLayer(128, 128, T_DEFAULT, agg).cuda().eval()
    args = gated_oracle_args({k: v.clone().cpu() for k, v in layer.state_dict().items()})
    got = _run(layer, h, adj_d, N, 8)
    x, ex, _ = R.aggregate(*R.messages(h, adj, args["edge_weights"], False, bf16), N, agg, bf16)
    if not bf16:
        assert float(x.abs().max()) < 65504           # the fp16 (hi | lo') aggregate holds it: no status flag (checked in _run)
    ref, bound = UR.gru(x.cuda(), ex.cuda(), h.cuda(), *(args[k] for k in ("gru_w_ih", "gru_w_hh", "gru_b_ih", "gru_b_hh")),
                        mode="bf16" if bf16 else "3xfp16")
    _check(got, ref.cpu(), bound.cpu(), f"{'bf16' if bf16 else 'fp32'} gated", f"gated {agg}")


# ---- regression: a block with edges followed by three blocks without edges in one CTA's round-robin order ----------------------
@pytest.mark.parametrize("bf16,agg", [(False, "sum"), (True, "max")])
def test_regression_sched_ring_deadlock_on_empty_blocks(bf16, agg):
    """Each CTA owns six blocks here; only its first and fifth have edges.  The gatherers used to look up the step after the
    last one of block 1 before publishing that step's data, and the look-up waited, past blocks 2-4, for a scheduler ring entry
    that the consumers release only after that data: the kernel trapped.  A step is now published before the look-up."""
    B, per_cta = 8, 6
    N = B * 132 * per_cta
    gen = torch.Generator().manual_seed(71)
    blocks = torch.cat([torch.arange(132), torch.arange(132) + 4 * 132])
    adj = []
    for _ in range(2):
        tgt = blocks[torch.randint(0, blocks.shape[0], (6000,), generator=gen)] * B + torch.randint(0, B, (6000,), generator=gen)
        adj.append((torch.randint(0, N, (6000,), generator=gen), tgt))
    adj_d = [(s.cuda(), t.cuda()) for s, t in adj]
    h = _states(N, 128, bf16, 1.0, 71)
    layer, w = _mlp(128, 2, agg, True, seed=71)
    got = _run(layer, h, adj_d, N, B)
    ref, bound, _ = R.aggregate(*R.messages(h, adj, w, True, bf16), N, agg, bf16)
    _check(got, ref, bound, f"{'bf16' if bf16 else 'fp32'} {agg}", f"empty-block runs {agg}")


def test_zz_report_worst_ratios():
    """Prints the largest error / bound ratio per instance family (run with -s); fails if a bound was never exercised."""
    if not WORST:
        pytest.skip("no bound-checked case ran in this session")
    for k in sorted(WORST):
        print(f"worst error/bound {k:>12}: {WORST[k]:.3f}")
    assert all(v <= 1.0 for v in WORST.values())
