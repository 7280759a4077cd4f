"""GPU tests of the native classification heads (csrc/classify.cu, DESIGN.md §3.17): logits' logsumexps, losses, argmaxes, PPI counts and
metrics against the float64 restatement (tests/classification_heads_reference.py) at the kernel's structural edges, the backward, bf16,
PPI's predictions at the sigmoid threshold, determinism, the absence of host synchronisation, the refusals and one training step of a
native GNN with the head."""
import os
import sys

import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import classification_heads_reference as R  # noqa: E402

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200 import autograd as AG  # noqa: E402
from ptgnn_b200 import heads as HD  # noqa: E402
from ptgnn_b200 import edgeplan  # noqa: E402
from ptgnn_b200.gnn import GnnOutput  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
TAU = 5e-5


class StubGnn(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.output_node_state_dim = dim
        self.output = None

    def forward(self, **kwargs):
        return self.output


def gnn_output(h, idx=None, graph_idx=None):
    refs = {} if idx is None else {"supernodes": idx}
    grefs = {} if idx is None else {"supernodes": graph_idx if graph_idx is not None else torch.zeros_like(idx)}
    return GnnOutput(h, h, torch.zeros(h.shape[0], dtype=torch.int64, device=h.device), refs, grefs, 1)


def g2c_case(N_, H, C, S, seed, ignore=True):
    gen = torch.Generator().manual_seed(seed)
    h = torch.randn(N_, H, generator=gen)
    idx = torch.randint(0, N_, (S,), generator=gen)
    target = torch.randint(0, C, (S,), generator=gen)
    if ignore and S > 2:
        target[::7] = R.IGNORE_INDEX
    w = torch.randn(C, H, generator=gen) / H ** 0.5
    b = torch.randn(C, generator=gen) * 0.1
    return h, idx, target, w, b


def g2c_module(H, C, w, b):
    m = P.Graph2ClassModule(StubGnn(H), C).to(DEV)
    with torch.no_grad():
        m._Graph2ClassModule__node_to_class.weight.copy_(w)
        m._Graph2ClassModule__node_to_class.bias.copy_(b)
    return m


def ppi_module(H, C, w, b):
    m = P.PPIClassification(StubGnn(H), C).to(DEV)
    with torch.no_grad():
        m._PPIClassification__output_representation_to_logits.weight.copy_(w)
        m._PPIClassification__output_representation_to_logits.bias.copy_(b)
    return m


def run_g2c(m, h, idx, target):
    m._Graph2ClassModule__gnn.output = gnn_output(h.to(DEV), idx.to(DEV))
    return m(graph_mb_data={}, target_classes=target.to(DEV), original_supernode_idxs=None)


def run_ppi(m, h, t):
    m._PPIClassification__gnn.output = gnn_output(h.to(DEV))
    return m(graph_data={}, targets=t.to(DEV))


G2C_SHAPES = [(8, 1, 0), (8, 2, 1), (64, 101, 63), (64, 101, 64), (64, 129, 65), (128, 101, 129), (128, 256, 200), (256, 121, 65),
              (256, 128, 129), (256, 256, 64), (256, 2, 300)]


@pytest.mark.parametrize("H,C,S", G2C_SHAPES)
def test_graph2class_forward_within_bounds(H, C, S):
    h, idx, target, w, b = g2c_case(max(S, 1) * 2, H, C, S, seed=H * 1000 + C + S)
    m = g2c_module(H, C, w, b)
    with torch.no_grad():
        loss = float(run_g2c(m, h, idx, target))
        logits, _ = m._logits({})
        prob, arg, _ = m.predict({})
    z, zb = R.logits(h, idx, w, b), R.logit_bound(h, idx, w, b)
    assert bool(((logits.double().cpu() - z).abs() <= zb).all()), "logits outside the bound"
    ref_loss, lb, lse, ref_arg, hits, n = R.ce(z, zb, target)
    assert R.nan_or_close(loss, ref_loss, lb), (loss, ref_loss, lb)
    if S and R.ce_hits_decidable(z, zb):
        assert torch.equal(arg.cpu(), ref_arg)
        assert m.report_metrics()["Accuracy"] == hits / S
    if S:
        ref_prob = torch.softmax(z, dim=1).max(dim=1).values
        assert bool(((prob.double().cpu() - ref_prob).abs() <= 2.0 ** -20 + 4 * zb.max(dim=1).values * ref_prob).all())


PPI_SHAPES = [(64, 101, 0), (8, 1, 1), (64, 2, 63), (64, 101, 64), (128, 129, 65), (256, 121, 129), (256, 256, 64), (256, 121, 200_000)]


def ppi_case(R_, H, C, seed):
    gen = torch.Generator().manual_seed(seed)
    h = torch.randn(R_, H, generator=gen)
    w = torch.randn(C, H, generator=gen) / H ** 0.5
    b = torch.randn(C, generator=gen) * 0.1
    t = torch.rand(R_, C, generator=gen) < 0.4
    return h, t, w, b


@pytest.mark.parametrize("H,C,R_", PPI_SHAPES)
def test_ppi_forward_within_bounds(H, C, R_):
    h, t, w, b = ppi_case(R_, H, C, seed=H + C + R_)
    m = ppi_module(H, C, w, b)
    with torch.no_grad():
        loss = float(run_ppi(m, h, t))
    z, zb = R.logits(h, None, w, b), R.logit_bound(h, None, w, b)
    ref_loss, lb, tp, fp, fn = R.bce(z, zb, t)
    assert R.nan_or_close(loss, ref_loss, lb), (loss, ref_loss, lb)
    if R_ and R.bce_counts_decidable(z, zb):
        precision, recall, fscore = R.ppi_metrics(tp, fp, fn)
        got = m.report_metrics()
        assert got == {"f1_score": float(fscore) * R_ / R_, "pr_score": float(precision) * R_ / R_, "re_score": float(recall) * R_ / R_}


def g2c_grads(m, h, idx, target, scale=1.0):
    hd = h.to(DEV).requires_grad_(True)
    m.zero_grad()
    loss = run_g2c(m, hd, idx, target) * scale
    loss.backward()
    lin = m._Graph2ClassModule__node_to_class
    return hd.grad, lin.weight.grad.clone(), lin.bias.grad.clone()


@pytest.mark.parametrize("H,C,S", [(8, 1, 1), (64, 101, 129), (128, 129, 65), (256, 256, 200), (64, 101, 5000)])
def test_graph2class_backward(H, C, S):
    h, idx, target, w, b = g2c_case(max(S // 2, 1), H, C, S, seed=7 + H + C)      # repeated supernode ids
    m = g2c_module(H, C, w, b)
    d_h, d_w, d_b = g2c_grads(m, h, idx, target)
    z = R.logits(h, idx, w, b)
    ref = R.param_grads(h, idx, w, R.ce_grad(z, target))
    for got, want in zip((d_h, d_w, d_b), ref):
        assert R.rel_err(got, want) <= TAU
    for k in (-17, 9):
        scaled = g2c_grads(m, h, idx, target, scale=2.0 ** k)
        for a, s in zip((d_h, d_w, d_b), scaled):
            assert torch.equal(a * 2.0 ** k, s), "gradients must scale by exactly 2^k"


@pytest.mark.parametrize("H,C,R_", [(8, 1, 1), (64, 101, 129), (256, 121, 3000), (256, 256, 65)])
def test_ppi_backward(H, C, R_):
    h, t, w, b = ppi_case(R_, H, C, seed=11 + C)
    m = ppi_module(H, C, w, b)
    hd = h.to(DEV).requires_grad_(True)
    run_ppi(m, hd, t).backward()
    lin = m._PPIClassification__output_representation_to_logits
    z = R.logits(h, None, w, b)
    d_logits = (torch.sigmoid(z) - t.double()) / R_
    for got, want in zip((hd.grad, lin.weight.grad, lin.bias.grad), R.param_grads(h, None, w, d_logits)):
        assert R.rel_err(got, want) <= TAU


@pytest.mark.parametrize("states_bf16", [False, True])
def test_bf16_against_the_rounded_restatement(states_bf16):
    H, C, S = 128, 101, 300
    h, idx, target, w, b = g2c_case(400, H, C, S, seed=3)
    h = h.to(torch.bfloat16).float()
    m = g2c_module(H, C, w, b)
    hh = h.to(DEV).to(torch.bfloat16) if states_bf16 else h.to(DEV)
    with torch.no_grad(), torch.autocast("cuda", torch.bfloat16):
        m._Graph2ClassModule__gnn.output = gnn_output(hh, idx.to(DEV))
        loss = float(m(graph_mb_data={}, target_classes=target.to(DEV), original_supernode_idxs=None))
        logits, _ = m._logits({})
    assert logits.dtype == torch.bfloat16
    z, zb = R.logits(h, idx, w, b, bf16=True), R.logit_bound(h, idx, w, b, bf16=True)
    assert bool(((logits.double().cpu() - z).abs() <= zb).all())
    ref_loss, lb, *_ = R.ce(z, zb, target)
    assert abs(loss - ref_loss) <= lb
    hp, t, wp, bp = ppi_case(500, 256, 121, seed=5)
    mp = ppi_module(256, 121, wp, bp)
    with torch.no_grad(), torch.autocast("cuda", torch.bfloat16):
        loss = float(run_ppi(mp, hp.to(torch.bfloat16) if states_bf16 else hp, t))
    z, zb = R.logits(hp, None, wp, bp, bf16=True), R.logit_bound(hp, None, wp, bp, bf16=True)
    ref_loss, lb, *_ = R.bce(z, zb, t)
    assert abs(loss - ref_loss) <= lb


@pytest.mark.parametrize("bf16", [False, True])
def test_ppi_predictions_at_the_threshold_are_torchs(bf16):
    """W = 0: the logit is the bias exactly; biases straddle the point where torch's sigmoid (fp32, or rounded to bf16) reaches 0.5."""
    C, R_, H = 256, 64, 64
    step = 2.0 ** -8 if bf16 else 2.0 ** -24
    k = torch.arange(C, dtype=torch.float64) - C // 2
    bias = (-step + k * step / 16).float()
    if bf16:
        bias = bias.to(torch.bfloat16).float()        # the bias the kernel adds is bf16-rounded, as autocast's Linear
    gen = torch.Generator().manual_seed(1)
    t = torch.rand(R_, C, generator=gen) < 0.5
    m = ppi_module(H, C, torch.zeros(C, H), bias)
    h = torch.randn(R_, H, generator=gen)
    with torch.no_grad(), torch.autocast("cuda", torch.bfloat16, enabled=bf16):
        run_ppi(m, h, t)
        logit = bias.to(DEV).expand(R_, C).to(torch.bfloat16 if bf16 else torch.float32)
        pred = (torch.sigmoid(logit) >= 0.5).cpu()
    assert pred.any() and (~pred).any(), "the biases must straddle the threshold"
    tp, fp, fn = int((pred & t).sum()), int((pred & ~t).sum()), int((~pred & t).sum())
    precision, recall, fscore = R.ppi_metrics(tp, fp, fn)
    assert m.report_metrics() == {"f1_score": float(fscore) * R_ / R_, "pr_score": float(precision) * R_ / R_,
                                  "re_score": float(recall) * R_ / R_}


def test_two_runs_are_bit_identical_and_make_no_host_synchronisation():
    h, idx, target, w, b = g2c_case(5000, 128, 101, 20000, seed=9)
    m = g2c_module(128, 101, w, b)
    first = g2c_grads(m, h, idx, target)
    hd, idx, target = h.to(DEV).requires_grad_(True), idx.to(DEV), target.to(DEV)
    hp, t, wp, bp = ppi_case(3000, 256, 121, seed=2)
    mp = ppi_module(256, 121, wp, bp)
    lin_p = mp._PPIClassification__output_representation_to_logits
    hpd, tt = hp.to(DEV).requires_grad_(True), t.to(DEV)
    run_ppi(mp, hpd, tt).backward()
    first_ppi = (hpd.grad.clone(), lin_p.weight.grad.clone(), lin_p.bias.grad.clone())
    mp.zero_grad()
    hpd.grad = None
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m.zero_grad()
        hd.grad = None
        loss = run_g2c(m, hd, idx, target)
        loss.backward()
        run_ppi(mp, hpd, tt).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    lin = m._Graph2ClassModule__node_to_class
    for a, b_ in zip(first + first_ppi, (hd.grad, lin.weight.grad, lin.bias.grad, hpd.grad, lin_p.weight.grad, lin_p.bias.grad)):
        assert torch.equal(a, b_)


def test_backward_leaves_the_plan_cache_unchanged():
    h, idx, target, w, b = g2c_case(300, 64, 101, 500, seed=4)
    m = g2c_module(64, 101, w, b)
    before = list(edgeplan._CACHE)
    g2c_grads(m, h, idx, target)
    assert list(edgeplan._CACHE) == before


@pytest.mark.parametrize("what", ["target", "supernode"])
def test_bad_ids_raise_value_error_once(what):
    h, idx, target, w, b = g2c_case(100, 64, 101, 50, seed=6)
    if what == "target":
        target[3] = 101
    else:
        idx[5] = 100
    m = g2c_module(64, 101, w, b)
    good_idx, good_target = g2c_case(100, 64, 101, 50, seed=6)[1:3]
    raised = 0
    with torch.no_grad():
        try:                                    # raises here when the kernel has already run at the poll after its launch
            run_g2c(m, h, idx, target)
        except ValueError:
            raised += 1
        torch.cuda.synchronize()
        try:                                    # else at the poll before this call launches anything
            run_g2c(m, h, good_idx, good_target)
        except ValueError:
            raised += 1
        assert raised == 1
        loss = run_g2c(m, h, good_idx, good_target)
        torch.cuda.synchronize()
        run_g2c(m, h, good_idx, good_target)      # nothing is left to report
    assert torch.isfinite(loss)


def test_bad_supernode_ids_in_a_training_step_raise_once_without_a_fault():
    """Forward and backward with supernode ids far outside [0, N), negative, and one that an int32 cast would wrap into range: the
    backward gathers and scatters through the forward's safe ids, so nothing reads or writes out of bounds; ValueError is raised once
    and the CUDA context keeps working."""
    h, idx, target, w, b = g2c_case(100, 64, 101, 50, seed=6)
    good_idx = idx.clone()
    idx[5], idx[7], idx[11] = 2 ** 40, -3, 2 ** 32 + 3
    m = g2c_module(64, 101, w, b)
    lin = m._Graph2ClassModule__node_to_class
    # the head's own forward + backward, with no poll in between: the backward runs before any report of the bad ids
    hd = h.to(DEV).requires_grad_(True)
    ops = m._ops(HD.CLASSIFY_CE, lin, hd, idx.to(DEV), target.to(DEV), True)
    AG.classify_with_grad(ops, torch.zeros(1, dtype=torch.int64, device=DEV), None, hd, lin.weight, lin.bias).backward()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(hd.grad).all()) and bool(torch.isfinite(lin.weight.grad).all())
    with pytest.raises(ValueError, match="3 supernode ids"):
        g2c_grads(m, h, good_idx, target)
    raised = 0                                  # through the module: once, after the forward's launch or before the next call's
    try:
        g2c_grads(m, h, idx, target)
    except ValueError:
        raised += 1
    torch.cuda.synchronize()
    try:
        g2c_grads(m, h, good_idx, target)
    except ValueError:
        raised += 1
    assert raised == 1
    d_h, d_w, d_b = g2c_grads(m, h, good_idx, target)
    torch.cuda.synchronize()
    z = R.logits(h, good_idx, w, b)
    for got, want in zip((d_h, d_w, d_b), R.param_grads(h, good_idx, w, R.ce_grad(z, target))):
        assert R.rel_err(got, want) <= TAU


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("C,top,near", [(1, [0], []), (101, [7, 50], []), (200, [150, 170], []), (200, [10, 150], []),
                                        (101, [3], [5]), (200, [20], [160])])
def test_argmax_ties_take_the_first_index_after_rounding(bf16, C, top, near):
    """W = 0: the logits are the biases.  ``top`` share the largest bias; ``near`` lie 2^-10 above it, which bf16 rounds onto it, so in
    bf16 the first of top + near wins and in fp32 the first of near.  Ties within and across the two column blocks of C > 128."""
    H, S = 64, 65
    bias = torch.full((C,), -1.0)
    bias[top] = 1.0
    bias[near] = 1.0 + 2.0 ** -10
    m = g2c_module(H, C, torch.zeros(C, H), bias)
    h = torch.randn(S * 2, H)
    idx = torch.randint(0, S * 2, (S,))
    z = bias.to(torch.bfloat16).float() if bf16 else bias
    want = int(torch.argmax(z.to(DEV)))
    assert want == min(top + near if bf16 else (near or top))
    with torch.no_grad(), torch.autocast("cuda", torch.bfloat16, enabled=bf16):
        m._Graph2ClassModule__gnn.output = gnn_output(h.to(DEV), idx.to(DEV))
        prob, arg, _ = m.predict({})
        m(graph_mb_data={}, target_classes=torch.full((S,), want, dtype=torch.int64, device=DEV), original_supernode_idxs=None)
    assert bool((arg == want).all())
    assert m.report_metrics()["Accuracy"] == 1.0
    ref_prob = float(torch.softmax(z.double(), dim=0).max())
    assert bool(((prob.double() - ref_prob).abs() <= 2.0 ** -20).all())


def test_refusals_leave_the_launch_count_unchanged():
    launches = N.launch_count()
    with torch.no_grad():
        for H, C in ((12, 10), (264, 10), (64, 257)):
            m = P.Graph2ClassModule(StubGnn(H), C).to(DEV)
            with pytest.raises(NotImplementedError):
                run_g2c(m, torch.zeros(4, H), torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.int64))
    m = g2c_module(64, 10, torch.zeros(10, 64), torch.zeros(10))
    with torch.autocast("cuda", torch.bfloat16), pytest.raises(NotImplementedError, match="bf16"):
        run_g2c(m, torch.zeros(4, 64).requires_grad_(True), torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.int64))
    assert N.launch_count() == launches


def test_training_step_matches_a_float64_torch_head():
    """Embedder + gated layer + the native Graph2Class head: the parameter gradients against the same stack with the head written as
    float64 torch ops."""
    from helpers import random_adjacency

    n, F, H, C = 4000, 50, 64, 101
    gen = torch.Generator().manual_seed(31)
    adj = [(s.to(DEV), t.to(DEV)) for s, t in random_adjacency(gen, n, [9000, 3000])]
    torch.manual_seed(31)
    gnn = P.GraphNeuralNetwork([P.GatedMessagePassingLayer(H, H, 2, "sum")], P.LinearFeatureEmbedder(F, H, nn.ReLU()), False, False).to(DEV)
    idx = torch.randint(0, n, (1500,), generator=gen).to(DEV)
    target = torch.randint(0, C, (1500,), generator=gen).to(DEV)
    target[::9] = R.IGNORE_INDEX
    x = torch.randn(n, F, generator=gen).to(DEV)
    graph_data = dict(node_data={"features": x}, adjacency_lists=adj, edge_feature_data=[], node_to_graph_idx=torch.zeros(n, dtype=torch.int64, device=DEV),
                      reference_node_ids={"supernodes": idx}, reference_node_graph_idx={"supernodes": torch.zeros_like(idx)}, num_graphs=1)
    torch.manual_seed(33)
    model = P.Graph2ClassModule(gnn, C).to(DEV).train()
    lin = model._Graph2ClassModule__node_to_class
    with torch.no_grad():
        lin.weight.mul_(0.05)               # uniform_ in [0, 1): a saturated softmax would leave little gradient to compare
    model(graph_data, target, None).backward()
    native = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    rows = gnn(**graph_data).output_node_representations[idx].double()
    nn.functional.cross_entropy(rows @ lin.weight.double().t() + lin.bias.double(), target).backward()
    for k, p in model.named_parameters():
        assert R.rel_err(native[k], p.grad) <= 1e-4, k
