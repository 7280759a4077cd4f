"""GPU tests of the native VarMisuse head (csrc/heads.cu, DESIGN.md §3.16): scores, logsumexps, loss and argmax element by element against
the float64 restatement (tests/heads_reference.py) on the reference's fixtures and at the kernel's structural edges, the backward at
training's gradient magnitudes, bf16 states, determinism, the absence of host synchronisation, the refusals and one training step of a
native GNN with the head."""
import os
import sys

import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import heads_reference as R  # noqa: E402
from helpers import load_golden  # noqa: E402

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200 import heads as HD  # noqa: E402
from ptgnn_b200.gnn import GnnOutput  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
GRAD_SCALES = (1.0, 2.0 ** -17, 2.0 ** -27, 2.0 ** -37, 2.0 ** 17)   # the magnitudes of test_gpu_backward_edges.py
TAU = 5e-5
KEY = "_VarMisuseGraphModel__candidate_scores.weight"


class StubGnn(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.output_node_state_dim = dim
        self.output = None

    def forward(self, **kwargs):
        return self.output


def case(num_nodes, H, sizes, seed, crossed=False, scale=1.0):
    """h [N, H], candidates of slot j = sizes[j] (slot ids shuffled), one correct candidate per slot (taken from another slot when
    ``crossed``), w [1, 2H]."""
    gen = torch.Generator().manual_seed(seed)
    h = torch.randn(num_nodes, H, generator=gen) * scale
    J = len(sizes)
    slot_nodes = torch.randint(0, num_nodes, (J,), generator=gen)
    slot_of = torch.cat([torch.full((n,), j, dtype=torch.int64) for j, n in enumerate(sizes)] or [torch.zeros(0, dtype=torch.int64)])
    slot_of = slot_of[torch.randperm(slot_of.shape[0], generator=gen)]
    cand = torch.randint(0, num_nodes, (slot_of.shape[0],), generator=gen)
    owners = [j for j in range(J) if sizes[j] > 0]
    correct = []
    for j in range(J):
        src = j if sizes[j] > 0 and not crossed else owners[(j + 1) % len(owners)]
        ks = (slot_of == src).nonzero().flatten()
        correct.append(int(ks[int(torch.randint(0, ks.shape[0], (1,), generator=gen))]))
    w = torch.randn(1, 2 * H, generator=gen) / H ** 0.5
    return h, cand, slot_of, slot_nodes, torch.tensor(correct, dtype=torch.int64), w


def dev(*ts):
    return [t.to(DEV) for t in ts]


def run_native(h, cand, slot_of, slot_nodes, correct, w):
    ops = HD.varmisuse_inputs(*dev(h, cand, slot_of, slot_nodes, correct, w))
    hits = torch.zeros(1, dtype=torch.int64, device=DEV)
    loss, score, lse, arg = HD.native_varmisuse(*ops, hits=hits)
    ops[6].poll()
    return ops, loss, score, lse, arg, hits


def check_forward(h, cand, slot_of, slot_nodes, correct, w, bf16=False):
    hh = h.to(torch.bfloat16) if bf16 else h
    _, loss, score, lse, arg, hits = run_native(hh, cand, slot_of, slot_nodes, correct, w)
    hr = hh.float()
    ref = R.varmisuse(hr, cand, slot_of, slot_nodes, correct, w, bf16=bf16)
    sb = R.score_bound(hr, cand, slot_of, slot_nodes, w, bf16)
    assert bool(((score.double().cpu() - ref["score"]).abs() <= sb).all()), "scores outside the bound"
    nonempty = torch.bincount(slot_of, minlength=slot_nodes.shape[0]) > 0
    lb = R.lse_bound(hr, cand, slot_of, slot_nodes, w, bf16)
    got_lse = lse.double().cpu()
    assert bool(((got_lse - ref["lse"]).abs() <= lb)[nonempty].all()), "logsumexps outside the bound"
    assert bool(torch.isneginf(got_lse[~nonempty]).all())
    # the argmax is exact unless two scores lie within the bound of each other
    same = arg.cpu() == ref["argmax"]
    for j in (~same).nonzero().flatten().tolist():
        a, b = int(arg[j]), int(ref["argmax"][j])
        assert abs(float(ref["score"][a] - ref["score"][b])) <= float(sb[a] + sb[b]), f"slot {j}: argmax {a} != {b}"
    if bool(same.all()):
        assert int(hits) == ref["hits"]
    if correct.shape[0]:
        assert abs(float(loss) - float(ref["loss"])) <= R.loss_bound(hr, cand, slot_of, slot_nodes, correct, w, bf16)
    else:
        assert bool(torch.isnan(loss))
    return ref


def check_backward(h, cand, slot_of, slot_nodes, correct, w, g=1.0):
    ops = HD.varmisuse_inputs(*dev(h, cand, slot_of, slot_nodes, correct, w))
    hl = h.to(DEV).requires_grad_(True)
    wl = w.to(DEV).requires_grad_(True)
    hits = torch.zeros(1, dtype=torch.int64, device=DEV)
    from ptgnn_b200 import autograd as AG

    ops = (hl.detach(),) + tuple(ops[1:])
    loss = AG.varmisuse_with_grad(ops, hits, hl, wl)
    loss.backward(torch.tensor(g, device=DEV))
    ref_h, ref_w = R.varmisuse_gradients(h, cand, slot_of, slot_nodes, correct, w, g)
    for got, ref, what in ((hl.grad, ref_h, "d h"), (wl.grad, ref_w, "d w")):
        assert got.shape == ref.shape, what
        err = float((got.double().cpu() - ref).abs().max()) / max(float(ref.abs().max()), 1e-300)
        assert err <= TAU, f"{what}: max err / max ref {err:.3e} (g={g})"
    return hl.grad, wl.grad


@pytest.mark.parametrize("name", ["heads_varmisuse", "heads_varmisuse_crossed"])
def test_fixtures(name):
    t = {k: torch.from_numpy(v) for k, v in load_golden(name).items()}
    args = (t["h"], t["cand"], t["slot_of"], t["slot_nodes"], t["correct"], t["w"])
    ref = check_forward(*args)
    assert ref["hits"] / args[3].shape[0] == float(t["accuracy"])
    d_h, d_w = check_backward(*args)
    for got, key in ((d_h, "grad_h"), (d_w, "grad_w")):
        want = t[key].double()
        assert float((got.double().cpu() - want).abs().max()) <= 1e-5 * max(1.0, float(want.abs().max())), key


EDGES = [
    (50, 4, [1, 2, 3]),                    # the smallest state size
    (50, 1024, [1, 31, 32, 33]),           # the largest
    (80, 1020, [5, 7]),                    # not a multiple of 128: the last lane group is partial
    (40, 64, [0, 4, 0, 9]),                # slots without candidates
    (500, 64, [300, 1, 2]),
    (80000, 64, [10] * 300),               # VarMisuse-sized minibatch
    (20000, 128, [1 + (j * 37) % 64 for j in range(2000)]),   # many slots: several column-sum blocks
]


@pytest.mark.parametrize("num_nodes,H,sizes", EDGES)
def test_forward_and_backward_at_the_edges(num_nodes, H, sizes):
    args = case(num_nodes, H, sizes, seed=num_nodes + H, crossed=0 in sizes)
    check_forward(*args)
    check_backward(*args)


def test_crossed_correct_candidates():
    check_backward(*case(300, 64, [3, 5, 8, 13], seed=3, crossed=True))


def test_no_slots_and_no_candidates():
    h = torch.randn(10, 16)
    e = torch.zeros(0, dtype=torch.int64)
    _, loss, score, lse, arg, hits = run_native(h, e, e, e, e, torch.randn(1, 32))
    assert bool(torch.isnan(loss)) and score.numel() == 0 and lse.numel() == 0 and int(hits) == 0


def test_gradient_scales_are_exact_powers_of_two():
    args = case(3000, 64, [1 + j % 40 for j in range(200)], seed=11)
    d_h1, d_w1 = check_backward(*args, g=1.0)
    for s in GRAD_SCALES[1:]:
        d_h, d_w = check_backward(*args, g=s)
        assert torch.equal(d_h, d_h1 * s) and torch.equal(d_w, d_w1 * s), s


@pytest.mark.parametrize("H,sizes", [(64, [1, 2, 31, 32, 33, 300]), (1024, [3, 40]), (4, [5, 1])])
def test_bf16_forward_against_the_bf16_restatement(H, sizes):
    check_forward(*case(2000, H, sizes, seed=H), bf16=True)


def test_two_runs_are_bit_identical():
    args = case(20000, 64, [1 + (j * 13) % 50 for j in range(500)], seed=5)
    first = check_backward(*args)
    second = check_backward(*args)
    assert all(torch.equal(a, b) for a, b in zip(first, second))
    _, l1, s1, *_ = run_native(*args)
    _, l2, s2, *_ = run_native(*args)
    assert torch.equal(l1, l2) and torch.equal(s1, s2)


def module_with(h, cand, slot_of, slot_nodes, seed=0):
    torch.manual_seed(seed)
    gnn = StubGnn(h.shape[1])
    m = P.VarMisuseGraphModel(gnn).to(DEV)
    gnn.output = GnnOutput(h, h, torch.zeros(h.shape[0], dtype=torch.int64, device=DEV),
                           {"candidate_nodes": cand, "slot_node_idx": slot_nodes}, {"candidate_nodes": slot_of}, 1)
    return m


def test_module_step_makes_no_host_synchronisation_and_counts_accuracy_on_the_device():
    h, cand, slot_of, slot_nodes, correct, _ = dev(*case(5000, 64, [2 + j % 9 for j in range(300)], seed=21))
    hl = h.clone().requires_grad_(True)
    m = module_with(hl, cand, slot_of, slot_nodes).train()
    m({}, correct).backward()                                    # warm-up: library load, plans
    m.reset_metrics()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            m({}, correct).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    w = m.state_dict()[KEY]
    ref = R.varmisuse(h.cpu(), cand.cpu(), slot_of.cpu(), slot_nodes.cpu(), correct.cpu(), w.cpu())
    assert m.report_metrics()["Accuracy"] == ref["hits"] / 300


def test_bad_indices_raise_value_error():
    h, cand, slot_of, slot_nodes, correct, w = dev(*case(100, 16, [3, 4], seed=1))
    for what in ("correct", "candidate", "slot node"):
        c, k, sn = correct.clone(), cand.clone(), slot_nodes.clone()
        if what == "correct":
            c[1] = cand.shape[0]
        elif what == "candidate":
            k[2] = 100
        else:
            sn[0] = 100
        m = module_with(h, k, slot_of, sn)
        with torch.no_grad(), pytest.raises(ValueError, match="out of range"):
            m({}, c)
            torch.cuda.synchronize()
            m({}, c)
    m = module_with(h, cand, slot_of, slot_nodes)     # reported once: the same slot plan is clean again
    with torch.no_grad():
        m({}, correct)
        torch.cuda.synchronize()
        m({}, correct)


def test_refusals_leave_the_launch_count_unchanged():
    h, cand, slot_of, slot_nodes, correct, _ = dev(*case(100, 16, [3, 4], seed=1))
    launches = N.launch_count()
    with pytest.raises(NotImplementedError, match="multiple of 4"):
        module_with(torch.zeros(100, 18, device=DEV), cand, slot_of, slot_nodes)({}, correct)
    with pytest.raises(NotImplementedError, match="bf16"):
        hb = h.to(torch.bfloat16).requires_grad_(True)
        module_with(hb, cand, slot_of, slot_nodes).train()({}, correct)
    assert N.launch_count() == launches


def test_gnn_with_the_head_trains_one_step_like_the_float64_head():
    """Embedder + gated layer + the native head: the GNN's parameter gradients against the same stack with the head written as float64
    torch ops (log_softmax per slot)."""
    from helpers import random_adjacency

    n, F, H = 4000, 50, 64
    gen = torch.Generator().manual_seed(31)
    adj = [(s.to(DEV), t.to(DEV)) for s, t in random_adjacency(gen, n, [9000, 3000])]
    torch.manual_seed(31)
    gnn = P.GraphNeuralNetwork([P.GatedMessagePassingLayer(H, H, 2, "sum")], P.LinearFeatureEmbedder(F, H, nn.ReLU()), False, False).to(DEV)
    _, cand, slot_of, slot_nodes, correct, _ = dev(*case(n, H, [3 + j % 11 for j in range(120)], seed=32))
    x = (torch.randn(n, F, generator=gen)).to(DEV)
    graph_data = dict(node_data={"features": x}, adjacency_lists=adj, edge_feature_data=[], node_to_graph_idx=torch.zeros(n, dtype=torch.int64, device=DEV),
                      reference_node_ids={"candidate_nodes": cand, "slot_node_idx": slot_nodes},
                      reference_node_graph_idx={"candidate_nodes": slot_of}, num_graphs=1)
    torch.manual_seed(33)
    model = P.VarMisuseGraphModel(gnn).to(DEV).train()
    model(graph_data, correct).backward()
    native = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    out = gnn(**graph_data).output_node_representations
    w = dict(model.named_parameters())[KEY]
    hd, wd = out.double(), w.double().reshape(-1)
    score = hd[cand] @ wd[:H] + hd[slot_nodes][slot_of] @ wd[H:]
    mx = torch.full((slot_nodes.shape[0],), -torch.inf, dtype=torch.float64, device=DEV).scatter_reduce(0, slot_of, score.detach(), "amax")
    lse = torch.zeros_like(mx).scatter_add(0, slot_of, (score - mx[slot_of]).exp()).log() + mx
    (-(score[correct] - lse[slot_of[correct]]).mean()).backward()
    for k, p in model.named_parameters():
        ref = p.grad.double()
        err = float((native[k].double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)
        assert err <= 1e-4, f"{k}: max err / max ref {err:.3e}"


def test_backward_leaves_the_shared_plan_cache_alone():
    from ptgnn_b200 import edgeplan

    from ptgnn_b200 import autograd as AG

    h, cand, slot_of, slot_nodes, correct, w = dev(*case(3000, 64, [4] * 50, seed=41))
    hl, wl = h.requires_grad_(True), w.requires_grad_(True)
    hits = torch.zeros(1, dtype=torch.int64, device=DEV)
    AG.varmisuse_with_grad(HD.varmisuse_inputs(hl, cand, slot_of, slot_nodes, correct, wl), hits, hl, wl).backward()
    before = list(edgeplan._CACHE)          # the slot plan is in it since the first forward
    for _ in range(2):
        AG.varmisuse_with_grad(HD.varmisuse_inputs(hl, cand, slot_of, slot_nodes, correct, wl), hits, hl, wl).backward()
    assert list(edgeplan._CACHE) == before


def test_backward_with_more_slot_blocks_than_a_grid_dimension_of_65535():
    """J = 4.3M slots of one candidate: ceil(J / 64) = 67,188 blocks of the d w column sum."""
    J, H = 4_300_000, 4
    gen = torch.Generator().manual_seed(43)
    num_nodes = J + 10
    h = torch.randn(num_nodes, H, generator=gen)
    slot_of = torch.arange(J)
    cand = torch.randint(0, num_nodes, (J,), generator=gen)
    slot_nodes = torch.randint(0, num_nodes, (J,), generator=gen)
    w = torch.randn(1, 2 * H, generator=gen)
    check_backward(h, cand, slot_of, slot_nodes, slot_of.clone(), w)
