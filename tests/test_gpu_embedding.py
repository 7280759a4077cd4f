"""The native node embedders on the GPU (DESIGN.md §3.12): the embedding-bag kernels against the float32 emulation of their order bit
for bit and against float64 under the derived bound, the modules against the reference's fixtures, gradients, the status word, the
eval-mode cache and CUDA-graph capture.  Reads only tests/golden/ and seeded inputs."""
import glob
import os
import sys

import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import embedding_reference as R  # noqa: E402
from helpers import GOLDEN_DIR, assert_close, load_golden  # noqa: E402

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200._native import NativeLibraryError  # noqa: E402
from ptgnn_b200.embeddings import native_embedding_bag, native_embedding_bag_backward, new_status, poll_status  # noqa: E402

pytestmark = pytest.mark.gpu
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "embed_*.npz")) if not p.endswith("_bf16ac.npz"))
KINDS = ("sum", "mean", "max")


def zipf_ids(shape, V, gen):
    p = 1.0 / torch.arange(1, V + 1, dtype=torch.float64)
    n = 1
    for s in shape:
        n *= s
    return torch.multinomial(p / p.sum(), n, replacement=True, generator=gen).reshape(shape)


def make_case(B, S, D, V, lengths="random", ids="zipf", seed=0):
    gen = torch.Generator().manual_seed(seed)
    table = torch.randn(V, D, generator=gen)
    if ids == "zipf":
        tok = zipf_ids((B, S), V, gen)
    else:                                   # one token takes every slot
        tok = torch.full((B, S), min(3, V - 1), dtype=torch.int64)
    if lengths == "random":
        lens = torch.randint(0, S + 1, (B,), generator=gen)
        lens[0] = S
    elif lengths == "zero":
        lens = torch.zeros(B, dtype=torch.int64)
    elif lengths == "full":
        lens = torch.full((B,), S, dtype=torch.int64)
    else:
        lens = None
    return table, tok, lens, torch.randn(B, D, generator=gen)


# name -> (B, S, D, V, lengths, ids, kinds, check the float64 bound)
SHAPES = {
    "typilus": (204800, 5, 64, 10000, "random", "zipf", ("mean", "max"), False),
    "typilus_tenth": (20480, 5, 64, 10000, "random", "zipf", KINDS, True),
    "graph2seq_token": (60000, 1, 128, 5000, None, "zipf", ("sum",), True),
    "one_row": (1, 5, 64, 50, "random", "zipf", KINDS, True),
    "one_slot_with_lengths": (777, 1, 64, 50, "random", "zipf", KINDS, True),
    "s64": (300, 64, 32, 100, "random", "zipf", KINDS, True),
    "d4": (1000, 5, 4, 30, "random", "zipf", KINDS, True),
    "d63": (1000, 5, 63, 30, "random", "zipf", KINDS, True),
    "d127": (1000, 5, 127, 30, "random", "zipf", KINDS, True),
    "d512": (500, 3, 512, 30, "random", "zipf", KINDS, True),
    "v1": (500, 4, 64, 1, "random", "zipf", KINDS, True),
    "v_above_b": (64, 5, 64, 1000, "random", "zipf", KINDS, True),
    "all_empty": (300, 5, 64, 40, "zero", "zipf", KINDS, True),
    "one_token": (4096, 5, 64, 40, "full", "same", KINDS, True),
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_kernels_match_emulation_bitwise_and_float64_within_bound(name):
    B, S, D, V, lmode, imode, kinds, check_bound = SHAPES[name]
    table, ids, lens, d_out = make_case(B, S, D, V, lmode, imode)
    tc, ic, lc, dc = table.cuda(), ids.cuda(), None if lens is None else lens.cuda(), d_out.cuda()
    status = new_status()
    for kind in kinds:
        exact = R.module_forward(table.double(), ids if S > 1 or lens is not None else ids[:, 0], lens, kind) if check_bound else None
        for dtype in (torch.float32, torch.bfloat16):
            emu, emu_arg = R.emulate_forward(table, ids, lens, kind, out_dtype=dtype)
            prefilled = torch.full((B, D), float("nan"), dtype=dtype, device="cuda")
            out, arg = native_embedding_bag(tc, ic, lc, kind, dtype, want_arg=True, status=status, out=prefilled)
            again = native_embedding_bag(tc, ic, lc, kind, dtype, status=status)
            assert out is prefilled and torch.equal(out, again), f"{name} {kind} {dtype}: two runs differ"
            assert torch.equal(out.cpu(), emu), f"{name} {kind} {dtype}: forward differs from the emulated order"
            if kind == "max":
                assert torch.equal(arg.cpu(), emu_arg)
            if check_bound:
                assert not torch.isnan(out).any()
                b = R.bound(table, ids, lens, kind, out_dtype=dtype)
                finite = torch.isfinite(exact)
                assert torch.equal(out.cpu().double()[~finite], exact[~finite])
                assert bool(((out.cpu().double() - exact)[finite].abs() <= b[finite]).all()), f"{name} {kind} {dtype}: outside the bound"
        # backward
        emu_arg = R.emulate_forward(table, ids, lens, kind)[1]
        arg = emu_arg.cuda() if kind == "max" else None
        got = native_embedding_bag_backward(dc, ic, lc, kind, V, arg)
        again = native_embedding_bag_backward(dc, ic, lc, kind, V, arg)
        assert torch.equal(got, again), f"{name} {kind}: two backward runs differ"
        want = R.emulate_backward(d_out, ids, lens, kind, V, emu_arg)
        assert torch.equal(got.cpu(), want), f"{name} {kind}: backward differs from the emulated order"
        absent = torch.bincount(R.occurrences(ids, lens, V)[2], minlength=V) == 0
        assert bool((got.cpu()[absent] == 0).all())
        if check_bound:
            exact_grad = torch.zeros(V, D, dtype=torch.float64)
            row, slot, tok = R.occurrences(ids, lens, V)
            term = d_out.double()[row]
            if kind == "mean":
                term = term / (R.clamp_lengths(ids, lens)[row].double() + 1e-10)[:, None]
            elif kind == "max":
                term = torch.where(emu_arg[row] == slot[:, None].to(torch.uint8), term, torch.zeros(()).double())
            exact_grad.index_add_(0, tok, term)
            assert bool(((got.cpu().double() - exact_grad).abs() <= R.backward_bound(d_out, ids, lens, kind, V, emu_arg)).all())
    torch.cuda.synchronize()
    poll_status(status, V)


def build_module(g):
    kind, D, V = str(g["kind"]), int(g["dim"]), int(g["vocabulary"])
    if kind == "token":
        m = P.TokenUnitEmbedder(V, D, 0.2)
    else:
        m = P.SubtokenUnitEmbedder(V, D, 0.2, kind, use_dense_output=bool(g["dense"]))
    m.load_state_dict({k[4:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd::")}, strict=True)
    return m.cuda(), kind


def module_args(g):
    ids = torch.from_numpy(g["token_idxs"]).cuda()
    return (ids,) if "lengths" not in g else (ids, torch.from_numpy(g["lengths"]).cuda())


@pytest.mark.parametrize("name", NAMES)
def test_modules_match_the_reference_fixtures(name):
    g = load_golden(name)
    m, kind = build_module(g)
    m.eval()
    with torch.no_grad():
        out = m(*module_args(g))
    assert out.dtype == torch.float32
    assert_close(out, torch.from_numpy(g["out"]), what=name)
    # training: gradients of every parameter (dropout 0 so that the fixture's eval-mode gradients apply)
    for mod in m.modules():
        if isinstance(mod, nn.Dropout):
            mod.p = 0.0
    m.train()
    (m(*module_args(g)) * torch.from_numpy(g["grad_out"]).cuda()).sum().backward()
    for n, p in m.named_parameters():
        assert_close(p.grad, torch.from_numpy(g["grad::" + n]), tol=1e-4, what=f"{name} d {n}")


def test_bf16_autocast_against_the_reference_autocast():
    """DESIGN §4 bf16 rule: rel. L2 <= 1e-2 against the reference's autocast output, and at least as close to the fp32 result."""
    g = load_golden("embed_sub_mean_dense_d64_bf16ac")
    m, _ = build_module(g)
    m.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        out = m(*module_args(g))
        tok = P.TokenUnitEmbedder(20, 64, 0.0).cuda().eval()(torch.arange(10).cuda())
    assert out.dtype == torch.bfloat16 and tok.dtype == torch.float32
    got, ref_ac, ref32 = out.float().cpu(), torch.from_numpy(g["out_autocast"]), torch.from_numpy(g["out_fp32"])
    assert ((got - ref_ac).norm() / ref_ac.norm()).item() <= 1e-2
    assert (got - ref32).abs().mean().item() <= 1.1 * (ref_ac - ref32).abs().mean().item()
    assert_close(got, ref32, tol=2.0 ** -8 * 1.01, what="bf16 output vs the fp32 fixture")
    m.train()
    with torch.autocast("cuda", dtype=torch.bfloat16), pytest.raises(NotImplementedError):
        m(*module_args(g))


@pytest.mark.parametrize("kind,dense,B", [("mean", True, 4000), ("sum", True, 20), ("max", True, 4000), ("mean", False, 500)])
def test_gradients_against_float64_autograd(kind, dense, B):
    """V = 64: B = 4000 takes the table-first dense path, B = 20 the pool-first one; max always pools first."""
    V, D, S = 64, 32, 6
    table, ids, lens, d_out = make_case(B, S, D, V, seed=5)
    ids = ids.clamp(max=V - 9)                      # the last 8 tokens never occur
    lens = lens.clamp(min=1)                        # max of no slot is -inf, and the dense layer makes NaN of it in the reference too
    torch.manual_seed(3)
    m = P.SubtokenUnitEmbedder(V, D, 0.0, kind, use_dense_output=dense).cuda()
    (m(ids.cuda(), lens.cuda()) * d_out.cuda()).sum().backward()
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in m.state_dict().items()}
    t64 = sd["_SubtokenUnitEmbedder__embeddings.weight"]
    w64 = sd.get("_SubtokenUnitEmbedder__out_layer.weight")
    (R.module_forward(t64, ids, lens, kind, w64) * d_out.double()).sum().backward()
    assert_close(m.embedding_layer.weight.grad, t64.grad, tol=1e-5, what="d table")
    assert bool((m.embedding_layer.weight.grad[V - 8:] == 0).all())
    if dense:
        assert_close(dict(m.named_parameters())["_SubtokenUnitEmbedder__out_layer.weight"].grad, w64.grad, tol=1e-4, what="d dense weight")


def test_module_outputs_within_bound_on_both_dense_paths():
    V, D, S = 64, 32, 6
    for B, table_first in ((4000, True), (20, False)):
        table, ids, lens, _ = make_case(B, S, D, V, seed=9)
        m = P.SubtokenUnitEmbedder(V, D, 0.0, "sum").cuda().eval()
        with torch.no_grad():
            m.embedding_layer.weight.copy_(table)
            out = m(ids.cuda(), lens.cuda()).cpu().double()
        w = m.state_dict()["_SubtokenUnitEmbedder__out_layer.weight"].cpu()
        exact = R.module_forward(table.double(), ids, lens, "sum", w.double())
        assert bool(((out - exact).abs() <= R.bound(table, ids, lens, "sum", w, table_first=table_first)).all())


def test_out_of_range_id_is_counted_and_raises_at_the_poll():
    m = P.SubtokenUnitEmbedder(10, 16, 0.0, "sum", use_dense_output=False).cuda().eval()
    ids = torch.tensor([[1, 10, 2], [3, 4, -1], [5, 6, 77]]).cuda()          # 10 and -1 are valid slots, 77 is padding
    lens = torch.tensor([3, 3, 2]).cuda()
    with torch.no_grad():
        try:
            out = m(ids, lens)
        except IndexError:
            out = None                      # the kernel had already finished at the poll inside the call
        torch.cuda.synchronize()
        if out is not None:
            table = m.embedding_layer.weight
            assert torch.equal(out[0], (table[1] + table[0]) + table[2]) and torch.equal(out[2], table[5] + table[6])
            with pytest.raises(IndexError, match="2 token ids outside"):
                m(ids, lens)
        torch.cuda.synchronize()
        good = torch.tensor([[1, 2, 3]]).cuda()
        m._status[0] = 0
        m(good, torch.tensor([3]).cuda())
        torch.cuda.synchronize()
        m(good, torch.tensor([3]).cuda())      # a clean status word raises nothing


@pytest.mark.parametrize("token", [True, False])
@pytest.mark.parametrize("how", ["deepcopy", "save_load_cuda", "save_load_cpu"])
def test_a_used_module_survives_save_restore_and_deepcopy(token, how):
    """abstractneuralmodel.py:155-163 saves with torch.save((self, module)) and restores with torch.load(map_location=device): the
    restored module polls a pinned word of its own, so a bad id is still an IndexError and nothing synchronises."""
    import copy
    import io

    V = 12
    m = (P.TokenUnitEmbedder(V, 16, 0.0) if token else P.SubtokenUnitEmbedder(V, 16, 0.0, "sum")).cuda().eval()
    assert m._status is not None and m._status.is_pinned()              # pinned on the move to the GPU, before any forward
    good = (torch.arange(8).cuda(),) if token else (torch.arange(64).reshape(32, 2).cuda() % V, torch.full((32,), 2).cuda())
    bad = (good[0] + V,) + good[1:]
    with torch.no_grad():
        want = m(*good)
        if how == "deepcopy":
            r = copy.deepcopy(m)
        else:
            buf = io.BytesIO()
            torch.save(m, buf)
            buf.seek(0)
            r = torch.load(buf, map_location="cuda" if how == "save_load_cuda" else "cpu", weights_only=False).cuda()
        assert r._status is None or (r._status is not m._status and r._status.is_pinned())
        assert torch.equal(r(*good), want)
        assert r._status.device.type == "cpu" and r._status.is_pinned() and r._status is not m._status
        try:
            r(*bad)
            torch.cuda.synchronize()
            with pytest.raises(IndexError):
                r(*good)
        except IndexError:
            pass                        # the kernel had already finished at the poll inside the call
        torch.cuda.synchronize()
        r._status[0] = 0
        assert int(m._status[0]) == 0 and torch.equal(m(*good), want)    # the original's word never saw the copy's ids


def test_ids_changed_in_place_before_the_backward_are_refused():
    m = P.SubtokenUnitEmbedder(10, 16, 0.0, "mean", use_dense_output=False).cuda()
    ids, lens = torch.randint(0, 10, (6, 3)).cuda(), torch.tensor([1, 2, 3, 3, 2, 1]).cuda()
    out = m(ids, lens)
    ids.add_(1).remainder_(10)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.sum().backward()


def test_eval_cache_follows_the_parameters():
    V, D, B = 16, 8, 64
    m = P.SubtokenUnitEmbedder(V, D, 0.0, "mean").cuda().eval()
    ids, lens = torch.randint(0, V, (B, 3)).cuda(), torch.randint(1, 4, (B,)).cuda()
    with torch.no_grad():
        a = m(ids, lens)
        cached = m._transformed[1]
        assert torch.equal(m(ids, lens), a) and m._transformed[1] is cached
        m.embedding_layer.weight.mul_(2.0)                     # an optimiser-style in-place update
        b = m(ids, lens)
        assert m._transformed[1] is not cached
        assert_close(b, 2.0 * a, what="after the parameter update")
        m.to(torch.float32)
        assert m._transformed is None
        m.train()
        m(ids, lens)
        assert m._transformed is None                          # trusted in eval mode only


def test_capture_and_replay_on_new_ids():
    V, D, B, S = 200, 64, 512, 5
    m = P.SubtokenUnitEmbedder(V, D, 0.1, "mean").cuda().eval()
    gen = torch.Generator().manual_seed(4)
    ids, lens = torch.randint(0, V, (B, S), generator=gen).cuda(), torch.randint(1, S + 1, (B,), generator=gen).cuda()
    with torch.no_grad():
        stream = torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            m(ids, lens)
        torch.cuda.current_stream().wait_stream(stream)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m(ids, lens)
        ids.copy_(torch.randint(0, V, (B, S), generator=gen))
        lens.copy_(torch.randint(1, S + 1, (B,), generator=gen))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, m(ids, lens))


class _RestatedEmbedder(nn.Module):
    """The reference's SubtokenUnitEmbedder written with library ops (embedding_reference.module_forward) on the same parameters."""

    def __init__(self, native):
        super().__init__()
        self.table = nn.Parameter(native.embedding_layer.weight.detach().clone())
        self.weight = nn.Parameter(native.state_dict()["_SubtokenUnitEmbedder__out_layer.weight"].detach().clone())

    def forward(self, token_idxs, lengths):
        emb = nn.functional.embedding(token_idxs, self.table)
        mask = (torch.arange(emb.shape[1], device=emb.device).unsqueeze(0) < lengths.unsqueeze(-1)).unsqueeze(-1).float()
        return nn.functional.linear((emb * mask).sum(dim=-2) / (lengths.unsqueeze(-1).float() + 1e-10), self.weight)


def test_gnn_with_native_embedder_trains_one_step():
    N_, D, V, S = 3000, 64, 500, 5
    gen = torch.Generator().manual_seed(8)
    adj = [(torch.randint(0, N_, (9000,), generator=gen).cuda(), torch.randint(0, N_, (9000,), generator=gen).cuda()) for _ in range(2)]
    n2g = torch.sort(torch.randint(0, 4, (N_,), generator=gen))[0].cuda()
    ids, lens = zipf_ids((N_, S), V, gen).cuda(), torch.randint(1, S + 1, (N_,), generator=gen).cuda()
    torch.manual_seed(1)
    layer = P.GatedMessagePassingLayer(D, D, 5, "sum")
    native = P.GraphNeuralNetwork([layer], P.SubtokenUnitEmbedder(V, D, 0.0, "mean"), True, True).cuda().train()
    restated_embedder = _RestatedEmbedder(native._GraphNeuralNetwork__node_embedder).cuda()
    results = []
    for embedder in (None, restated_embedder):
        if embedder is not None:
            native._GraphNeuralNetwork__node_embedder = embedder
        native.zero_grad()
        opt = torch.optim.SGD(native.parameters(), lr=0.1)
        out = native(node_data=dict(token_idxs=ids, lengths=lens), adjacency_lists=adj, edge_feature_data=[], node_to_graph_idx=n2g,
                     reference_node_ids={}, reference_node_graph_idx={}, num_graphs=4)
        loss = out.output_node_representations.square().mean()
        loss.backward()
        emb = native._GraphNeuralNetwork__node_embedder
        table = emb.table if embedder is not None else emb.embedding_layer.weight
        before = table.detach().clone()
        grad = table.grad.detach().clone()
        opt.step()
        results.append((out.input_node_representations.detach().cpu(), loss.item(), grad.cpu(), (table.detach() - before).cpu()))
        for p in layer.parameters():                 # the second run starts from the same layer parameters
            if p.grad is not None:
                p.data.add_(p.grad, alpha=0.1)
    (init_n, loss_n, grad_n, step_n), (init_r, loss_r, grad_r, step_r) = results
    w = restated_embedder.weight.detach().cpu()
    b = R.bound(restated_embedder.table.detach().cpu() - step_r, ids.cpu(), lens.cpu(), "mean", w, table_first=True)
    assert bool(((init_n.double() - init_r.double()).abs() <= 2 * b + 4 * R.U * init_r.double().abs()).all())
    assert abs(loss_n - loss_r) <= 1e-5 * max(1.0, abs(loss_r))
    assert_close(grad_n, grad_r, tol=1e-5, what="d table through the GNN")
    # the step as seen through table_after - table_before: off by the rounding of table entries below 1
    assert step_n.abs().max() > 0 and torch.allclose(step_n, -0.1 * grad_n, rtol=1e-5, atol=1e-6)


def test_unsupported_cases_raise():
    ids, lens = torch.zeros(4, 3, dtype=torch.int64).cuda(), torch.ones(4, dtype=torch.int64).cuda()
    with torch.no_grad():
        with pytest.raises(NotImplementedError):
            P.SubtokenUnitEmbedder(5, 516, 0.0, "sum", use_dense_output=False).cuda()(ids, lens)                     # D > 512
        with pytest.raises(NotImplementedError):
            P.SubtokenUnitEmbedder(5, 8, 0.0, "sum").cuda()(torch.zeros(4, 65, dtype=torch.int64).cuda(), lens)       # S > 64
        with pytest.raises(NotImplementedError):
            P.SubtokenUnitEmbedder(5, 63, 0.0, "sum").cuda()(ids, lens)                                              # dense with D % 4 != 0
    with pytest.raises(NativeLibraryError):
        native_embedding_bag(torch.zeros(5, 8), ids.cpu(), lens.cpu(), "sum")
    with pytest.raises(NativeLibraryError):
        native_embedding_bag_backward(torch.zeros(4, 8), ids.cpu(), lens.cpu(), "sum", 5)
    with pytest.raises(ValueError):
        native_embedding_bag(torch.zeros(5, 8).cuda(), ids, lens, "median")
