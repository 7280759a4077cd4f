"""CPU checks of the unfused-kernel test infrastructure (tests/unfused_reference.py): the structured graph contains every case
it is built for, a bit-level emulation of the 3xTF32 arithmetic stays inside the per-element bound while 1xTF32 (hi*hi only)
and a result with 16 columns left unwritten break it, and the reduce / GRU / dense / LayerNorm references accept an fp32
evaluation of the same operation and reject a plausible kernel mistake."""
import numpy as np
import pytest
import torch

import fused_reference as FR
import unfused_reference as R
from oracle import ptgnn_oracle as O


def _tf32_hi(x: np.ndarray) -> np.ndarray:
    return ((x.view(np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _tf32_trunc(x: np.ndarray) -> np.ndarray:
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _emulate_tf32(X: np.ndarray, W: np.ndarray, passes: int = 3) -> np.ndarray:
    """fp32 X [E, K] times W [D, K]^T as the tensor-core pipeline computes it: TF32 (hi, lo) split, hi*hi into the main and
    hi*lo + lo*hi into the correction accumulator, each 8-wide k-step rounded once to fp32, the two accumulators added last.
    passes = 1: hi*hi alone."""
    xh, wh = _tf32_hi(X), _tf32_hi(W)
    xl, wl = _tf32_trunc(X - xh), _tf32_trunc(W - wh)
    f = lambda a: a.astype(np.float64)
    main = np.zeros((X.shape[0], W.shape[0]), np.float32)
    corr = np.zeros_like(main)
    for k in range(0, X.shape[1], 8):
        s = slice(k, k + 8)
        main = (f(main) + f(xh[:, s]) @ f(wh[:, s]).T).astype(np.float32)
        if passes == 3:
            corr = (f(corr) + f(xh[:, s]) @ f(wl[:, s]).T + f(xl[:, s]) @ f(wh[:, s]).T).astype(np.float32)
    return main + corr


@pytest.mark.parametrize("N", [12800, 12801, 12799, 12816])
def test_structured_graph_covers_the_tile_edges(N):
    adj, runs = R.structured_graph(N)
    f = R.structure_facts(adj, N)
    assert set(R.TYPE_COUNTS) <= set(f["type_counts"])
    assert f["tiles"] >= 3 * R.SM_COUNT + 1                           # >= 3 waves of the persistent grid
    assert f["max_in_degree"] >= 2000
    want = {(L, w) for L in R.EMPTY_RUNS for w in ("start", "middle", "end")}
    assert want <= f["empty_runs"], want - f["empty_runs"]
    assert len(runs) == len(want) and f["trailing_empty"] == 3
    assert f["duplicates"] > 0 and f["same_type_duplicates"] > 0
    assert (f["mod16"], f["mod128"]) == (N % 16, N % 128)
    counts = f["type_counts"]                                         # the small counts sit between large types
    assert counts[0] >= 10_000 and counts[6] >= 10_000 and counts[-1] >= 5_000


def _small_problem(H, D, use_target, seed=5):
    N = 2049
    adj, _ = R.structured_graph(N, big=3000, seed=seed)
    gen = torch.Generator().manual_seed(seed)
    h = torch.randn(N, H, generator=gen)
    Kw = 2 * H if use_target else H
    w = [torch.randn(D, Kw, generator=gen) / Kw ** 0.5 for _ in adj]
    return N, adj, h, w


def _emulated_messages(h, adj, w, use_target, passes):
    out = []
    for (s, t), wt in zip(adj, w):
        X = torch.cat([h[s], h[t]], 1) if use_target else h[s]
        out.append(torch.from_numpy(_emulate_tf32(X.numpy(), wt.numpy(), passes)).double())
    return torch.cat(out)


@pytest.mark.parametrize("H,D,use_target", [(36, 112, True), (100, 48, False), (32, 144, True)])
def test_tf32_bound_is_sound_and_sharp(H, D, use_target):
    N, adj, h, w = _small_problem(H, D, use_target)
    tgt, m, err = R.fp32_messages(h, adj, w, use_target, mode="tc")
    got3 = _emulated_messages(h, adj, w, use_target, 3)
    ratio = FR.check_bound(got3, m, err, "3xTF32 emulation")
    assert ratio < 0.5, ratio
    with pytest.raises(AssertionError):
        FR.check_bound(_emulated_messages(h, adj, w, use_target, 1), m, err, "1xTF32")
    hole = got3.clone()
    hole[:, D - 16:] = 0                                               # the last 16 columns never written
    with pytest.raises(AssertionError):
        FR.check_bound(hole, m, err, "16 columns at 0")
    # through the reduce: the bit-exact sum of the emulated messages stays inside the aggregate bound, hi*hi alone does not
    ref, bound, _ = FR.aggregate(tgt, m, err, N, "sum", False)
    agg3, _ = R.reduce_exact(tgt, got3.float(), N, "sum")
    FR.check_bound(agg3, ref, bound, "3xTF32 aggregate")
    agg1, _ = R.reduce_exact(tgt, _emulated_messages(h, adj, w, use_target, 1).float(), N, "sum")
    with pytest.raises(AssertionError):
        FR.check_bound(agg1, ref, bound, "1xTF32 aggregate")


@pytest.mark.parametrize("reduce", ["sum", "mean", "max", "min"])
def test_reduce_reference_matches_the_scatter_oracle(reduce):
    gen = torch.Generator().manual_seed(9)
    n, E, D = 300, 4000, 12
    src = torch.randn(E, D, generator=gen)
    idx = torch.randint(0, n - 5, (E,), generator=gen)
    src[7], idx[7] = src[3], idx[3]                                   # an exact tie: the first occurrence wins
    out, arg = R.reduce_exact(idx, src, n, reduce)
    ref, ref_arg = O.scatter_with_arg(src, idx, n, reduce)
    if reduce in ("max", "min"):
        assert torch.equal(out, ref) and torch.equal(arg, ref_arg)
        assert bool((arg[n - 5:] == E).all()) and bool((out[n - 5:] == 0).all())
        assert int(arg[idx[3], 0]) != 7
    else:
        assert torch.allclose(out.double(), ref.double(), rtol=1e-5, atol=1e-5)
        assert bool((out[n - 5:] == 0).all())


def test_bf16_unwritten_columns_break_the_bound():
    gen = torch.Generator().manual_seed(4)
    N, H, D = 2049, 64, 112
    adj, _ = R.structured_graph(N, big=2500, seed=4)
    h = torch.randn(N, H, generator=gen).to(torch.bfloat16)
    w = [torch.randn(D, H, generator=gen) / 8 for _ in adj]
    ref, bound, _ = FR.aggregate(*FR.messages(h, adj, w, False, True), N, "sum", True)
    FR.check_bound(ref, ref, bound, "exact")
    hole = ref.clone()
    hole[:, 96:112] = 0
    with pytest.raises(AssertionError):
        FR.check_bound(hole, ref, bound, "columns 96-111 at 0")


def _gru_params(H, D, seed):
    torch.manual_seed(seed)
    cell = torch.nn.GRUCell(D, H)
    return cell, [p.detach() for p in (cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh)]


@pytest.mark.parametrize("H,D", [(32, 36), (96, 200)])
def test_gru_bound_accepts_fp32_and_rejects_swapped_gates(H, D):
    cell, p = _gru_params(H, D, H + D)
    gen = torch.Generator().manual_seed(1)
    x, h = 2 * torch.randn(500, D, generator=gen), torch.randn(500, H, generator=gen)
    ref, bound = R.gru(x, None, h, *p, mode="ffma")                   # gamma_K: any fp32 summation order
    with torch.no_grad():
        FR.check_bound(cell(x, h), ref, bound, "fp32 GRUCell")
        w_ih = p[0].clone()
        w_ih[:H], w_ih[H:2 * H] = p[0][H:2 * H], p[0][:H]             # r and z weights swapped
        bad = torch.nn.functional.linear(x, w_ih, p[2])
    gh = torch.nn.functional.linear(h, p[1], p[3])
    r = torch.sigmoid(bad[:, :H] + gh[:, :H])
    z = torch.sigmoid(bad[:, H:2 * H] + gh[:, H:2 * H])
    n = torch.tanh(bad[:, 2 * H:] + r * gh[:, 2 * H:])
    with pytest.raises(AssertionError):
        FR.check_bound((1 - z) * n + z * h, ref, bound, "r/z swapped")
    ref_b, bound_b = R.gru(x.bfloat16().double(), None, h.bfloat16().double(), *p, mode="bf16")
    FR.check_bound(ref_b, ref_b, bound_b, "bf16 exact")


@pytest.mark.parametrize("act", [None, "gelu", "tanh", "relu"])
def test_dense_and_layer_norm_bounds(act):
    gen = torch.Generator().manual_seed(2)
    y = torch.randn(400, 100, generator=gen)
    W, b = torch.randn(112, 100, generator=gen) / 10, torch.randn(112, generator=gen)
    ref, bound = R.dense(y.double(), None, W, b, act, "ffma")
    fn = {None: lambda t: t, "gelu": torch.nn.functional.gelu, "tanh": torch.tanh, "relu": torch.relu}[act]
    got = fn(torch.nn.functional.linear(y, W, b))
    FR.check_bound(got, ref, bound, "fp32 dense")
    hole = got.clone()
    hole[:, 96:] = 0
    with pytest.raises(AssertionError):
        FR.check_bound(hole, ref, bound, "16 columns at 0")
    lw, lb = torch.rand(100, generator=gen) + 0.5, torch.randn(100, generator=gen)
    x = fn(y.double())
    lref, lbound = R.layer_norm(x, 8 * R.U * (x.abs() + 1), lw, lb, 1e-5)
    FR.check_bound(torch.nn.functional.layer_norm(fn(y), (100,), lw, lb, 1e-5), lref, lbound, "fp32 LayerNorm")
    with pytest.raises(AssertionError):                               # LayerNorm without its bias
        FR.check_bound(torch.nn.functional.layer_norm(fn(y), (100,), lw, None, 1e-5), lref, lbound, "no bias")
