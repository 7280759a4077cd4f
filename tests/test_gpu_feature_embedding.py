"""GPU tests of the native LinearFeatureEmbedder (csrc/feature_embed.cu, DESIGN.md §3.15): the kernel element by element against float64
under the bound of tests/feature_embedding_reference.py at the row-tile edges, bf16 under autocast, the backward at training's gradient
magnitudes, the packed output, the hand-off to a first fused layer, CUDA-graph capture and the overflow report."""
import os
import sys

import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import feature_embedding_reference as R  # noqa: E402
from helpers import split_f16  # noqa: E402

import ptgnn_b200 as P  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402
from ptgnn_b200 import embeddings as EMB  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
ACTS = {"none": lambda: None, "relu": nn.ReLU, "tanh": nn.Tanh, "gelu": nn.GELU}
ROWS = (0, 1, 63, 64, 65, 127, 128, 129, 133 * 128 + 17)      # the last: not a whole wave of 128-row tiles over the CTAs
GRAD_SCALES = (1.0, 2.0 ** -17, 2.0 ** -27, 2.0 ** -37, 2.0 ** 17)   # the magnitudes of test_gpu_backward_edges.py
TAU = 5e-5


def module(F, D, act, seed=0):
    torch.manual_seed(seed)
    return P.LinearFeatureEmbedder(F, D, ACTS[act]()).to(DEV).eval()


def weight(m):
    return m.state_dict()["_LinearFeatureEmbedder__linear_map.weight"]


def features(n, F, seed, scale=2.0):
    return (torch.randn(n, F, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


def check_elements(got, x, w, act, bf16=False):
    exact = R.forward(x.cpu(), w.cpu(), act, bf16=bf16)
    err = (got.double().cpu() - exact).abs()
    b = R.bound(x.cpu(), w.cpu(), act, bf16=bf16)
    bad = err > b
    assert not bool(bad.any()), f"{int(bad.sum())} of {bad.numel()} elements outside the bound; worst excess {float((err - b).max()):.3e}"


@pytest.mark.parametrize("F,D,act", [(50, 64, "none"), (50, 64, "relu"), (50, 64, "tanh"), (50, 64, "gelu"), (1, 8, "relu"),
                                     (121, 256, "gelu"), (512, 256, "tanh"), (200, 200, "none"), (33, 24, "relu"), (128, 128, "gelu")])
def test_fp32_forward_per_element_at_the_tile_edges(F, D, act):
    m = module(F, D, act)
    w = weight(m)
    for n in ROWS:
        x = features(n, F, seed=n + F)
        with torch.no_grad():
            out = m(x)
        assert out.dtype == torch.float32 and tuple(out.shape) == (n, D)
        check_elements(out, x, w, act)


def test_unaligned_and_strided_features():
    """Rows of 50 floats start 8-byte aligned; a storage offset of one float leaves 4-byte alignment (the 4-byte copies); a strided
    view is made contiguous."""
    m = module(50, 64, "tanh")
    w = weight(m)
    n = 1000
    flat = torch.randn(n * 50 + 1, generator=torch.Generator().manual_seed(3)).to(DEV)
    x = flat[1:].view(n, 50)
    assert x.data_ptr() % 8 == 4
    wide = features(n, 100, seed=4)
    with torch.no_grad():
        check_elements(m(x), x, w, "tanh")
        check_elements(m(wide[:, ::2]), wide[:, ::2].contiguous(), w, "tanh")


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("F,D", [(50, 64), (121, 256), (1, 8)])
def test_bf16_forward_per_element_under_autocast(F, D, act):
    m = module(F, D, act)
    w = weight(m)
    for n in (1, 129, 133 * 128 + 17):
        x = features(n, F, seed=7 + n)
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            out = m(x)
        assert out.dtype == torch.bfloat16
        check_elements(out.float(), x, w, act, bf16=True)


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("F,D", [(50, 64), (121, 256)])
def test_backward_at_training_gradient_magnitudes(F, D, act):
    m = module(F, D, act).train()
    w = weight(m)
    n = 5000
    x0 = features(n, F, seed=21)
    g0 = torch.randn(n, D, generator=torch.Generator().manual_seed(22)).to(DEV)
    for s in GRAD_SCALES:
        for x_grad in (False, True):
            m.zero_grad(set_to_none=True)
            x = x0.clone().requires_grad_(x_grad)
            out = m(x)
            out.backward(g0 * s)
            d_w_ref, d_x_ref = R.gradients(x0.cpu(), w.cpu(), act, (g0 * s).cpu())
            got = [(dict(m.named_parameters())["_LinearFeatureEmbedder__linear_map.weight"].grad, d_w_ref)]
            if x_grad:
                got.append((x.grad, d_x_ref))
            else:
                assert x.grad is None
            for d, ref in got:
                err = (d.double().cpu() - ref).abs().max() / ref.abs().max()
                assert float(err) <= TAU and R.rel_l2(d.cpu(), ref) <= TAU, f"s={s} x_grad={x_grad}: max err / max ref {float(err):.3e}"


def test_bf16_with_gradients_raises():
    m = module(50, 64, "relu").train()
    with torch.autocast("cuda", dtype=torch.bfloat16), pytest.raises(NotImplementedError, match="gradients with a bf16 output"):
        m(features(10, 50, seed=1))


@pytest.mark.parametrize("act", list(ACTS))
def test_packed_output_is_the_split_of_the_fp32_output(act):
    m = module(50, 64, act)
    for n in (1, 129, 133 * 128 + 17):
        x = features(n, 50, seed=n)
        prepared = EMB.feature_embed_prepare(weight(m), False, None)
        out, packed, _ = EMB.native_feature_embed(x, prepared, 64, N.ACT_NONE if act == "none" else {
            "relu": N.ACT_RELU, "tanh": N.ACT_TANH, "gelu": N.ACT_GELU}[act], want_packed=True)
        assert packed.numel() == N.lib().ptgnn_b200_packed_state_bytes(n, 64)
        hi, lo = split_f16(out)
        rows = packed[:n * 64 * 4].view(torch.float16).view(n, 128)
        assert torch.equal(rows[:, :64].view(torch.int16), hi.view(torch.int16))
        assert torch.equal(rows[:, 64:].view(torch.int16), lo.view(torch.int16))


def test_first_fused_layer_takes_the_packed_output_bit_identically():
    """Embedder, then a fused gated layer in a container: the same output with and without the hand-off, one launch (the packing
    pass) fewer with it."""
    from helpers import random_adjacency, unchained

    n, F, H = 6000, 50, 64
    gen = torch.Generator().manual_seed(9)
    torch.manual_seed(9)
    adj = [(s.to(DEV), t.to(DEV)) for s, t in random_adjacency(gen, n, [9000, 4000, 700])]
    layer = P.GatedMessagePassingLayer(H, 128, 3, "sum")      # message dimension 128: the fused aggregation kernel
    assert N.lib().ptgnn_b200_fused_supported(0, H, 128)
    gnn = P.GraphNeuralNetwork([layer], P.LinearFeatureEmbedder(F, H, nn.ReLU()), False, False).to(DEV).eval()
    x = features(n, F, seed=10)
    kw = dict(node_data={"features": x}, adjacency_lists=adj, edge_feature_data=[], node_to_graph_idx=torch.zeros(n, dtype=torch.int64,
              device=DEV), reference_node_ids={}, reference_node_graph_idx={}, num_graphs=1)
    with torch.no_grad():
        gnn(**kw)                                   # plan and weight caches
        l0 = N.launch_count()
        chained = gnn(**kw).output_node_representations
        l1 = N.launch_count()
        with unchained():
            plain = gnn(**kw).output_node_representations
        l2 = N.launch_count()
    assert torch.equal(chained, plain)
    assert (l2 - l1) - (l1 - l0) == 1, f"chained {l1 - l0} launches, unchained {l2 - l1}"


def test_cuda_graph_replay_is_bit_identical_to_eager():
    m = module(50, 64, "gelu")
    n = 3000
    x_static = features(n, 50, seed=30)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        for _ in range(2):
            m(x_static)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph):
        out_static = m(x_static)
    for seed in (31, 32):
        x_new = features(n, 50, seed=seed)
        x_static.copy_(x_new)
        graph.replay()
        with torch.no_grad():
            eager = m(x_new)
        torch.cuda.synchronize()
        assert torch.equal(out_static, eager)


@pytest.mark.parametrize("where", ["feature", "weight"])
def test_overflow_is_reported_at_the_next_poll(where):
    """The call polls the status word before its launch and after it without synchronising: the report comes from the call itself
    (when the kernel has already run) or from the next one; once reported, the word is clear again."""
    m = module(50, 64, "relu")
    x = features(500, 50, seed=40)
    if where == "feature":
        x[17, 3] = 7e4
    else:
        with torch.no_grad():
            m._LinearFeatureEmbedder__linear_map.weight[5, 7] = -1e5
    with torch.no_grad(), pytest.raises(FloatingPointError, match="fp16 range"):
        m(x)
        torch.cuda.synchronize()
        m(x[:10])
    if where == "feature":
        with torch.no_grad():
            m(x[:10])
            torch.cuda.synchronize()
            m(x[:10])
