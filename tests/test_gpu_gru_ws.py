"""The weights-stationary GRU kernel (csrc/gru_ws.cu) at its structural edges, through the fused gated layer.

The kernel walks 64-row tiles: the CTAs of one 32-hidden-unit block take every (132 / (H / 32))-th tile and alternate them
between their two consumer warpgroups.  The row counts below give a single partial tile (1, 63), exact tiles (64), one row
past a tile (65, 129), fewer tiles than CTAs per hidden-unit block (1,000 rows), a tile count that the CTAs do not divide
evenly with an odd count per CTA, and enough tiles that the operand ring wraps many times.  fp32 (3xFP16) is compared with
float64 (the fused reference aggregate, then ``gru_cell``) at the bar of ``test_fused_gated_structured``; bf16 at the bars of
``test_gpu_bf16.py``.  Every case runs twice and must be bit-identical.  Through a layer the message dimension is 128 (what the
fused aggregation kernel takes), so D = 128 and H in {64, 128}, and 256 in bf16 (8 hidden-unit blocks, 16 CTAs each)."""
import pytest
import torch

import fused_reference as R
from helpers import assert_close, gated_oracle_args, random_adjacency, unchained
from oracle import ptgnn_oracle as O

pytestmark = pytest.mark.gpu

T = 3
D = 128
N_ROWS = (1, 63, 64, 65, 127, 129, 1000, 64 * (33 * 3 + 5) + 17, 40_000)


def _layer(H, seed):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    layer = P.GatedMessagePassingLayer(H, D, T, "sum").cuda().eval()
    return layer, gated_oracle_args({k: v.clone().cpu() for k, v in layer.state_dict().items()})


def _graph(N, seed):
    gen = torch.Generator().manual_seed(seed)
    adj = random_adjacency(gen, N, [max(1, 2 * N), max(1, N), max(1, N // 2)])
    return adj, [(s.cuda(), t.cuda()) for s, t in adj], gen


def _twice(layer, h, adj_d):
    with torch.no_grad():
        a = layer(h.cuda(), adj_d)
        b = layer(h.cuda(), adj_d)
    assert torch.equal(a, b), "gated layer output is not run-to-run bit-identical"
    return a.float().cpu()


@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("N", N_ROWS)
def test_gru_ws_fp32_against_float64(N, H):
    adj, adj_d, gen = _graph(N, 100 + N + H)
    h = torch.randn(N, H, generator=gen) * 0.5
    layer, args = _layer(H, N + H)
    got = _twice(layer, h, adj_d)
    tgt, m, err = R.messages(h, adj, args["edge_weights"], False, False)
    _, _, agg64 = R.aggregate(tgt, m, err, N, "sum", False)
    assert float(agg64.abs().max()) < 65504
    ref = O.gru_cell(agg64, h.double(), *(args[k].double() for k in ("gru_w_ih", "gru_w_hh", "gru_b_ih", "gru_b_hh")))
    assert_close(got, ref, what=f"fp32 gated N={N} H={H}")


@pytest.mark.parametrize("H", [64, 128, 256])
@pytest.mark.parametrize("N", N_ROWS)
def test_gru_ws_bf16(N, H):
    adj, adj_d, gen = _graph(N, 200 + N + H)
    h = (torch.randn(N, H, generator=gen) * 0.5).to(torch.bfloat16)
    layer, args = _layer(H, N + H + 1)
    got = _twice(layer, h, adj_d)
    ref = O.gated_layer_forward(h.float(), adj, [torch.empty(a[0].shape[0], 0) for a in adj], aggregation_fn="sum", **args)
    rel = ((got - ref).norm() / ref.norm()).item()
    frac = ((got - ref).abs() <= 1e-2 * ref.abs().clamp(min=1)).float().mean().item()
    assert rel <= 1e-2 and frac >= 0.999, f"bf16 gated N={N} H={H}: rel L2 {rel:.2e}, within 1e-2: {frac:.4f}"


@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("N", [63, 65, 129, 64 * (33 * 3 + 5) + 17])
def test_gru_ws_packed_output_chains_bit_identical(N, H):
    """In a container, each layer's GRU also writes its output as the packed fp16 (hi | lo') rows the next layer takes.  The
    chained run must equal the run that packs every layer's input itself, which holds only if the packed output equals
    pack_states(out) bit for bit, the rows of the partial last tile included."""
    import ptgnn_b200 as P

    class _Embed(torch.nn.Module):
        def forward(self, x):
            return x

    adj, adj_d, gen = _graph(N, 300 + N + H)
    h = torch.randn(N, H, generator=gen).cuda()
    torch.manual_seed(N + H)
    gnn = P.GraphNeuralNetwork([P.GatedMessagePassingLayer(H, D, T, "sum") for _ in range(3)], _Embed(), False, False).cuda().eval()
    with torch.no_grad():
        chained = gnn.gnn(h, adj_d, None, None, {}, {}, return_all_states=True)
        with unchained():
            plain = gnn.gnn(h, adj_d, None, None, {}, {}, return_all_states=True)
    assert torch.equal(chained, plain), "chained layer outputs differ from the unchained ones"
