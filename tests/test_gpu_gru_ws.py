"""The weights-stationary GRU kernel (csrc/gru_ws.cu) hands its output on in packed form: a container's chained layers must equal
layers that pack their own inputs.  Its values are checked element by element against float64 in ``test_gpu_gru_ws_edges.py``."""
import pytest
import torch

from helpers import random_adjacency, unchained

pytestmark = pytest.mark.gpu

T = 3
D = 128


def _graph(N, seed):
    gen = torch.Generator().manual_seed(seed)
    adj = random_adjacency(gen, N, [max(1, 2 * N), max(1, N), max(1, N // 2)])
    return adj, [(s.cuda(), t.cuda()) for s, t in adj], gen


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
