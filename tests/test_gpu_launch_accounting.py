"""Launch accounting: every kernel the library launches is counted once by ptgnn_b200_launch_count and timed once by the per-kernel
timing records.  For one small call per kind of kernel (forward and backward where both exist), the number of library kernels the
CUDA profiler sees, the launch-count delta and the timing records' summed launches must all be equal.  Library kernels are those whose
names contain ``ptgnn::``: every kernel the library defines lives in that namespace."""
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from helpers import random_adjacency

pytestmark = pytest.mark.gpu


def _adjacency(n, counts, seed=5):
    return [(s.cuda(), t.cuda()) for s, t in random_adjacency(torch.Generator().manual_seed(seed), n, counts)]


def _graph_map(sizes=(40, 0, 130, 7, 300)):
    return torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes)).cuda()


def _plan_build():
    import ptgnn_b200 as P

    adj = _adjacency(700, [2000, 900, 0, 1500])
    return lambda: P.EdgePlan(adj, 700, block_targets=64).validate()


def _gated(H, D, train):
    import ptgnn_b200 as P

    torch.manual_seed(0)
    adj = _adjacency(900, [3000, 1200, 800])
    layer = P.GatedMessagePassingLayer(H, D, len(adj), "sum").cuda().train(train)
    h = torch.randn(900, H, device="cuda", requires_grad=train)
    layer(h, adj)                   # the edge plan of `adj` is built once, outside the counted call

    def call():
        if train:
            layer(h, adj).square().sum().backward()
        else:
            with torch.no_grad():
                layer(h, adj)
    return call


def _egc(dtype):
    import ptgnn_b200 as P

    torch.manual_seed(1)
    adj = _adjacency(800, [2500, 1000])
    layer = P.EGCMessagePassingLayer(128, 128, len(adj), "sum", num_bases=4, num_heads=8).cuda().eval()
    h = torch.randn(800, 128, device="cuda").to(dtype)

    def call():
        with torch.no_grad():
            layer(h, adj)
    return call


def _graph_norm():
    import ptgnn_b200 as P

    n2g = _graph_map()
    layer = P.GraphNorm(64).cuda().train()
    x = torch.randn(n2g.numel(), 64, device="cuda", requires_grad=True)
    return lambda: layer(x, [], n2g, {}, {}, []).square().sum().backward()


def _selfatt_backward():
    import ptgnn_b200 as P

    n2g = _graph_map()
    layer = P.MultiHeadSelfAttentionMessagePassing(32, 16, 16, 32, 64, 2).cuda().train()
    x = torch.randn(n2g.numel(), 32, device="cuda", requires_grad=True)
    return lambda: layer(x, [], n2g, {}, {}, []).square().sum().backward()


def _char_cnn_prepare():
    from ptgnn_b200.embeddings import CharUnitEmbedder, CnnConfig

    torch.manual_seed(2)
    module = CharUnitEmbedder(40, 64, CnnConfig(64, 3, 64, 3, 2)).cuda().eval()
    chars = torch.randint(0, 40, (300, 12), device="cuda")

    def call():
        with torch.no_grad():
            module(chars)           # the first call in eval mode derives the prepared weights, then runs the CNN
    return call


CASES = {
    "plan_build": _plan_build,
    "gated_fused_forward": lambda: _gated(128, 128, False),
    "gated_fused_forward_backward": lambda: _gated(128, 128, True),
    "gated_unfused_forward": lambda: _gated(96, 36, False),
    "gated_unfused_forward_backward": lambda: _gated(96, 36, True),
    "egc_fp32": lambda: _egc(torch.float32),
    "egc_bf16": lambda: _egc(torch.bfloat16),
    "graph_norm_forward_backward": _graph_norm,
    "selfatt_forward_backward": _selfatt_backward,
    "char_cnn_prepare_forward": _char_cnn_prepare,
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_every_launch_is_counted_and_timed_once(case):
    from ptgnn_b200 import _native as N

    call = CASES[case]()
    torch.cuda.synchronize()
    N.kernel_timing(True)
    try:
        N.read_kernel_timing()                      # drop earlier records
        before = N.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        counted = N.launch_count() - before
        timed = sum(launches for _, launches in N.read_kernel_timing().values())
    finally:
        N.kernel_timing(False)
    seen = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "ptgnn::" in e.name]
    assert len(seen) > 0, f"{case}: no library kernel ran"
    assert (len(seen), counted, timed) == (len(seen), len(seen), len(seen)), \
        f"{case}: profiler saw {len(seen)} library kernels, launch_count moved by {counted}, timing recorded {timed}"
