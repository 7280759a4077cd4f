"""Derived-weight cache of GatedMessagePassingLayer (ptgnn_b200_gated_forward, ptgnn_b200_gated_forward_fused): results must be bit-identical
to the fill path, and any in-place parameter update must invalidate it."""
import copy

import pytest
import torch

from helpers import random_adjacency

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_weight_cache_reuse_and_invalidation(dtype):
    import ptgnn_b200 as P
    from ptgnn_b200 import _native as N

    gen = torch.Generator().manual_seed(11)
    torch.manual_seed(3)
    n, H, counts = 2500, 128, [6000, 0, 4000]
    adj = [(s.cuda(), t.cuda()) for s, t in random_adjacency(gen, n, counts)]
    h = torch.randn(n, H, generator=gen).to(dtype).cuda()
    layer = P.GatedMessagePassingLayer(H, H, len(counts), "sum").cuda().eval()
    with torch.no_grad():
        P.GatedMessagePassingLayer(H, H, len(counts), "sum").cuda().eval()(h, adj)   # builds the edge plan of `adj` (cached by identity)
        l0 = N.launch_count()
        out_fill = layer(h, adj)            # derives the working copies into the cache
        l1 = N.launch_count()
        out_hit = layer(h, adj)             # reuses them
        l2 = N.launch_count()
    assert torch.equal(out_fill, out_hit)
    # a cached call launches only the compute kernels -- (state packing,) fused aggregation, GRU -- and skips exactly the two
    # weight-derivation launches: edge-weight packing and GRU gate-block packing
    assert (l2 - l1) == (3 if dtype == torch.float32 else 2) and (l1 - l0) == (l2 - l1) + 2

    # in-place update (what load_state_dict / an optimiser step does): the cache must not be used
    with torch.no_grad():
        for p in layer.parameters():
            p.mul_(0.5)
        out_new = layer(h, adj)
        fresh = copy.deepcopy(layer)        # same parameter values, empty cache
        fresh.invalidate_weight_cache()
        out_ref = fresh(h, adj)
    assert torch.equal(out_new, out_ref)
    assert not torch.equal(out_new, out_hit)

    # training mode never trusts the cache (edits through .data are invisible to the version counter)
    layer.train()
    with torch.no_grad():
        l3 = N.launch_count()
        layer(h, adj)
        l4 = N.launch_count()
    assert (l4 - l3) == (l1 - l0)


def test_mlp_layer_derived_weight_cache():
    """MlpMessagePassingLayer (fused fp32 path): packed edge weights + split dense weight are derived once per parameter version."""
    import ptgnn_b200 as P
    from ptgnn_b200 import _native as N
    from helpers import random_adjacency

    gen = torch.Generator().manual_seed(6)
    torch.manual_seed(6)
    n, counts, H = 3000, [8000, 2500, 0, 40], 128
    adj = [(s.cuda(), t.cuda()) for s, t in random_adjacency(gen, n, counts)]
    h = torch.randn(n, H, generator=gen).cuda()
    layer = P.MlpMessagePassingLayer(H, H, H, len(counts), "max").cuda().eval()
    with torch.no_grad():
        P.MlpMessagePassingLayer(H, H, H, len(counts), "max").cuda().eval()(h, adj)     # builds the plan of `adj`
        l0 = N.launch_count()
        first = layer(h, adj)
        l1 = N.launch_count()
        again = layer(h, adj)
        l2 = N.launch_count()
        assert torch.equal(first, again)
        assert (l1 - l0) - (l2 - l1) == 2, f"the cached call must skip the two weight-derivation launches ({l1 - l0} vs {l2 - l1})"
        for p in layer.parameters():
            p.mul_(1.5)                                                                   # optimiser step / load_state_dict
        changed = layer(h, adj)
        l3 = N.launch_count()
        assert (l3 - l2) == (l1 - l0) and not torch.equal(changed, first)
        fresh = P.MlpMessagePassingLayer(H, H, H, len(counts), "max").cuda().eval()
        fresh.load_state_dict(layer.state_dict())
        assert torch.equal(fresh(h, adj), changed)                                        # the re-derived copies are the right ones
