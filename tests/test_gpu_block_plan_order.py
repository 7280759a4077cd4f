"""The block plan (csrc/plan.cu) byte for byte against its definition: edges ordered by (target block, edge type, target - block
start, edge id), computed here with numpy's lexsort.  The GPU builds it with atomic slots and per-group sorts, so the cases reach
what that can get wrong: the benchmark graphs, the smallest and largest block sizes, groups too large for one warp's shared-memory
sort (a hub target, a dense block), empty types and blocks, source ids bounded separately from targets, and out-of-range ids."""
import numpy as np
import pytest
import torch

from helpers import random_adjacency

pytestmark = pytest.mark.gpu


def _expanded(adj, n):
    ident = torch.arange(n, dtype=torch.int64)
    return list(adj) + [(t, s) for s, t in adj] + [(ident, ident)]


def _reference(adj, n, n_src, B):
    src = np.concatenate([s.numpy() for s, _ in adj])
    tgt = np.concatenate([t.numpy() for _, t in adj])
    src = np.where((src < 0) | (src >= n_src), 0, src)       # out-of-range ids are routed to node 0 (and counted)
    tgt = np.where((tgt < 0) | (tgt >= n), 0, tgt)
    T = len(adj)
    etype = np.repeat(np.arange(T), [s.shape[0] for s, _ in adj])
    blk, tl = tgt // B, tgt % B
    order = np.lexsort((np.arange(src.shape[0]), tl, etype, blk))
    nblk = (n + B - 1) // B
    group_off = np.zeros(nblk * T + 1, dtype=np.int64)
    np.cumsum(np.bincount(blk * T + etype, minlength=nblk * T), out=group_off[1:])
    row_ptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(tgt, minlength=n), out=row_ptr[1:])
    return {"group_off": group_off.astype(np.int32), "src_f": src[order].astype(np.int32), "tl_f": tl[order].astype(np.uint8),
            "row_ptr": row_ptr.astype(np.int32), "src32": src.astype(np.int32), "tgt32": tgt.astype(np.int32)}


def _block_plan(plan, B):
    """ptgnn_b200_block_plan_build at any B the C entry point takes ([8, 256]); EdgePlan itself caps B at the fused kernel's 176."""
    from ptgnn_b200 import _native as N

    dev = plan.device
    nblk = (plan.num_nodes + B - 1) // B
    group_off = torch.full((nblk * plan.num_types + 1,), -7, dtype=torch.int32, device=dev)
    src_f = torch.full((max(plan.num_edges, 1),), -7, dtype=torch.int32, device=dev)
    tl_f = torch.full((max(plan.num_edges, 1),), 0xAB, dtype=torch.uint8, device=dev)
    ws_bytes = N.lib().ptgnn_b200_block_plan_workspace_bytes(plan.num_nodes, plan.num_edges, plan.num_types, B)
    ws = torch.full((max(ws_bytes, 1),), 0x5A, dtype=torch.uint8, device=dev)     # stale contents must not matter
    N.call("ptgnn_b200_block_plan_build", dev, plan.num_nodes, plan.num_types, plan.type_off_c, N.ptr(plan.src32), N.ptr(plan.tgt32), B,
           N.ptr(group_off), N.ptr(src_f), N.ptr(tl_f), N.ptr(ws), ws_bytes)
    torch.cuda.synchronize()
    return group_off, src_f, tl_f


def _check(adj, n, block_targets, n_src=None, expect_bad=0):
    import ptgnn_b200 as P

    plan = P.EdgePlan([(s.cuda(), t.cuda()) for s, t in adj], n, num_source_nodes=n_src)
    torch.cuda.synchronize()
    assert int(plan.status[0]) == expect_bad
    E = plan.num_edges
    for B in block_targets:
        if B is None:                                           # the size EdgePlan picks, through its own block plan
            plan.block_plan()
            B = plan.block_targets
            _, group_off, src_f, tl_f, _ = plan._block
            torch.cuda.synchronize()
        else:
            group_off, src_f, tl_f = _block_plan(plan, B)
        ref = _reference(adj, n, n if n_src is None else n_src, B)
        got = {"group_off": group_off, "src_f": src_f[:E], "tl_f": tl_f[:E], "row_ptr": plan.row_ptr, "src32": plan.src32,
               "tgt32": plan.tgt32}
        for k, want in ref.items():
            have = got[k].cpu().numpy()
            assert have.dtype == want.dtype and np.array_equal(have, want), (B, k)
        again = _block_plan(plan, B)                           # a rebuild is byte-identical, whatever order the atomics took
        assert all(torch.equal(a, b) for a, b in zip(again, (group_off, src_f, tl_f))), B


def test_graph2class_config():
    from ptgnn_b200.synthetic import graph2class_batch

    b = graph2class_batch()
    _check(_expanded(b.adjacency_lists, b.num_nodes), b.num_nodes, [None, 8, 256])


def test_varmisuse_config():
    from ptgnn_b200.synthetic import varmisuse_batch

    b = varmisuse_batch()
    _check(_expanded(b.adjacency_lists, b.num_nodes), b.num_nodes, [None, 8, 256])


def test_star_graph():
    """One target with 300,000 in-edges of one type: a group far above a warp's 256 words, sorted in several radix passes."""
    gen = torch.Generator().manual_seed(3)
    n = 5000
    hub = (torch.randint(0, n, (300_000,), generator=gen), torch.full((300_000,), 1234, dtype=torch.int64))
    adj = [hub] + random_adjacency(gen, n, [20_000, 700])
    _check(adj, n, [None, 8, 256])


def test_dense_blocks():
    """Few nodes, many edges: every group is large and its targets vary, so each of the five digits of a word takes a pass."""
    gen = torch.Generator().manual_seed(4)
    _check(random_adjacency(gen, 200, [70_000, 257, 256, 3000]), 200, [None, 8, 256])


def test_empty_types_and_blocks():
    """Types without edges, and targets only in a few node ranges, so most (block, type) groups and whole blocks are empty."""
    gen = torch.Generator().manual_seed(5)
    n = 3000
    tgt = torch.cat([torch.randint(0, 40, (900,), generator=gen), torch.randint(2600, 2700, (600,), generator=gen)])
    adj = [(torch.zeros(0, dtype=torch.int64),) * 2, (torch.randint(0, n, (1500,), generator=gen), tgt),
           (torch.zeros(0, dtype=torch.int64),) * 2, (torch.randint(0, n, (3,), generator=gen), torch.tensor([2999, 0, 2999]))]
    _check(adj, n, [None, 8, 256])


def test_separate_source_bound():
    """num_source_nodes != num_nodes, as on node-range shards: sources index a larger gathered state array."""
    gen = torch.Generator().manual_seed(6)
    n, n_src = 1500, 40_000
    adj = [(torch.randint(0, n_src, (c,), generator=gen), torch.randint(0, n, (c,), generator=gen)) for c in (5000, 0, 2500)]
    _check(adj, n, [None, 8, 256], n_src=n_src)


def test_out_of_range_ids():
    """Out-of-range sources and targets are counted in the status word and the plan is built with them routed to node 0."""
    gen = torch.Generator().manual_seed(7)
    n = 1000
    adj = random_adjacency(gen, n, [4000, 1200])
    adj[0][0][[3, 17]] = torch.tensor([-1, n])
    adj[1][1][[0, 5, 9]] = torch.tensor([n, n + 100, -5])
    _check(adj, n, [None, 8, 256], expect_bad=5)
