"""The host-buffer C-ABI entry point (`ptgnn_b200_gated_gnn_forward_host_f32`) and the alternative operand-staging mode
of the tensor-core pipeline."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import assert_close, gated_oracle_args, random_adjacency
from oracle import ptgnn_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ptrs(arrs, ctype):
    tab = (ctypes.c_void_p * len(arrs))()
    for i, a in enumerate(arrs):
        tab[i] = a.ctypes.data
    return tab


@pytest.mark.parametrize("agg", ["sum", "max"])
def test_gnn_forward_from_host_buffers(agg):
    import ptgnn_b200 as P
    from ptgnn_b200 import _native as N

    n, H, L, counts = 2000, 64, 3, [7000, 0, 3000]
    gen = torch.Generator().manual_seed(5)
    torch.manual_seed(6)
    adj = random_adjacency(gen, n, counts)
    h = torch.randn(n, H, generator=gen)
    layers = [P.GatedMessagePassingLayer(H, H, len(counts), agg) for _ in range(L)]
    sds = [{k: v.clone() for k, v in l.state_dict().items()} for l in layers]
    ref = h
    for sd in sds:
        ref = O.gated_layer_forward(ref, adj, [torch.empty(c, 0) for c in counts], aggregation_fn=agg, **gated_oracle_args(sd))

    srcs = [np.ascontiguousarray(s.numpy()) for s, _ in adj]
    tgts = [np.ascontiguousarray(t.numpy()) for _, t in adj]
    cnt = (ctypes.c_int64 * len(counts))(*counts)
    ws, wih, whh, bih, bhh = [], [], [], [], []
    for sd in sds:
        a = gated_oracle_args(sd)
        ws += [np.ascontiguousarray(w.numpy()) for w in a["edge_weights"]]
        wih.append(np.ascontiguousarray(a["gru_w_ih"].numpy())); whh.append(np.ascontiguousarray(a["gru_w_hh"].numpy()))
        bih.append(np.ascontiguousarray(a["gru_b_ih"].numpy())); bhh.append(np.ascontiguousarray(a["gru_b_hh"].numpy()))
    h_np = np.ascontiguousarray(h.numpy())
    out = np.zeros_like(h_np)
    rc = N.lib().ptgnn_b200_gated_gnn_forward_host_f32(
        h_np.ctypes.data, n, H, len(counts), _ptrs(srcs, ctypes.c_int64), _ptrs(tgts, ctypes.c_int64), cnt, L,
        _ptrs(ws, ctypes.c_float), _ptrs(wih, ctypes.c_float), _ptrs(whh, ctypes.c_float), _ptrs(bih, ctypes.c_float),
        _ptrs(bhh, ctypes.c_float), N.REDUCE[agg], out.ctypes.data)
    N.check(rc, "ptgnn_b200_gated_gnn_forward_host_f32")
    assert_close(torch.from_numpy(out), ref, tol=3e-5, what=f"host entry point, {L} chained layers")   # 3 layers deep


def test_host_entry_point_reports_bad_indices():
    from ptgnn_b200 import _native as N

    n, H = 10, 32
    src = np.array([0, 99], dtype=np.int64)
    tgt = np.array([1, 2], dtype=np.int64)
    w = np.zeros((H, H), np.float32); w3 = np.zeros((3 * H, H), np.float32); b = np.zeros(3 * H, np.float32)
    h = np.zeros((n, H), np.float32); out = np.zeros_like(h)
    rc = N.lib().ptgnn_b200_gated_gnn_forward_host_f32(
        h.ctypes.data, n, H, 1, _ptrs([src], ctypes.c_int64), _ptrs([tgt], ctypes.c_int64), (ctypes.c_int64 * 1)(2), 1,
        _ptrs([w], ctypes.c_float), _ptrs([w3], ctypes.c_float), _ptrs([w3], ctypes.c_float), _ptrs([b], ctypes.c_float),
        _ptrs([b], ctypes.c_float), 0, out.ctypes.data)
    assert rc == -5 and b"outside" in N.lib().ptgnn_b200_last_error()


