"""Device-side minibatch finalisation for the graph-structure part of a GNN minibatch (SURVEY.md §8 row f-2).

Host-side mirror of the three minibatching methods of the reference's ``GraphNeuralNetworkModel``
(`/root/reference/ptgnn/neuralmodels/gnn/graphneuralnetwork.py:372-493`): ``initialize_minibatch`` / ``extend_minibatch_with`` /
``finalize_minibatch`` -- same dictionary keys, same tensors (int64, on the device) -- for everything that does not belong to
the node / edge embedders (those keep their own ``extend_minibatch_with`` / ``finalize_minibatch``).

What moves to the GPU: the reference offsets every graph's edge arrays in numpy as the graph is appended (:419-424, :436),
concatenates per edge type (:463-469) and materialises ``node_to_graph_idx`` through a Python generator that yields once per node
(:441-443) -- at 200k nodes per minibatch that loop alone is ~100x the layer time.  Here ``extend_minibatch_with`` only records
references to the graphs' local int32 arrays; ``finalize_minibatch`` concatenates them (one memcpy per array), ships ONE pinned
host buffer per minibatch and lets two kernels (csrc/batching.cu) add the node offsets and expand the segment ids.
"""
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _native as N


class MinibatchAssembler:
    """``initialize_minibatch() -> dict``, ``extend_minibatch_with(graph, dict) -> bool``, ``finalize_minibatch(dict, device) -> dict``
    with the reference's contract; ``graph`` is anything with ``adjacency_lists`` (per edge type a pair of int arrays with LOCAL
    node ids), ``reference_nodes`` (name -> int array) and ``num_nodes`` -- i.e. the reference's ``TensorizedGraphData``."""

    def __init__(self, num_edge_types: int, stop_extending_minibatch_after_num_nodes: int = 10000):
        self.num_edge_types = int(num_edge_types)
        self.stop_extending_minibatch_after_num_nodes = int(stop_extending_minibatch_after_num_nodes)

    def initialize_minibatch(self) -> Dict[str, Any]:
        return {
            "adjacency_lists": [([], []) for _ in range(self.num_edge_types)],
            "num_nodes_per_graph": [],
            "reference_node_ids": {},
            "num_nodes_in_mb": 0,
        }

    def extend_minibatch_with(self, tensorized_datapoint, partial_minibatch: Dict[str, Any]) -> bool:
        adj = tensorized_datapoint.adjacency_lists
        assert len(adj) == self.num_edge_types, "one adjacency list per edge type is required"
        graph_idx = len(partial_minibatch["num_nodes_per_graph"])
        num_nodes = int(tensorized_datapoint.num_nodes)
        if not 0 <= num_nodes < 2 ** 31:
            raise ValueError("a graph's node count must fit int32 (local ids travel as int32)")
        for (src, tgt), (mb_src, mb_tgt) in zip(adj, partial_minibatch["adjacency_lists"]):
            assert len(src) == len(tgt)
            mb_src.append(np.asarray(src))        # LOCAL ids (< num_nodes of this graph): the node offset is added on the device
            mb_tgt.append(np.asarray(tgt))
        for ref_name, ref_nodes in tensorized_datapoint.reference_nodes.items():
            partial_minibatch["reference_node_ids"].setdefault(ref_name, []).append((graph_idx, np.asarray(ref_nodes)))
        partial_minibatch["num_nodes_per_graph"].append(int(tensorized_datapoint.num_nodes))
        partial_minibatch["num_nodes_in_mb"] += int(tensorized_datapoint.num_nodes)
        return partial_minibatch["num_nodes_in_mb"] < self.stop_extending_minibatch_after_num_nodes

    # ---- finalisation ---------------------------------------------------------------------------------------------------------
    def finalize_minibatch(self, accumulated_minibatch_data: Dict[str, Any], device: Union[str, torch.device]) -> Dict[str, Any]:
        device = torch.device(device)
        if device.type != "cuda":
            raise N.NativeLibraryError("MinibatchAssembler.finalize_minibatch builds the minibatch on a CUDA device (no CPU fallback)")
        sizes = np.asarray(accumulated_minibatch_data["num_nodes_per_graph"], dtype=np.int64)
        G = int(sizes.shape[0])
        node_ptr = np.zeros(G + 1, dtype=np.int64)
        np.cumsum(sizes, out=node_ptr[1:])
        num_nodes = int(node_ptr[-1])

        # one staging buffer: int64 pointer arrays first (8-byte aligned), then the int32 local ids
        ptr_arrays: List[np.ndarray] = [node_ptr]
        id_arrays: List[np.ndarray] = []
        jobs: List[Tuple[str, Any, int, int, int]] = []         # (kind, key, ptr slot, id slot, item count)

        def add_job(kind: str, key, per_graph: Sequence[np.ndarray]):
            counts = np.fromiter((len(a) for a in per_graph), dtype=np.int64, count=G)
            item_ptr = np.zeros(G + 1, dtype=np.int64)
            np.cumsum(counts, out=item_ptr[1:])
            total = int(item_ptr[-1])
            local = np.concatenate(per_graph).astype(np.int32, copy=False) if total else np.zeros(0, dtype=np.int32)
            return item_ptr, local, total

        for t, (srcs, tgts) in enumerate(accumulated_minibatch_data["adjacency_lists"]):
            item_ptr, local_src, total = add_job("adj", t, srcs)
            _, local_tgt, _ = add_job("adj", t, tgts)
            ptr_arrays.append(item_ptr)
            id_arrays += [local_src, local_tgt]
            jobs.append(("adj", t, len(ptr_arrays) - 1, len(id_arrays) - 2, total))
        empty = np.zeros(0, dtype=np.int32)
        for name, entries in accumulated_minibatch_data["reference_node_ids"].items():
            per_graph = [empty] * G
            for g, arr in entries:
                per_graph[g] = arr if per_graph[g] is empty else np.concatenate([per_graph[g], arr])
            item_ptr, local, total = add_job("ref", name, per_graph)
            ptr_arrays.append(item_ptr)
            id_arrays.append(local)
            jobs.append(("ref", name, len(ptr_arrays) - 1, len(id_arrays) - 1, total))

        ptr_words = sum(a.shape[0] for a in ptr_arrays)
        id_words = sum(a.shape[0] for a in id_arrays)
        staging = torch.empty(ptr_words * 8 + id_words * 4, dtype=torch.uint8).pin_memory()
        host = staging.numpy()
        ptr_view = host[: ptr_words * 8].view(np.int64)
        id_view = host[ptr_words * 8:].view(np.int32)
        ptr_off, id_off, o = [], [], 0
        for a in ptr_arrays:
            ptr_view[o:o + a.shape[0]] = a
            ptr_off.append(o)
            o += a.shape[0]
        o = 0
        for a in id_arrays:
            id_view[o:o + a.shape[0]] = a
            id_off.append(o)
            o += a.shape[0]
        dev = staging.to(device, non_blocking=True)
        ptr_dev = dev[: ptr_words * 8].view(torch.int64)
        id_dev = dev[ptr_words * 8:].view(torch.int32)

        def offset(id_slot: int, ptr_slot: int, total: int) -> torch.Tensor:
            out = torch.empty(total, dtype=torch.int64, device=device)
            if total:
                N.call("ptgnn_b200_offset_ids", device, id_dev[id_off[id_slot]:].data_ptr(), total, ptr_dev[ptr_off[ptr_slot]:].data_ptr(),
                       ptr_dev.data_ptr(), G, out.data_ptr())
            return out

        def segments(ptr_slot: int, total: int) -> torch.Tensor:
            out = torch.empty(total, dtype=torch.int64, device=device)
            if total:
                N.call("ptgnn_b200_segment_ids", device, ptr_dev[ptr_off[ptr_slot]:].data_ptr(), G, total, out.data_ptr())
            return out

        adjacency_lists: List[Optional[Tuple[torch.Tensor, torch.Tensor]]] = [None] * self.num_edge_types
        reference_node_ids: Dict[str, torch.Tensor] = {}
        reference_node_graph_idx: Dict[str, torch.Tensor] = {}
        for kind, key, ptr_slot, id_slot, total in jobs:
            if kind == "adj":
                adjacency_lists[key] = (offset(id_slot, ptr_slot, total), offset(id_slot + 1, ptr_slot, total))
            else:
                reference_node_ids[key] = offset(id_slot, ptr_slot, total)
                reference_node_graph_idx[key] = segments(ptr_slot, total)
        node_to_graph_idx = segments(0, num_nodes)
        return {
            "adjacency_lists": adjacency_lists,
            "node_to_graph_idx": node_to_graph_idx,
            "reference_node_graph_idx": reference_node_graph_idx,
            "reference_node_ids": reference_node_ids,
            "num_graphs": G,
        }
