"""Edge plan: the per-minibatch integer bookkeeping shared by every message-passing layer.

The reference re-derives the same information inside every layer call: it concatenates the per-type target lists
(`/root/reference/ptgnn/neuralmodels/gnn/messagepassing/gatedmessagepassing.py:46`,
`mlpmessagepassing.py:102-109`) and lets ``torch_scatter.scatter`` group rows by target
(`abstractmessagepassing.py:44-50`).  Here that grouping is computed ONCE per minibatch on the GPU
(``ptgnn_b200_plan_build``: int64->int32, degree histogram, scan, stable radix sort by target) and reused by all
L layers (the reference's weight-shared stacks call the same layer 7-8 times on the same adjacency).
"""
import os
import threading
from collections import OrderedDict
from typing import List, Optional, Sequence, Tuple

import torch

from . import _native as N

Adjacency = Sequence[Tuple[torch.Tensor, torch.Tensor]]


class EdgePlan:
    """Device-resident CSR-by-target plan (all int32 unless noted).  Field meanings: include/ptgnn_b200.h."""

    __slots__ = (
        "num_nodes", "num_source_nodes", "num_edges", "num_types", "type_off", "type_off_c", "row_ptr", "src32", "tgt32", "status", "device", "_keepalive", "_validated", "_block", "_sorted", "_counts_c",
        "_block_targets",
    )

    # status words (pinned host memory the kernels write directly, so the host can poll them without synchronising):
    # [0] number of out-of-range edge indices, [1] a node state / [2] an edge weight outside the fp16 range of the fp32-exact
    # fused path (csrc/fused_mp.cuh), [3] number of out-of-range indices a task head met (heads.py: candidate, slot node or correct ids)
    STATUS_WORDS = 4

    def __init__(self, adjacency_lists: Adjacency, num_nodes: int, validate: bool = False,
                 num_source_nodes: Optional[int] = None, block_targets: Optional[int] = None):
        """``num_nodes`` = number of TARGET rows (CSR rows).  ``num_source_nodes`` (default: the same) bounds the source
        ids; it differs only for node-range shards, where targets are local rows and sources index the gathered states.
        ``block_targets`` fixes the fused kernel's target-block size B (a multiple of 8 in [8, 176]); None picks
        ``recommended_block_targets(num_nodes)``.  Results do not depend on B; tests use it to reach block layouts (many
        blocks per CTA, small or odd half-blocks) that the recommended size would not produce for their graph."""
        if block_targets is not None:
            bt = int(block_targets)
            if bt != block_targets or bt % 8 != 0 or not 8 <= bt <= 176:     # 176 = fused_mp.cuh kMaxBlockTargets
                raise ValueError(f"block_targets={block_targets!r} must be a multiple of 8 in [8, 176]")
            block_targets = bt
        self._block_targets = block_targets
        if len(adjacency_lists) > 128:
            raise NotImplementedError("more than 128 edge types")
        if len(adjacency_lists) == 0:
            raise ValueError("at least one edge type is required")
        device = adjacency_lists[0][0].device
        srcs = [N.require_cuda(s, f"adjacency_lists[{i}][0]", torch.int64) for i, (s, _) in enumerate(adjacency_lists)]
        tgts = [N.require_cuda(t, f"adjacency_lists[{i}][1]", torch.int64) for i, (_, t) in enumerate(adjacency_lists)]
        counts = [int(s.shape[0]) for s in srcs]
        for s, t in zip(srcs, tgts):
            if s.dim() != 1 or t.shape != s.shape:
                raise ValueError("adjacency lists must be pairs of equal-length 1-D tensors")
        E = sum(counts)
        self.num_nodes, self.num_edges, self.num_types, self.device = int(num_nodes), E, len(counts), device
        self.num_source_nodes = int(num_source_nodes) if num_source_nodes is not None else int(num_nodes)
        self.type_off = [0]
        for c in counts:
            self.type_off.append(self.type_off[-1] + c)
        self.type_off_c = N.i64_array(self.type_off)

        def i32(n):
            return torch.empty(n, dtype=torch.int32, device=device)

        # phase 1 now (int32 edge lists, range check, row_ptr); the target-sorted arrays are built on first use (`_sorted`):
        # layers that run on the fused kernel only need phase 1 + the block plan
        self.row_ptr = i32(num_nodes + 1)
        self.src32, self.tgt32 = i32(E), i32(E)
        self._sorted = None
        self.status = torch.zeros(self.STATUS_WORDS, dtype=torch.int32).pin_memory()
        self._block = None
        self._counts_c = N.i64_array(counts)
        lib = N.lib()
        ws_bytes = lib.ptgnn_b200_plan_workspace_bytes(num_nodes, E)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
        N.call("ptgnn_b200_plan_convert", device, num_nodes, self.num_source_nodes, len(counts), N.ptr_table(srcs), N.ptr_table(tgts),
               self._counts_c, N.ptr(self.row_ptr), N.ptr(self.src32), N.ptr(self.tgt32), N.ptr(self.status), N.ptr(ws), ws_bytes)
        self._keepalive = (srcs, tgts)
        self._validated = False
        if validate:
            self.validate()

    # ---- target-sorted arrays (unfused kernels, scatter): built on first access ---------------------------------------------
    def _sort(self):
        if self._sorted is None:
            E, dev = self.num_edges, self.device
            perm, pos, src_sorted = (torch.empty(E, dtype=torch.int32, device=dev) for _ in range(3))
            etype_sorted = torch.empty(E, dtype=torch.uint8, device=dev)
            if E:
                lib = N.lib()
                ws_bytes = lib.ptgnn_b200_plan_workspace_bytes(self.num_nodes, E)
                ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
                N.call("ptgnn_b200_plan_sort", dev, self.num_nodes, self.num_types, self._counts_c, N.ptr(perm), N.ptr(pos), N.ptr(src_sorted),
                       N.ptr(etype_sorted), N.ptr(self.src32), N.ptr(self.tgt32), N.ptr(ws), ws_bytes)
            self._sorted = (perm, pos, src_sorted, etype_sorted)
        return self._sorted

    perm = property(lambda self: self._sort()[0])
    pos = property(lambda self: self._sort()[1])
    src_sorted = property(lambda self: self._sort()[2])
    etype_sorted = property(lambda self: self._sort()[3])

    def validate(self) -> None:
        """Synchronises the current stream and raises if the plan or a layer that used it reported an error."""
        if not self._validated:
            torch.cuda.current_stream(self.device).synchronize()
            self.poll()
            self._validated = True

    def poll(self) -> None:
        """Host-side look at the status words, WITHOUT synchronising: errors of work that has already executed are raised
        here (every layer call and plan lookup polls), errors of work still in flight at the next poll or `validate()`.
        The reference fails in the same situations (IndexError from F.embedding / a device assert from scatter)."""
        st = self.status
        if int(st[0]):
            raise IndexError(f"{int(st[0])} edge indices outside [0, {self.num_nodes}) (targets) / [0, {self.num_source_nodes}) "
                             "(sources); the kernels route such edges to node 0, results are not valid")
        if int(st[1]) or int(st[2]):
            what = "node states" if int(st[1]) else "edge weights"
            raise FloatingPointError(
                f"{what} outside the fp16 range (|x| >= 65504, inf or NaN) reached the fp32-exact fused kernel (3xFP16 split); "
                "set PTGNN_B200_FP32_MODE=tf32 to use the unfused 3xTF32 kernels for such inputs")
        bad = int(st[3])
        if bad:
            st[3] = 0          # the head's other inputs change from call to call, while this plan may be reused
            raise ValueError(f"{bad} task-head indices out of range (a candidate or slot node id outside [0, N), or a correct candidate "
                             "outside [0, K)); the kernels skipped them, results are not valid")

    # ---- block plan of the fused kernel (built on first use, shared by all layers of the minibatch) ---------------------
    def block_plan(self) -> "N.BlockPlanStruct":
        if self._block is None:
            lib = N.lib()
            B = self._block_targets
            if B is None:
                B = int(lib.ptgnn_b200_block_plan_block_targets(self.num_nodes))
            nblk = (self.num_nodes + B - 1) // B
            dev = self.device
            group_off = torch.empty(nblk * self.num_types + 1, dtype=torch.int32, device=dev)
            src_f = torch.empty(max(self.num_edges, 1), dtype=torch.int32, device=dev)
            tl_f = torch.empty(max(self.num_edges, 1), dtype=torch.uint8, device=dev)
            ws_bytes = lib.ptgnn_b200_block_plan_workspace_bytes(self.num_nodes, self.num_edges, self.num_types, B)
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
            N.call("ptgnn_b200_block_plan_build", dev, self.num_nodes, self.num_types, self.type_off_c, N.ptr(self.src32), N.ptr(self.tgt32),
                   B, N.ptr(group_off), N.ptr(src_f), N.ptr(tl_f), N.ptr(ws), ws_bytes)
            struct = N.BlockPlanStruct(B, N.ptr(group_off), N.ptr(src_f), N.ptr(tl_f), self.status.data_ptr() + 4)
            self._block = (struct, group_off, src_f, tl_f, B)
        return self._block[0]

    @property
    def block_targets(self) -> int:
        self.block_plan()
        return self._block[4]


# ---- small identity-keyed cache so that the L layers of one forward share one plan ----------------
_CACHE: "OrderedDict[tuple, EdgePlan]" = OrderedDict()
_CACHE_SIZE = 4


def _version(t: torch.Tensor):
    try:
        return t._version
    except RuntimeError:       # inference tensors carry no version counter: a sentinel that never compares equal
        return object()


def _key(adjacency_lists: Adjacency, num_nodes: int, num_source_nodes: Optional[int] = None) -> tuple:
    parts: list = [num_nodes, -1 if num_source_nodes is None else num_source_nodes]
    for s, t in adjacency_lists:
        parts += [s.data_ptr(), s.shape[0], _version(s), t.data_ptr(), _version(t)]
    return tuple(parts)


# ---- plan hand-off from a container to its layers: per thread, never process-global ---------------------------------------
_TLS = threading.local()


def current_shared_plan() -> Optional[EdgePlan]:
    return getattr(_TLS, "plan", None)


class shared_plan:
    """`with shared_plan(plan):` -- layers called inside (on this thread) use `plan` if it matches their adjacency lists'
    edge / node counts; nests; other threads are unaffected (the reference builds minibatches on background threads)."""

    def __init__(self, plan: Optional[EdgePlan]):
        self.plan, self.previous = plan, None

    def __enter__(self):
        self.previous = getattr(_TLS, "plan", None)
        _TLS.plan = self.plan
        return self.plan

    def __exit__(self, *exc):
        _TLS.plan = self.previous
        return False


class shared_num_graphs:
    """`with shared_num_graphs(G):` -- per-thread hand-off of the minibatch's graph count from a container to its global-exchange
    layers (ptgnn_b200.globalexchange), which then never read it from the device.  None hands nothing over; nests."""

    def __init__(self, num_graphs: Optional[int]):
        self.num_graphs, self.previous = num_graphs, None

    def __enter__(self):
        self.previous = getattr(_TLS, "num_graphs", None)
        _TLS.num_graphs = self.num_graphs
        return self.num_graphs

    def __exit__(self, *exc):
        _TLS.num_graphs = self.previous
        return False


def current_num_graphs() -> Optional[int]:
    return getattr(_TLS, "num_graphs", None)


class state_chain:
    """`with state_chain() as chain:` -- per-thread hand-off of PACKED node states between consecutive layers of one layer loop.
    The fp32 fused path computes on fp16 (hi | lo') pairs; a GatedMessagePassingLayer called with `chain.want_output` set also
    returns that packed form of its output (written by its GRU kernel), and the next layer -- if it is handed the very same tensor
    object -- skips its packing pass.  Nothing is attached to tensors and nothing outlives the `with` block."""

    def __init__(self):
        self.want_output = False
        self._tensor: Optional[torch.Tensor] = None
        self._packed: Optional[torch.Tensor] = None
        self._version = None
        self.previous = None

    def __enter__(self):
        self.previous = getattr(_TLS, "chain", None)
        _TLS.chain = self
        return self

    def __exit__(self, *exc):
        _TLS.chain = self.previous
        self._tensor = self._packed = None
        return False

    def lookup(self, node_states: torch.Tensor) -> Optional[torch.Tensor]:
        if self._tensor is node_states and self._packed is not None and _version(node_states) == self._version:
            return self._packed
        return None

    def store(self, out_states: torch.Tensor, packed: Optional[torch.Tensor]) -> None:
        self._tensor, self._packed = (out_states, packed) if packed is not None else (None, None)
        self._version = _version(out_states) if packed is not None else None


def current_state_chain() -> Optional[state_chain]:
    if os.environ.get("PTGNN_B200_CHAIN", "1") == "0":
        return None
    return getattr(_TLS, "chain", None)


def plan_for(adjacency_lists: Adjacency, num_nodes: int, plan: Optional[EdgePlan] = None,
             num_source_nodes: Optional[int] = None) -> EdgePlan:
    """Returns the plan for these adjacency tensors, building it on a cache miss.  Entries keep their index tensors
    alive, so a (data_ptr, version) key cannot alias different contents."""
    if plan is not None and _matches(plan, adjacency_lists, num_nodes, num_source_nodes):
        plan.poll()
        return plan
    key = _key(adjacency_lists, num_nodes, num_source_nodes)
    hit = _CACHE.get(key)
    if hit is not None:
        _CACHE.move_to_end(key)
        hit.poll()
        return hit
    built = EdgePlan(adjacency_lists, num_nodes, num_source_nodes=num_source_nodes)
    _CACHE[key] = built
    while len(_CACHE) > _CACHE_SIZE:
        _CACHE.popitem(last=False)
    return built


def _matches(plan: EdgePlan, adjacency_lists: Adjacency, num_nodes: int, num_source_nodes: Optional[int]) -> bool:
    """A handed-over plan is only used for the call it was built for (same node / edge / type counts per type)."""
    if plan.num_nodes != num_nodes or plan.num_types != len(adjacency_lists):
        return False
    if num_source_nodes is not None and plan.num_source_nodes != num_source_nodes:
        return False
    return all(plan.type_off[i + 1] - plan.type_off[i] == int(s.shape[0]) for i, (s, _) in enumerate(adjacency_lists))


def clear_plan_cache() -> None:
    _CACHE.clear()
