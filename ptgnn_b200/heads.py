"""Task heads with the reference's ``nn.Module`` API, on native kernels.

``VarMisuseGraphModel`` is the counterpart of `implementations/varmisuse/varmisuse.py:41-91` of the reference: it calls its GNN exactly as
the reference does, then scores every candidate with ``Linear(2H -> 1, bias=False)`` on ``[candidate row ; its slot's row]``, takes the
log-softmax of the scores within each slot, and returns the mean negative log-probability of the correct candidates.  Here the whole
head is ``ptgnn_b200_varmisuse_forward`` (DESIGN.md §3.16): one warp per slot computes the scores, the slot's logsumexp and its argmax in
one walk over the slot's candidates, so the ``[K, 2H]`` concatenation is never formed.  The accuracy count stays on the device; reading
``_module_metrics()`` is the only host synchronisation.

* Gradients (fp32): ``autograd._VarMisuseFn``.  Its backward is the full softmax gradient,
  ``d score_k = (g / S) (p_k n_slot(k) - m_k)``, scattered into ``[N, H]`` in a fixed order.  The reference run on
  ``ptgnn_b200.torch_scatter_shim`` gets no gradient through the normaliser (the shim's ``scatter_max`` / ``scatter_sum`` are not
  differentiable); this class is what ``overlay.install(native_heads=True)`` binds in its place.
* bf16 node states (under autocast) run the forward with the weight rounded to bf16 and the products accumulated in fp32; gradients
  with bf16 states raise ``NotImplementedError``.
* A candidate or slot node id outside ``[0, N)`` or a correct candidate outside ``[0, K)`` is counted in the slot plan's status word:
  ``ValueError`` at the next poll (this call if the kernel has already run).  A slot id outside ``[0, num_slots)`` is an ``IndexError``
  of the plan.  Not supported (``NotImplementedError``): a state size that is not a multiple of 4 in [4, 1024].
``Graph2ClassModule`` (`implementations/typilus/graph2class.py:63-102`, the Typilus model) and ``PPIClassification``
(`implementations/ppi/ppi.py:13-62`) are the reference's classification heads on ``ptgnn_b200_classify_forward`` (DESIGN.md §3.17): one
wgmma kernel forms ``logits = rows W^T + b`` (rows gathered through the supernode ids for Graph2Class) and reduces each row in its
epilogue to the cross-entropy's logsumexp, target logit and argmax, or to the BCE sum and the TP / FP / FN counts of PPI's
``sigmoid(x) >= 0.5``; the ``[rows, C]`` logits never reach memory.  The loss and the metrics are finished on the device: the accuracy
counter and PPI's fscore / precision / recall sums (fp64, the reference's Python-double arithmetic) stay there until
``_module_metrics()``, the only host synchronisation -- the reference's PPI head synchronises three times per forward.

* Gradients (fp32): ``autograd._ClassifyFn``: d logits from one launch that recomputes the logits, d W and d b as split library GEMMs
  and a column sum, d states on the native linear, summed per node over repeated supernode ids in a fixed order.
* bf16 (``torch.autocast("cuda", torch.bfloat16)`` or bf16 states): one bf16 product; the logits are rounded to bf16 where autocast's
  Linear rounds them, and the losses, the argmax and the sigmoid (itself rounded to bf16) are taken on the rounded values.  Gradients
  with bf16 raise ``NotImplementedError``.
* A supernode id outside ``[0, N)`` or a target class outside ``[0, C)`` (other than ``-100``, ignored as ``nn.CrossEntropyLoss`` does)
  is counted on the device and raises ``ValueError`` at the next poll (this call when the kernel has already run).  Not supported
  (``NotImplementedError``, before any launch): a state size that is not a multiple of 8 in [8, 256], more than 256 classes.
* ``predict`` takes the largest probability as ``1 / sum exp(logit - max)``, which is torch's softmax at its maximum.  Where two logits
  are within a probability rounding of each other, torch's ``torch.max`` over the rounded probabilities can pick the other index; the
  kernel picks the first largest logit.
"""
from typing import Any, Dict, Optional

import torch
from torch import nn

from . import _native as N
from .edgeplan import EdgePlan
from .embeddings import _NativeEmbedder
from .reduceops import graph_plan

_STATUS_WORD = 3        # the word of EdgePlan.status the head kernels count bad indices in (EdgePlan.poll raises ValueError)


def register_with_reference_metrics() -> bool:
    """Makes the native heads (virtual) subclasses of the reference's ``ModuleWithMetrics`` once that class has been imported, so that a
    reference parent's ``report_metrics()`` / ``reset_metrics()`` reach them (as ``gnn.register_with_reference_metrics`` does for the
    container)."""
    import sys

    base = getattr(sys.modules.get("ptgnn.baseneuralmodel.modulewithmetrics"), "ModuleWithMetrics", None)
    if base is None or not hasattr(base, "register"):
        return False
    for cls in (VarMisuseGraphModel, Graph2ClassModule, PPIClassification):
        if not issubclass(cls, base):
            base.register(cls)
    return True


def varmisuse_check(H: int) -> None:
    if not N.lib().ptgnn_b200_varmisuse_supported(H):
        raise NotImplementedError(f"the VarMisuse head kernel takes a state size that is a multiple of 4 in [4, 1024], got {H}")


def _index(t: torch.Tensor, name: str) -> torch.Tensor:
    t = N.require_cuda(t, name, torch.int64)
    if t.dim() != 1:
        raise ValueError(f"{name} must be a 1-D tensor, got {tuple(t.shape)}")
    return t


def _states(h: torch.Tensor, bf16: bool) -> torch.Tensor:
    h = N.require_cuda(h.detach(), "output_node_representations", torch.bfloat16 if bf16 else torch.float32)
    if h.dim() != 2:
        raise ValueError(f"output_node_representations must be [N, H], got {tuple(h.shape)}")
    return h if h.data_ptr() % 16 == 0 else h.clone()       # the kernels load four columns at once


def varmisuse_inputs(h, candidate_nodes, candidate_slot, slot_nodes, correct, weight):
    """Checked kernel operands: (h, cand, slot_of, slot_nodes, correct, w [2H] fp32, plan of the slots)."""
    bf16 = h.dtype == torch.bfloat16
    H = h.shape[-1]
    varmisuse_check(H)
    h = _states(h, bf16)
    cand, slot_of = _index(candidate_nodes, "candidate_nodes"), _index(candidate_slot, "candidate slot ids")
    slot_nodes, correct = _index(slot_nodes, "slot_node_idx"), _index(correct, "correct_candidate_idxs")
    if slot_of.shape != cand.shape:
        raise ValueError(f"{cand.shape[0]} candidate nodes but {slot_of.shape[0]} candidate slot ids")
    w = N.require_cuda(weight.detach(), "candidate score weight", torch.float32).reshape(-1)
    if w.shape[0] != 2 * H:
        raise ValueError(f"the candidate score weight must have 2 H = {2 * H} entries, got {w.shape[0]}")
    return h, cand, slot_of, slot_nodes, correct, w, graph_plan(slot_of, slot_nodes.shape[0])


def native_varmisuse(h, cand, slot_of, slot_nodes, correct, w, plan: EdgePlan, hits=None):
    """``ptgnn_b200_varmisuse_forward``: (loss [] fp32, score [K] fp32, lse [J] fp32, argmax [J] int64) for checked operands
    (``varmisuse_inputs``).  ``hits``: a device int64 [1] the number of correctly ranked slots is added to (when S == J)."""
    dev = h.device
    K, J, S = cand.shape[0], slot_nodes.shape[0], correct.shape[0]
    loss = torch.empty((), dtype=torch.float32, device=dev)
    score = torch.empty(K, dtype=torch.float32, device=dev)
    lse = torch.empty(J, dtype=torch.float32, device=dev)
    arg = torch.empty(J, dtype=torch.int64, device=dev)
    N.call("ptgnn_b200_varmisuse_forward", dev, int(h.dtype == torch.bfloat16), N.ptr(h), h.shape[0], h.shape[1], N.ptr(cand), N.ptr(slot_of),
           N.ptr(plan.row_ptr), N.ptr(plan.perm) if K else None, K, N.ptr(slot_nodes), J, N.ptr(correct), S, N.ptr(w), N.ptr(score),
           N.ptr(lse), N.ptr(arg), N.ptr(loss), N.ptr(hits), plan.status.data_ptr() + 4 * _STATUS_WORD)
    return loss, score, lse, arg


def native_varmisuse_backward(h, cand, slot_of, slot_nodes, correct, w, plan: EdgePlan, score, lse, grad_loss):
    """``ptgnn_b200_varmisuse_backward_f32``: (d h [N, H], d w [2H]) for d loss = grad_loss (a device scalar), fp32 states."""
    dev = h.device
    num_nodes, H = h.shape
    K, J, S = cand.shape[0], slot_nodes.shape[0], correct.shape[0]
    node_ids = torch.cat([cand, slot_nodes])
    # a plan of this call's own, outside the plan cache: its ids are new on every call, so a cached entry would never be hit and
    # would only push out the plans the GNN layers share
    node_plan = EdgePlan([(node_ids, node_ids)], num_nodes)
    ws_bytes = N.lib().ptgnn_b200_varmisuse_workspace_bytes(K, J, H)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    d_h = torch.empty(num_nodes, H, dtype=torch.float32, device=dev)
    d_w = torch.empty(2 * H, dtype=torch.float32, device=dev)
    g = N.require_cuda(grad_loss.reshape(()), "grad_loss", torch.float32)
    N.call("ptgnn_b200_varmisuse_backward_f32", dev, N.ptr(h), num_nodes, H, N.ptr(cand), N.ptr(slot_of), N.ptr(plan.row_ptr),
           N.ptr(plan.perm) if K else None, K, N.ptr(slot_nodes), J, N.ptr(correct), S, N.ptr(w), N.ptr(score), N.ptr(lse), N.ptr(g),
           N.ptr(node_plan.row_ptr), N.ptr(node_plan.perm) if K + J else None, N.ptr(d_h), N.ptr(d_w), N.ptr(ws), ws_bytes)
    node_plan.poll()
    return d_h, d_w


class _MetricsProtocol(nn.Module):
    """The reference's ``ModuleWithMetrics`` protocol (modulewithmetrics.py:8-77) over a subclass's ``_module_metrics`` and
    ``_reset_module_metrics``."""

    def report_metrics(self) -> Dict[str, Any]:
        metrics = self._module_metrics()
        for child in self.modules():
            if child is not self and hasattr(child, "_module_metrics"):
                metrics.update(child._module_metrics())
        return metrics

    def reset_metrics(self) -> None:
        for child in self.modules():
            if hasattr(child, "_reset_module_metrics"):
                child._reset_module_metrics()

    def train(self, mode: bool = True):
        self.reset_metrics()
        return super().train(mode=mode)

    def eval(self):
        self.reset_metrics()
        return super().eval()


class VarMisuseGraphModel(_MetricsProtocol):
    """The reference's VarMisuse model (GNN + candidate-selection head) with the head on ``ptgnn_b200_varmisuse_forward`` (DESIGN.md
    §3.16).  Implements the reference's ``ModuleWithMetrics`` protocol; ``Accuracy`` is counted on the device."""

    def __init__(self, gnn: nn.Module):
        super().__init__()
        self._reset_module_metrics()
        self._gnn = gnn
        self.__candidate_scores = nn.Linear(
            self._gnn.output_node_state_dim + self._gnn.output_node_state_dim,
            1,
            bias=False,
        )
        register_with_reference_metrics()

    def _reset_module_metrics(self) -> None:
        self.__sum_acc = 0          # an int, or a device int64 [1] once a forward has run
        self.__num_samples = 0

    def _module_metrics(self) -> Dict[str, Any]:
        return {"Accuracy": int(self.__sum_acc) / self.__num_samples}

    def _hits(self, device: torch.device) -> torch.Tensor:
        acc = self.__sum_acc
        if not isinstance(acc, torch.Tensor):
            acc = torch.full((1,), acc, dtype=torch.int64, device=device)
        elif acc.device != device:
            acc = acc.to(device)
        self.__sum_acc = acc
        return acc

    def forward(self, graph_data, correct_candidate_idxs):
        from . import autograd as _ag

        gnn_output = self._gnn(**graph_data)
        h = gnn_output.output_node_representations
        weight = self.__candidate_scores.weight
        grad = torch.is_grad_enabled() and (h.requires_grad or weight.requires_grad)
        if grad and h.dtype == torch.bfloat16:
            raise NotImplementedError("VarMisuseGraphModel: gradients with bf16 node states have no native kernel; train in fp32")
        ops = varmisuse_inputs(h, gnn_output.node_idx_references["candidate_nodes"], gnn_output.node_graph_idx_reference["candidate_nodes"],
                               gnn_output.node_idx_references["slot_node_idx"], correct_candidate_idxs, weight)
        num_slots, plan = ops[3].shape[0], ops[6]
        if ops[4].shape[0] != num_slots:
            raise ValueError(f"{ops[4].shape[0]} correct candidates for {num_slots} slots: the head takes one per slot")
        hits = self._hits(h.device)
        if grad:
            loss = _ag.varmisuse_with_grad(ops, hits, h, weight)
        else:
            loss = native_varmisuse(*ops, hits=hits)[0]
        plan.poll()
        self.__num_samples += int(num_slots)
        return loss


# ---- classification heads (DESIGN.md §3.17) --------------------------------------------------------------------------------------
CLASSIFY_LOGITS, CLASSIFY_CE, CLASSIFY_BCE = 0, 1, 2


def classify_check(H: int, C: int) -> None:
    if not N.lib().ptgnn_b200_classify_supported(H, C):
        raise NotImplementedError(f"the classification head kernel takes a state size that is a multiple of 8 in [8, 256] and 1 to 256 "
                                  f"classes, got H={H}, C={C}")


def classify_prepare(weight: torch.Tensor, bf16: bool, status: Optional[torch.Tensor]) -> torch.Tensor:
    """``ptgnn_b200_classify_prepare``: W [C, H] in the feature embedder's prepared format, columns padded to 16."""
    C, H = weight.shape
    w = N.require_cuda(weight.detach(), "weight", torch.float32)
    nbytes = N.lib().ptgnn_b200_classify_prepared_bytes(int(bf16), H, C)
    prepared = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
    N.call("ptgnn_b200_classify_prepare", w.device, int(bf16), N.ptr(w), H, C, N.ptr(prepared), nbytes,
           None if status is None else status.data_ptr() + 4)
    return prepared


def poll_classify_status(status: torch.Tensor, what: str) -> None:
    bad, out_of_range = int(status[0]), int(status[1])
    if bad:
        status[0] = 0
        raise ValueError(f"{what}: {bad} supernode ids outside [0, num_nodes) or target classes outside [0, num_classes) (other than "
                         "-100); their rows were skipped, results are not valid")
    if out_of_range:
        status[1] = 0
        raise FloatingPointError(f"{what}: an fp32 state or weight is outside the fp16 range (|x| >= 65504) of the kernel's split "
                                 "products; results are not valid")


class ClassifyOps:
    """Checked operands of one head call: mode, states, row ids (or None), targets, prepared weights and bias, bf16 flag."""

    def __init__(self, mode, h, idx, targets, prepared, bias, bf16, status):
        self.mode, self.h, self.idx, self.targets, self.prepared, self.bias, self.bf16, self.status = (
            mode, h, idx, targets, prepared, bias, bf16, status)
        self.rows = h.shape[0] if idx is None else idx.shape[0]


def native_classify(ops: ClassifyOps, num_classes: int, hits=None, metrics=None, want_logits=False, want_prob=False):
    """``ptgnn_b200_classify_forward``: (loss [] or None, lse [R], argmax [R] int64, valid [1] int32, max_prob [R] or None, logits [R, C] or
    None, safe ids [R] int32 or None).  The safe ids (with row ids) are the row ids with those outside [0, N) replaced by 0: a backward
    gathers and scatters through them, since a bad id may not have been reported yet when it runs."""
    h, dev, R, C = ops.h, ops.h.device, ops.rows, num_classes
    loss = torch.empty((), dtype=torch.float32, device=dev) if ops.mode != CLASSIFY_LOGITS else None
    lse = torch.empty(R, dtype=torch.float32, device=dev)
    arg = torch.empty(R, dtype=torch.int64, device=dev)
    valid = torch.zeros(1, dtype=torch.int32, device=dev)
    prob = torch.empty(R, dtype=torch.float32, device=dev) if want_prob else None
    logits = torch.empty(R, C, dtype=torch.float32, device=dev) if want_logits else None
    safe = torch.empty(R, dtype=torch.int32, device=dev) if ops.idx is not None else None
    lib = N.lib()
    ws_bytes = lib.ptgnn_b200_classify_workspace_bytes(int(ops.bf16), R, h.shape[1], C)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    N.call("ptgnn_b200_classify_forward", dev, ops.mode, int(ops.bf16), int(h.dtype == torch.bfloat16), N.ptr(h), h.shape[0], h.shape[1],
           N.ptr(ops.idx), R, C, N.ptr(ops.prepared), ops.prepared.numel(), N.ptr(ops.bias), N.ptr(ops.targets), N.ptr(logits), N.ptr(loss),
           N.ptr(lse), N.ptr(arg), N.ptr(prob), N.ptr(valid), N.ptr(hits), N.ptr(metrics), N.ptr(safe), N.ptr(ws), ws_bytes,
           ops.status.data_ptr())
    return loss, lse, arg, valid, prob, logits, safe


def native_classify_backward(ops: ClassifyOps, num_classes: int, lse, valid, grad_loss) -> torch.Tensor:
    """``ptgnn_b200_classify_backward_f32``: d logits [R, C] fp32 for d loss = grad_loss (a device scalar); zero rows for bad ids."""
    h, dev = ops.h, ops.h.device
    d_logits = torch.empty(ops.rows, num_classes, dtype=torch.float32, device=dev)
    g = N.require_cuda(grad_loss.reshape(()), "grad_loss", torch.float32)
    N.call("ptgnn_b200_classify_backward_f32", dev, ops.mode, N.ptr(h), h.shape[0], h.shape[1], N.ptr(ops.idx), ops.rows, num_classes,
           N.ptr(ops.prepared), ops.prepared.numel(), N.ptr(ops.bias), N.ptr(ops.targets), N.ptr(lse), N.ptr(valid), N.ptr(g),
           N.ptr(d_logits))
    return d_logits


def classify_input_grads(ops: ClassifyOps, safe_idx, weight: torch.Tensor, d_logits: torch.Tensor, want_h: bool, want_w: bool,
                         want_b: bool):
    """(d h [N, H], d W [C, H], d b [C]) from d logits [R, C]: d W = d logits^T rows as split library GEMMs (rows gathered and split in
    one native pass), d b its column sum, d rows = d logits W on the native linear, summed into the nodes of the supernode ids in id
    order through a plan of this call's own (kept out of the plan cache, as the VarMisuse backward's).  ``safe_idx``: the forward's
    int32 safe ids (``native_classify``), or None without row ids; the gather has no bounds check of its own."""
    from . import autograd as _ag
    from . import composed as C
    from .edgeplan import EdgePlan

    h = ops.h
    d_w = d_b = d_h = None
    if want_w:
        rows = _ag._split16(h, safe_idx)
        d_w = _ag._mm_t_split(_ag._split16(d_logits), rows)
    if want_b:
        d_b = d_logits.sum(dim=0)
    if want_h:
        d_rows = C.linear(d_logits, weight.detach().t().contiguous())
        if safe_idx is None:
            d_h = d_rows
        else:
            ids = safe_idx.long()
            plan = EdgePlan([(ids, ids)], h.shape[0])
            d_h = C.segment_reduce(d_rows, plan, N.REDUCE["sum"])
            plan.poll()
    return d_h, d_w, d_b


class _ClassificationHead(_NativeEmbedder, _MetricsProtocol):
    """What both classification heads share: the pinned status words ([0] bad ids, [1] fp16 range), the prepared weights of eval
    mode and the call of the kernels."""

    _STATUS_WORDS = 2

    def _prepared(self, weight: torch.Tensor, bf16: bool, status: torch.Tensor) -> torch.Tensor:
        """Derived on every call in training mode; kept in eval mode while the weight is not modified in place, re-assigned or moved."""
        if self.training:
            return classify_prepare(weight, bf16, status)
        key = (bf16, weight.data_ptr(), weight._version, weight.device, weight.dtype)
        if self._transformed is None or self._transformed[0] != key:
            self._transformed = (key, classify_prepare(weight, bf16, status))
        return self._transformed[1]

    def _ops(self, mode: int, linear: nn.Linear, h: torch.Tensor, idx: Optional[torch.Tensor], targets, grad: bool) -> ClassifyOps:
        from .embeddings import _bf16_autocast

        what = type(self).__name__
        weight, bias = linear.weight, linear.bias
        C, H = weight.shape
        classify_check(H, C)
        bf16 = h.dtype == torch.bfloat16 or _bf16_autocast(weight.device)
        if grad and bf16:
            raise NotImplementedError(f"{what}: gradients with bf16 logits have no native kernel; train in fp32")
        if h.dim() != 2 or h.shape[1] != H:
            raise ValueError(f"output_node_representations must be [N, {H}], got {tuple(h.shape)}")
        h = _states(h, h.dtype == torch.bfloat16)
        if idx is not None:
            idx = _index(idx, "supernode ids")
        rows = h.shape[0] if idx is None else idx.shape[0]
        if mode == CLASSIFY_CE:
            targets = _index(targets, "target_classes")
            if targets.shape[0] != rows:
                raise ValueError(f"{targets.shape[0]} target classes for {rows} supernodes")
        elif mode == CLASSIFY_BCE:
            targets = N.require_cuda(targets, "targets", torch.bool)
            if tuple(targets.shape) != (rows, C):
                raise ValueError(f"targets must be [{rows}, {C}], got {tuple(targets.shape)}")
        N.require_cuda(weight, "weight", torch.float32)
        b = N.require_cuda(bias.detach(), "bias", torch.float32)
        status = self._status_word()
        poll_classify_status(status, what)
        return ClassifyOps(mode, h, idx, targets, self._prepared(weight, bf16, status), b, bf16, status)

    def _loss(self, mode: int, linear: nn.Linear, h: torch.Tensor, idx, targets, hits=None, metrics=None) -> torch.Tensor:
        from . import autograd as _ag

        grad = torch.is_grad_enabled() and (h.requires_grad or linear.weight.requires_grad or linear.bias.requires_grad)
        ops = self._ops(mode, linear, h, idx, targets, grad)
        if grad:
            loss = _ag.classify_with_grad(ops, hits, metrics, h, linear.weight, linear.bias)
        else:
            loss = native_classify(ops, linear.weight.shape[0], hits=hits, metrics=metrics)[0]
        poll_classify_status(ops.status, type(self).__name__)
        return loss


def _device_accumulator(acc, shape, dtype, device: torch.device) -> torch.Tensor:
    if not isinstance(acc, torch.Tensor):
        return torch.full(shape, acc, dtype=dtype, device=device)
    return acc if acc.device == device else acc.to(device)


class Graph2ClassModule(_ClassificationHead):
    """The reference's Typilus model (GNN + supernode classifier, graph2class.py:63-102) with the head on ``ptgnn_b200_classify_forward``
    (DESIGN.md §3.17).  Implements the ``ModuleWithMetrics`` protocol; ``Accuracy`` is counted on the device."""

    def __init__(self, gnn: nn.Module, num_target_classes: int):
        super().__init__()
        self._reset_module_metrics()
        self.__gnn = gnn
        self.__node_to_class = nn.Linear(in_features=gnn.output_node_state_dim, out_features=num_target_classes)
        nn.init.uniform_(self.__node_to_class.weight)
        nn.init.zeros_(self.__node_to_class.bias)
        self.__loss = nn.CrossEntropyLoss()
        register_with_reference_metrics()

    def _reset_module_metrics(self) -> None:
        self.__num_samples = 0
        self.__sum_accuracy = 0         # an int, or a device int64 [1] once a forward has run

    def _module_metrics(self) -> Dict[str, Any]:
        return {"Accuracy": int(self.__sum_accuracy) / int(self.__num_samples)}

    def _supernodes(self, graph_mb_data):
        graph_output = self.__gnn(**graph_mb_data)
        return (graph_output.output_node_representations, graph_output.reference_nodes_idx["supernodes"],
                graph_output.reference_nodes_graph_idx["supernodes"])

    def _logits(self, graph_mb_data):
        """(logits [S, C], supernode graph ids): fp32, bf16 under autocast, as the reference's Linear returns them."""
        from . import autograd as _ag

        h, idx, graph_idx = self._supernodes(graph_mb_data)
        lin = self.__node_to_class
        grad = torch.is_grad_enabled() and (h.requires_grad or lin.weight.requires_grad or lin.bias.requires_grad)
        ops = self._ops(CLASSIFY_LOGITS, lin, h, idx, None, grad)
        if grad:
            logits = _ag.classify_logits_with_grad(ops, h, lin.weight, lin.bias)
        else:
            logits = native_classify(ops, lin.weight.shape[0], want_logits=True)[5]
        poll_classify_status(ops.status, "Graph2ClassModule")
        return (logits.to(torch.bfloat16) if ops.bf16 else logits), graph_idx

    def predict(self, graph_mb_data):
        """(largest class probability [S] fp32, its class [S] int64, supernode graph ids [S])."""
        with torch.no_grad():
            h, idx, graph_idx = self._supernodes(graph_mb_data)
            lin = self.__node_to_class
            ops = self._ops(CLASSIFY_LOGITS, lin, h, idx, None, False)
            _, _, arg, _, prob, _, _ = native_classify(ops, lin.weight.shape[0], want_prob=True)
            poll_classify_status(ops.status, "Graph2ClassModule")
            return prob, arg, graph_idx

    def forward(self, graph_mb_data, target_classes, original_supernode_idxs):
        h, idx, _ = self._supernodes(graph_mb_data)
        hits = self.__sum_accuracy = _device_accumulator(self.__sum_accuracy, (1,), torch.int64, h.device)
        loss = self._loss(CLASSIFY_CE, self.__node_to_class, h, idx, target_classes, hits=hits)
        self.__num_samples += target_classes.shape[0]
        return loss


class PPIClassification(_ClassificationHead):
    """The reference's PPI model (GNN + per-node multi-label classifier, ppi.py:13-62) with the head on ``ptgnn_b200_classify_forward``
    (DESIGN.md §3.17).  The fscore, precision and recall sums stay on the device until ``_module_metrics()``."""

    def __init__(self, gnn: nn.Module, num_target_classes: int):
        super().__init__()
        self._reset_module_metrics()
        self.__gnn = gnn
        self.__output_representation_to_logits = nn.Linear(in_features=gnn.output_node_state_dim, out_features=num_target_classes)
        nn.init.xavier_uniform_(self.__output_representation_to_logits.weight)
        nn.init.zeros_(self.__output_representation_to_logits.bias)
        register_with_reference_metrics()

    def _reset_module_metrics(self) -> None:
        self.__num_samples = 0
        self.__sums = 0.0               # fscore, precision, recall times samples: a float, or a device fp64 [3] once a forward has run

    def _module_metrics(self) -> Dict[str, Any]:
        f1, pr, re = self.__sums.tolist() if isinstance(self.__sums, torch.Tensor) else (self.__sums,) * 3
        return {"f1_score": f1 / self.__num_samples, "pr_score": pr / self.__num_samples, "re_score": re / self.__num_samples}

    def forward(self, graph_data, targets):
        gnn_output = self.__gnn(**graph_data)
        h = gnn_output.output_node_representations
        sums = self.__sums = _device_accumulator(self.__sums, (3,), torch.float64, h.device)
        loss = self._loss(CLASSIFY_BCE, self.__output_representation_to_logits, h, None, targets, metrics=sums)
        self.__num_samples += int(h.shape[0])
        return loss
