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
"""
from typing import Any, Dict

import torch
from torch import nn

from . import _native as N
from .edgeplan import EdgePlan
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
    for cls in (VarMisuseGraphModel,):
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


class VarMisuseGraphModel(nn.Module):
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

    # ---- metrics protocol (modulewithmetrics.py:8-77) ---------------------------------------------
    def _reset_module_metrics(self) -> None:
        self.__sum_acc = 0          # an int, or a device int64 [1] once a forward has run
        self.__num_samples = 0

    def _module_metrics(self) -> Dict[str, Any]:
        return {"Accuracy": int(self.__sum_acc) / self.__num_samples}

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
