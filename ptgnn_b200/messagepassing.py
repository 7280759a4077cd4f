"""Message-passing layers with the reference's ``nn.Module`` API, computed by the CUDA library.

Drop-in for the classes the reference's factories construct
(`/root/reference/ptgnn/implementations/typilus/train.py:39-99`, `ppi/train.py:36-57`, `varmisuse/train.py:42-107`):

* ``AbstractMessagePassingLayer``  -- `/root/reference/ptgnn/neuralmodels/gnn/messagepassing/abstractmessagepassing.py:8-60`
* ``GatedMessagePassingLayer``     -- `.../gatedmessagepassing.py:8-77`
* ``MlpMessagePassingLayer``       -- `.../mlpmessagepassing.py:12-125`
* ``MLP``                          -- `/root/reference/ptgnn/neuralmodels/mlp.py:9-80`

Constructor signatures, properties, parameter initialisation order and (name-mangled) ``state_dict`` keys are the
reference's, so reference checkpoints load with ``load_state_dict``.  ``forward`` never touches PyTorch arithmetic:
it hands raw device pointers to ``libptgnn_b200.so``.  Configurations without a native kernel raise
``NotImplementedError`` (there is no silent fallback): training-mode dropout outside the gated layer's fp32 paths, autograd
outside the trainable layers (SURVEY.md §8 f-1), edge features (f-4), hidden message-MLP layers and module aggregators such as
PNA (f-3).
"""
from abc import abstractmethod
from typing import Dict, List, Optional, Tuple, Union

import torch
from torch import nn

import ctypes
import os

from . import _native as N
from .edgeplan import EdgePlan, current_shared_plan, current_state_chain, plan_for

_ACTIVATION_CODES = {type(None): N.ACT_NONE, nn.GELU: N.ACT_GELU, nn.Tanh: N.ACT_TANH, nn.ReLU: N.ACT_RELU}


def _activation_code(module: Optional[nn.Module], what: str) -> int:
    code = _ACTIVATION_CODES.get(type(module))
    if code is None or (isinstance(module, nn.GELU) and getattr(module, "approximate", "none") != "none"):
        raise NotImplementedError(f"{what}={module!r} has no native kernel (supported: GELU(erf), Tanh, ReLU, None)")
    return code


def _reduce_code(name) -> int:
    if not isinstance(name, str) or name not in N.REDUCE:
        raise NotImplementedError(f"message aggregation {name!r} has no native kernel (supported: sum, mean, max, min)")
    return N.REDUCE[name]


def _refuse_autograd(module: nn.Module, node_states: torch.Tensor) -> None:
    if torch.is_grad_enabled() and (node_states.requires_grad or any(p.requires_grad for p in module.parameters())):
        raise NotImplementedError(
            "this configuration is forward-only (backward, SURVEY.md §8 row f-1, exists for GatedMessagePassingLayer with fp32 "
            "states and no edge features, and for MlpMessagePassingLayer with its default message MLP: fp32 states, or bf16 states "
            "with a string aggregation): call it under torch.no_grad() / torch.inference_mode(), or set requires_grad_(False) "
            "on the parameters"
        )


def fused_allowed(bf16: bool) -> bool:
    """The fused gather -> Linear -> reduce kernel runs wherever it supports the dimensions, except for fp32 states under
    PTGNN_B200_FP32_MODE=tf32, which selects the round-1 three-kernel path (3xTF32 instead of 3xFP16: needed for states /
    weights beyond the fp16 range)."""
    return bf16 or os.environ.get("PTGNN_B200_FP32_MODE", "") != "tf32"


def _use_fused(lib, bf16: bool, H: int, D: int) -> bool:
    return fused_allowed(bf16) and bool(lib.ptgnn_b200_fused_supported(int(bf16), H, D))


def _native_dropout(lib, H: int, D: int) -> bool:
    """GatedMessagePassingLayer's per-edge dropout (fp32 states) runs natively at these dims: inside the fused aggregation where it
    takes them, else on the three-kernel path's masked message kernel."""
    return _use_fused(lib, False, H, D) or bool(lib.ptgnn_b200_gated_dropout_supported(H, D))


def _mlp_bf16_grad_supported(lib, H: int, D: int, use_target: bool) -> bool:
    """MlpMessagePassingLayer (default message MLP, string aggregation) trains with bf16 states at these dims: the bf16 forward runs
    (fused or three-kernel), the gathered weight-gradient kernel takes them, and the bf16 aggregation runs on the transposed graph
    (K = D, D' = H) for d h."""
    forward = _use_fused(lib, True, H, D) or bool(lib.ptgnn_b200_edge_messages_bf16_supported(H, D))
    transposed = _use_fused(lib, True, D, H) or bool(lib.ptgnn_b200_edge_messages_bf16_supported(D, H))
    return forward and transposed and bool(lib.ptgnn_b200_edge_weight_grad_bf16_supported(H, D))


def _check_states(node_states: torch.Tensor, expected_dim: int, what: str) -> None:
    if node_states.dim() != 2 or node_states.shape[1] != expected_dim:
        raise ValueError(f"{what}: node_states must be [num_nodes, {expected_dim}], got {tuple(node_states.shape)}")


def _check_shape(t: torch.Tensor, shape: Tuple[int, ...], name: str) -> None:
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} must have shape {tuple(shape)}, got {tuple(t.shape)}")


def _check_no_edge_features(edge_features: Optional[List[torch.Tensor]]) -> None:
    for f in edge_features or []:
        if f is not None and f.dim() == 2 and f.shape[1] != 0:
            raise NotImplementedError("edge features (F > 0) have no native kernel yet (SURVEY.md §8 row f-4)")


class AbstractMessagePassingLayer(nn.Module):
    """Interface of a message passing layer over multiple edge types (same contract as the reference's)."""

    @abstractmethod
    def forward(
        self,
        node_states: torch.Tensor,
        adjacency_lists: List[Tuple[torch.Tensor, torch.Tensor]],
        node_to_graph_idx: torch.Tensor,
        reference_node_ids: Dict[str, torch.Tensor],
        reference_node_graph_idx: Dict[str, torch.Tensor],
        edge_features: List[torch.Tensor],
    ) -> torch.Tensor:
        """[num_nodes, D] states + per-type (src, tgt) int64 lists -> [num_nodes, D'] states."""

    def _aggregate_messages(self, messages: torch.Tensor, message_targets: torch.Tensor, num_nodes, aggregation_fn: str):
        """Same contract as the reference helper: fp32 reduce, result cast back to the message dtype."""
        from .scatter import scatter

        return scatter(messages.to(torch.float32), message_targets, dim=0, dim_size=num_nodes, reduce=aggregation_fn).to(
            messages.dtype
        )

    def _plan(self, adjacency_lists, num_nodes: int, num_source_nodes: Optional[int] = None) -> EdgePlan:
        """The plan a container prepared for this minibatch on this thread (`edgeplan.shared_plan`) if it matches the call,
        else the identity-keyed cache / a fresh build."""
        return plan_for(adjacency_lists, num_nodes, current_shared_plan(), num_source_nodes)

    # ---- derived-weight cache ------------------------------------------------------------------------------------------
    def _weight_cache(self, kind: str, nbytes: int, params: List[torch.Tensor], device: torch.device):
        """Returns (buffer or None, valid).  The buffer holds the kernels' working copies of the parameters (TF32 hi/lo
        splits and the gate-blocked GRU packing, or their bf16 versions); it is valid while no parameter has been
        modified in place (`Tensor._version`), re-assigned (`data_ptr`) or moved since the call that filled it.  All
        uses are ordered on the layer's CUDA stream; a call on a different stream refills the buffer."""
        if nbytes <= 0:
            return None, False
        stream = torch.cuda.current_stream(device).cuda_stream
        def version(p: torch.Tensor):
            try:
                return p._version
            except RuntimeError:        # inference tensors carry no version counter: never reuse
                return object()

        key = (tuple((p.data_ptr(), version(p)) for p in params), nbytes, stream)
        if not hasattr(self, "_derived_weights"):
            self._derived_weights = {}
        entry = self._derived_weights.get((kind, device))
        if entry is None or entry["buf"].numel() != nbytes:
            entry = {"buf": torch.empty(nbytes, dtype=torch.uint8, device=device), "key": None, "pending": None}
            self._derived_weights[(kind, device)] = entry
        # eval mode only: in-place edits made through `param.data` do not move the version counter, and training loops
        # are where those happen -- in training mode the copies are simply re-derived every call
        valid = (not self.training) and entry["key"] == key
        entry["pending"] = key
        return entry["buf"], valid

    def invalidate_weight_cache(self) -> None:
        """Forget the derived copies (needed only after editing parameters through `.data` in eval mode)."""
        self._derived_weights = {}

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_derived_weights"] = {}      # device scratch, not part of the module's state
        return state

    def _weight_cache_filled(self, kind: str, device: torch.device) -> None:
        entry = getattr(self, "_derived_weights", {}).get((kind, device))
        if entry is not None and entry["pending"] is not None:
            entry["key"], entry["pending"] = entry["pending"], None

    def _apply(self, fn, *args, **kwargs):
        # .to() / .cuda() / .float(): device copies of the parameters derived for the old placement are dead
        if hasattr(self, "_derived_weights"):
            self._derived_weights = {}
        return super()._apply(fn, *args, **kwargs)

    @staticmethod
    def _gather_source(gather_states: Optional[torch.Tensor], h: torch.Tensor) -> Optional[torch.Tensor]:
        """Node-range shards (ptgnn_b200.sharding): `node_states` holds this rank's rows (targets, local ids) and
        `gather_states` the all-gathered states that the source ids index.  None in the ordinary single-GPU case."""
        if gather_states is None:
            return None
        g = N.require_cuda(gather_states, "gather_states", h.dtype)
        if g.dim() != 2 or g.shape[1] != h.shape[1]:
            raise ValueError("gather_states must be [num_source_nodes, H]")
        return g

    @property
    @abstractmethod
    def input_state_dimension(self) -> int:
        pass

    @property
    @abstractmethod
    def output_state_dimension(self) -> int:
        pass


class AbstractMessageAggregation(nn.Module):
    @abstractmethod
    def forward(self, messages: torch.Tensor, message_targets: torch.Tensor, num_nodes):
        pass

    @abstractmethod
    def output_state_size(self, message_input_size: int) -> int:
        pass


class GatedMessagePassingLayer(AbstractMessagePassingLayer):
    """GGNN layer:  m_e = W_t(e) h_src(e);  a_v = reduce m_e;  h'_v = GRUCell(a_v, h_v)."""

    def __init__(
        self,
        state_dimension: int,
        message_dimension: int,
        num_edge_types: int,
        message_aggregation_function: str,
        dropout_rate: float = 0.0,
        edge_feature_dimension: int = 0,
    ):
        super().__init__()
        # construction + initialisation order follows the reference (gatedmessagepassing.py:20-35) so that the
        # same torch seed yields the same parameters.
        self.__edge_message_transformation_layers = nn.ModuleList(
            nn.Linear(state_dimension + edge_feature_dimension, message_dimension, bias=False)
            for _ in range(num_edge_types)
        )
        gain = (1 / num_edge_types) ** 0.5
        for linear in self.__edge_message_transformation_layers:
            nn.init.xavier_normal_(linear.weight, gain=gain)
        self.__state_update = nn.GRUCell(input_size=message_dimension, hidden_size=state_dimension)
        nn.init.orthogonal_(self.__state_update.weight_hh)
        nn.init.xavier_uniform_(self.__state_update.weight_ih)
        nn.init.normal_(self.__state_update.bias_hh, std=1e-5)
        nn.init.normal_(self.__state_update.bias_ih, std=1e-5)
        self.__state_dimension = state_dimension
        self.__message_dimension = message_dimension
        self.__edge_feature_dimension = edge_feature_dimension
        self.__aggregation_fn = message_aggregation_function
        self.__dropout = nn.Dropout(p=dropout_rate)
        # device copies of the parameters in the kernels' working formats, keyed by the parameters' storage + version
        # counters (see _weight_cache): derived once per set of parameter values instead of once per call
        self._derived_weights = {}

    def forward(
        self,
        node_states: torch.Tensor,
        adjacency_lists: List[Tuple[torch.Tensor, torch.Tensor]],
        node_to_graph_idx: torch.Tensor = None,
        reference_node_ids: Dict[str, torch.Tensor] = None,
        reference_node_graph_idx: Dict[str, torch.Tensor] = None,
        edge_features: List[torch.Tensor] = None,
        gather_states: Optional[torch.Tensor] = None,
    ) -> torch.Tensor:
        linears = self.__edge_message_transformation_layers
        assert len(adjacency_lists) == len(linears), "one adjacency list per edge type is required"
        if self.__edge_feature_dimension == 0:
            _check_no_edge_features(edge_features)
        reduce = _reduce_code(self.__aggregation_fn)
        from . import autograd as _ag
        drop_p = self.__dropout.p if self.training else 0.0
        grad = _ag.needs_grad(self, node_states)
        if (drop_p > 0 and gather_states is None and node_states.dtype == torch.float32 and self.__edge_feature_dimension == 0
                and _native_dropout(N.lib(), self.__state_dimension, self.__message_dimension)):
            # per-edge dropout (gatedmessagepassing.py:59) inside the native kernels: the mask is a function of a per-call key
            _check_states(node_states, self.__state_dimension, "GatedMessagePassingLayer")
            h = N.require_cuda(node_states, "node_states", torch.float32)
            if grad:
                gru = self.__state_update
                return _ag.gated_dropout_with_grad(self, h, adjacency_lists, self.__aggregation_fn, drop_p, gru.weight_ih, gru.weight_hh,
                                                   gru.bias_ih, gru.bias_hh, [lin.weight for lin in linears])
            return self._forward_dropout(h, adjacency_lists, _ag.draw_dropout_key(h.device), drop_p)
        if drop_p > 0 or (grad and self.__edge_feature_dimension != 0):
            # per-edge dropout outside the native kernels' dimensions / edge features under autograd: the gathered rows have to exist --
            # the layer as the reference writes it, Linear / scatter / GRUCell on the native kernels as differentiable operators
            if gather_states is not None or node_states.dtype != torch.float32:
                raise NotImplementedError("training-mode dropout / edge features with gradients: fp32 states, unsharded only")
            _check_states(node_states, self.__state_dimension, "GatedMessagePassingLayer")
            h = N.require_cuda(node_states, "node_states", torch.float32)
            return _ag.gated_forward_composed([lin.weight for lin in linears], self.__state_update, h, adjacency_lists,
                                              edge_features if self.__edge_feature_dimension != 0 else None, self.__aggregation_fn, drop_p)
        if grad:
            # backward (SURVEY.md §8 f-1): fp32 states, unsharded; the forward below runs unchanged under no_grad inside the Function
            if gather_states is not None or node_states.dtype != torch.float32:
                _refuse_autograd(self, node_states)
            _check_states(node_states, self.__state_dimension, "GatedMessagePassingLayer")
            gru = self.__state_update
            return _ag.gated_forward_with_grad(self, node_states, adjacency_lists, self.__aggregation_fn, gru.weight_ih, gru.weight_hh,
                                               gru.bias_ih, gru.bias_hh, [lin.weight for lin in linears])
        if self.__edge_feature_dimension != 0:
            return self._forward_with_edge_features(node_states, adjacency_lists, edge_features, gather_states, reduce)

        state_dtype = node_states.dtype if node_states.dtype == torch.bfloat16 else torch.float32
        _check_states(node_states, self.__state_dimension, "GatedMessagePassingLayer")
        h = N.require_cuda(node_states, "node_states", state_dtype)
        num_nodes, H = h.shape
        D = self.__message_dimension
        gsrc = self._gather_source(gather_states, h)
        plan = self._plan(adjacency_lists, num_nodes, None if gsrc is None else gsrc.shape[0])
        gru = self.__state_update
        weights = [N.require_cuda(lin.weight, "edge weight", torch.float32) for lin in linears]
        w_ih, w_hh = N.require_cuda(gru.weight_ih, "weight_ih", torch.float32), N.require_cuda(gru.weight_hh, "weight_hh", torch.float32)
        b_ih, b_hh = N.require_cuda(gru.bias_ih, "bias_ih", torch.float32), N.require_cuda(gru.bias_hh, "bias_hh", torch.float32)
        for i, w in enumerate(weights):      # raw pointers cross the C ABI next: the shapes must be what the kernels assume
            _check_shape(w, (D, H), f"edge weight {i}")
        _check_shape(w_ih, (3 * H, D), "GRUCell.weight_ih"); _check_shape(w_hh, (3 * H, H), "GRUCell.weight_hh")
        _check_shape(b_ih, (3 * H,), "GRUCell.bias_ih"); _check_shape(b_hh, (3 * H,), "GRUCell.bias_hh")

        lib = N.lib()
        params = weights + [w_ih, w_hh, b_ih, b_hh]
        bf16 = state_dtype == torch.bfloat16
        if plan.num_edges > 0 and _use_fused(lib, bf16, H, D):
            # gather -> W_t -> segmented reduce in ONE kernel (no [E, D] message tensor), then the GRUCell kernel
            kind = "bf16_fused" if bf16 else "f32_fused"
            cache, valid = self._weight_cache(kind, lib.ptgnn_b200_gated_fused_weight_cache_bytes(int(bf16), plan.num_types, H, D), params, h.device)
            ns = num_nodes if gsrc is None else gsrc.shape[0]
            ws_bytes = lib.ptgnn_b200_gated_fused_workspace_bytes(int(bf16), num_nodes, ns, plan.num_types, H, D)
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=h.device)
            out = torch.empty_like(h)
            bp = plan.block_plan()
            # inside a container's layer loop (fp32 states): take the packed form of the input from the previous layer, hand the
            # packed form of the output to the next one (edgeplan.state_chain) -- one packing pass per stack instead of one per layer
            chain = None if bf16 else current_state_chain()
            packed_in = chain.lookup(node_states) if (chain is not None and h is node_states) else None
            packed_out = None
            if chain is not None and chain.want_output:
                packed_out = torch.empty(max(lib.ptgnn_b200_packed_state_bytes(num_nodes, H), 1), dtype=torch.uint8, device=h.device)
            N.call("ptgnn_b200_gated_forward_fused", h.device, int(bf16), N.ptr(h), N.ptr(gsrc), N.ptr(packed_in), num_nodes, ns, H, D,
                   plan.num_types, ctypes.byref(bp), N.ptr(plan.row_ptr), N.ptr_table(weights), N.ptr(w_ih), N.ptr(w_hh), N.ptr(b_ih),
                   N.ptr(b_hh), reduce, N.ptr(out), N.ptr(packed_out), N.ptr(ws), ws_bytes, N.ptr(cache),
                   0 if cache is None else cache.numel(), int(valid))
            self._weight_cache_filled(kind, h.device)
            if chain is not None:
                chain.store(out, packed_out)
            return out
        # round-1 three-kernel path; bf16 states: fp32 parameters (converted inside the library), fp32 accumulation
        kind = "bf16" if bf16 else "f32"
        cache, valid = self._weight_cache(kind, lib.ptgnn_b200_gated_weight_cache_bytes(int(bf16), plan.num_types, H, D), params, h.device)
        ws_bytes = lib.ptgnn_b200_gated_workspace_bytes(int(bf16), num_nodes, plan.num_edges, plan.num_types, H, D)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=h.device)
        out = torch.empty_like(h)
        N.call("ptgnn_b200_gated_forward", h.device, int(bf16), N.ptr(h), N.ptr(gsrc), num_nodes, H, D, plan.num_types, plan.type_off_c,
               N.ptr(plan.row_ptr), N.ptr(plan.pos), N.ptr(plan.src32), N.ptr_table(weights), N.ptr(w_ih), N.ptr(w_hh), N.ptr(b_ih),
               N.ptr(b_hh), reduce, N.ptr(out), N.ptr(ws), ws_bytes, N.ptr(cache), 0 if cache is None else cache.numel(), int(valid))
        self._weight_cache_filled(kind, h.device)
        return out

    @property
    def edge_dropout_active(self) -> bool:
        """Training mode with per-edge dropout at dims the fused kernel takes: the layer's fused path then needs the plan's
        ``block_edge_ids`` (the three-kernel path reads the mask in cat(types) order and needs none)."""
        return self.training and self.__dropout.p > 0 and _use_fused(N.lib(), False, self.__state_dimension, self.__message_dimension)

    def _dropout_params(self, H: int, D: int):
        """(edge weights, w_ih, w_hh, b_ih, b_hh) of the dropout paths, checked for the shapes the kernels assume."""
        gru = self.__state_update
        weights = [N.require_cuda(lin.weight, "edge weight", torch.float32) for lin in self.__edge_message_transformation_layers]
        w_ih, w_hh = N.require_cuda(gru.weight_ih, "weight_ih", torch.float32), N.require_cuda(gru.weight_hh, "weight_hh", torch.float32)
        b_ih, b_hh = N.require_cuda(gru.bias_ih, "bias_ih", torch.float32), N.require_cuda(gru.bias_hh, "bias_hh", torch.float32)
        for i, w in enumerate(weights):
            _check_shape(w, (D, H), f"edge weight {i}")
        _check_shape(w_ih, (3 * H, D), "GRUCell.weight_ih"); _check_shape(w_hh, (3 * H, H), "GRUCell.weight_hh")
        _check_shape(b_ih, (3 * H,), "GRUCell.bias_ih"); _check_shape(b_hh, (3 * H,), "GRUCell.bias_hh")
        return weights, w_ih, w_hh, b_ih, b_hh

    def _forward_dropout(self, h: torch.Tensor, adjacency_lists, key: torch.Tensor, p: float) -> torch.Tensor:
        """Per-edge dropout (fp32 states, unsharded, no edge features) for the mask of ``key`` (int32 [2], device): on the fused kernel
        where it takes the dims, else on the three-kernel path."""
        if _use_fused(N.lib(), False, self.__state_dimension, self.__message_dimension):
            return self._forward_fused_dropout(h, adjacency_lists, key, p)
        return self._forward_unfused_dropout(h, adjacency_lists, key, p)

    def _forward_unfused_dropout(self, h: torch.Tensor, adjacency_lists, key: torch.Tensor, p: float) -> torch.Tensor:
        """The three-kernel path with per-edge dropout: the keep bits in cat(types) order, the masked tensor-core message kernel (the
        dropped elements of each gathered row are cleared before the products, which are scaled by 1 / (1 - p)), the segmented reduce
        and the GRUCell step.  The derived weights are those of the path without dropout, so the two share a weight-cache entry."""
        num_nodes, H = h.shape
        D = self.__message_dimension
        plan = self._plan(adjacency_lists, num_nodes)
        weights, w_ih, w_hh, b_ih, b_hh = self._dropout_params(H, D)
        lib = N.lib()
        cache, valid = self._weight_cache("f32", lib.ptgnn_b200_gated_weight_cache_bytes(0, plan.num_types, H, D),
                                          weights + [w_ih, w_hh, b_ih, b_hh], h.device)
        ws_bytes = lib.ptgnn_b200_gated_dropout_workspace_bytes(num_nodes, plan.num_edges, plan.num_types, H, D)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=h.device)
        out = torch.empty_like(h)
        N.call("ptgnn_b200_gated_forward_dropout", h.device, N.ptr(h), num_nodes, H, D, plan.num_types, plan.type_off_c, N.ptr(plan.row_ptr),
               N.ptr(plan.pos), N.ptr(plan.src32), N.ptr_table(weights), N.ptr(w_ih), N.ptr(w_hh), N.ptr(b_ih), N.ptr(b_hh),
               _reduce_code(self.__aggregation_fn), N.ptr(key), float(p), N.ptr(out), N.ptr(ws), ws_bytes, N.ptr(cache),
               0 if cache is None else cache.numel(), int(valid))
        self._weight_cache_filled("f32", h.device)
        return out

    def _forward_fused_dropout(self, h: torch.Tensor, adjacency_lists, key: torch.Tensor, p: float) -> torch.Tensor:
        """The fused path with per-edge dropout (fp32 states, unsharded, no edge features) for the mask of ``key`` (int32 [2], device):
        the keep bits are generated up front, the fused kernel clears the dropped features of the gathered rows, and 1 / (1 - p) is
        folded into the packed edge weights (a weight-cache entry of its own per p)."""
        num_nodes, H = h.shape
        D = self.__message_dimension
        plan = self._plan(adjacency_lists, num_nodes)
        weights, w_ih, w_hh, b_ih, b_hh = self._dropout_params(H, D)
        lib = N.lib()
        kind = ("f32_fused_dropout", float(p))
        cache, valid = self._weight_cache(kind, lib.ptgnn_b200_gated_fused_weight_cache_bytes(0, plan.num_types, H, D),
                                          weights + [w_ih, w_hh, b_ih, b_hh], h.device)
        ws_bytes = lib.ptgnn_b200_gated_fused_dropout_workspace_bytes(num_nodes, plan.num_edges, plan.num_types, H, D)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=h.device)
        out = torch.empty_like(h)
        bp = plan.block_plan(edge_ids=True)
        chain = current_state_chain()           # the packed states stay unmasked: the mask is applied to the gathered copies
        packed_in = chain.lookup(h) if chain is not None else None
        packed_out = None
        if chain is not None and chain.want_output:
            packed_out = torch.empty(max(lib.ptgnn_b200_packed_state_bytes(num_nodes, H), 1), dtype=torch.uint8, device=h.device)
        N.call("ptgnn_b200_gated_forward_fused_dropout", h.device, N.ptr(h), N.ptr(packed_in), num_nodes, plan.num_edges, H, D, plan.num_types,
               ctypes.byref(bp), N.ptr(plan.block_edge_ids), N.ptr(plan.row_ptr), N.ptr_table(weights), N.ptr(w_ih), N.ptr(w_hh), N.ptr(b_ih),
               N.ptr(b_hh), _reduce_code(self.__aggregation_fn), N.ptr(key), float(p), N.ptr(out), N.ptr(packed_out), N.ptr(ws), ws_bytes,
               N.ptr(cache), 0 if cache is None else cache.numel(), int(valid))
        self._weight_cache_filled(kind, h.device)
        if chain is not None:
            chain.store(out, packed_out)
        return out

    def _forward_with_edge_features(self, node_states, adjacency_lists, edge_features, gather_states, reduce: int) -> torch.Tensor:
        """F > 0 (gatedmessagepassing.py:59: ``cat([h_src, f_e])`` into the per-type Linear): composed from the stand-alone native
        pieces -- see ptgnn_b200/composed.py.  fp32 states only."""
        from . import composed as C

        if node_states.dtype != torch.float32:
            raise NotImplementedError("edge features with bf16 states have no native kernel")
        _check_states(node_states, self.__state_dimension, "GatedMessagePassingLayer")
        h = N.require_cuda(node_states, "node_states", torch.float32)
        gsrc = h if gather_states is None else N.require_cuda(gather_states, "gather_states", torch.float32)
        plan = self._plan(adjacency_lists, h.shape[0], None if gather_states is None else gsrc.shape[0])
        H, Fd = self.__state_dimension, self.__edge_feature_dimension
        weights = [lin.weight for lin in self.__edge_message_transformation_layers]
        for i, w in enumerate(weights):
            _check_shape(w, (self.__message_dimension, H + Fd), f"edge weight {i}")
        feats = C._edge_feature_list(edge_features, plan, Fd, h.device)
        msg = C.first_layer_messages(plan, gsrc, None, weights, [None] * plan.num_types, feats, H)
        agg = C.segment_reduce(msg, plan, reduce)
        return C.grucell(agg, h, self.__state_update)

    @property
    def input_state_dimension(self) -> int:
        return self.__state_dimension

    @property
    def output_state_dimension(self) -> int:
        return self.__state_dimension


class MLP(nn.Module):
    """Parameter container with the layout of the reference MLP (mlp.py:9-80): Sequential(Dropout, Linear,
    [activation, Dropout, Linear]...), bias-free by default, no final activation.  Only the zero-hidden-layer
    form (a single Linear) is executed natively, inside the edge-message kernel."""

    def __init__(
        self,
        input_dimension: int,
        output_dimension: int,
        hidden_layers: Union[List[int], int] = 1,
        use_biases: bool = False,
        activation: Optional[nn.Module] = nn.ReLU(),
        dropout_rate: float = 0.0,
    ):
        super().__init__()
        if isinstance(hidden_layers, int):
            width = 32 if output_dimension == 1 else output_dimension
            hidden_sizes = [width] * hidden_layers
        else:
            hidden_sizes = list(hidden_layers)
        assert len(hidden_sizes) <= 1 or activation is not None, "Multiple linear layers without an activation"
        sizes = hidden_sizes + [output_dimension]
        with_act: List[nn.Module] = []
        fan_in = input_dimension
        for i, size in enumerate(sizes):
            linear = nn.Linear(fan_in, size, bias=use_biases)
            nn.init.xavier_uniform_(linear.weight)
            with_act += [nn.Dropout(p=dropout_rate), linear]
            if i + 1 < len(sizes) and activation is not None:  # no activation after the output layer
                with_act.append(activation)
            fan_in = size
        self.__mlp_modules = nn.Sequential(*with_act)
        self.num_hidden_layers = len(hidden_sizes)
        self.uses_biases = use_biases

    @property
    def single_linear(self) -> nn.Linear:
        return self.__mlp_modules[1]

    @property
    def linears(self) -> List[nn.Linear]:
        return [m for m in self.__mlp_modules if isinstance(m, nn.Linear)]

    @property
    def activation(self) -> Optional[nn.Module]:
        acts = [m for m in self.__mlp_modules if not isinstance(m, (nn.Linear, nn.Dropout))]
        return acts[0] if acts else None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """mlp.py:79-80 on the native dense kernel (one launch per Linear, bias + activation fused); eval-mode dropout = identity.
        Inside MlpMessagePassingLayer the zero-hidden-layer form never runs as a module: it is the fused kernel's per-type weight."""
        from . import composed as C

        if self.training and any(isinstance(m, nn.Dropout) and m.p > 0 for m in self.__mlp_modules):
            raise NotImplementedError("training-mode dropout has no native kernel (forward-only)")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("ptgnn_b200.MLP is forward-only: call it under torch.no_grad()")
        lead = x.shape[:-1]
        y = x.reshape(-1, x.shape[-1]).to(torch.float32)
        lin = self.linears
        for i, layer in enumerate(lin):
            y = C.linear(y, layer.weight, layer.bias, self.activation if i + 1 < len(lin) else None)
        return y.reshape(*lead, y.shape[-1]).to(x.dtype)


class MlpMessagePassingLayer(AbstractMessagePassingLayer):
    """m_e = MLP_t([h_src ; h_tgt]);  a_v = reduce m_e;  h'_v = Dropout(act(W LN(GELU(a_v)) + b))."""

    def __init__(
        self,
        input_state_dimension: int,
        output_state_dimension: int,
        message_dimension: int,
        num_edge_types: int,
        message_aggregation_function: Union[str, AbstractMessageAggregation],
        message_activation: Optional[nn.Module] = nn.GELU(),
        use_target_state_as_message_input: bool = True,
        mlp_hidden_layers: Union[List[int], int] = 0,
        use_layer_norm: bool = True,
        use_dense_layer: bool = True,
        dropout_rate: float = 0.0,
        dense_activation: Optional[nn.Module] = nn.Tanh(),
        features_dimension: int = 0,
    ):
        super().__init__()
        self.__input_state_dim = input_state_dimension
        self.__use_target_state_as_message_input = use_target_state_as_message_input
        self.__output_state_dim = output_state_dimension
        self.__message_dim = message_dimension
        self.__features_dim = features_dimension
        message_input = (2 if use_target_state_as_message_input else 1) * input_state_dimension
        self.__edge_message_transformation_layers = nn.ModuleList(
            MLP(input_dimension=message_input + features_dimension, output_dimension=message_dimension,
                hidden_layers=mlp_hidden_layers)
            for _ in range(num_edge_types)
        )
        self.__aggregation_fn = message_aggregation_function
        if isinstance(message_aggregation_function, str):
            aggregated_size = message_dimension
        else:
            aggregated_size = message_aggregation_function.output_state_size(message_dimension)
        self.__aggregated_size = aggregated_size
        self.__message_activation = message_activation

        update: List[nn.Module] = []
        if use_layer_norm:
            update.append(nn.LayerNorm(aggregated_size))
        if use_dense_layer:
            update.append(nn.Linear(aggregated_size, output_state_dimension))
            nn.init.xavier_uniform_(update[-1].weight)
            if dense_activation is not None:
                update.append(dense_activation)
        update.append(nn.Dropout(p=dropout_rate))
        self.__state_update = nn.Sequential(*update)

    def forward(
        self,
        node_states: torch.Tensor,
        adjacency_lists: List[Tuple[torch.Tensor, torch.Tensor]],
        node_to_graph_idx: torch.Tensor = None,
        reference_node_ids: Dict[str, torch.Tensor] = None,
        reference_node_graph_idx: Dict[str, torch.Tensor] = None,
        edge_features: List[torch.Tensor] = None,
        gather_states: Optional[torch.Tensor] = None,
    ) -> torch.Tensor:
        mlps = self.__edge_message_transformation_layers
        assert len(adjacency_lists) == len(mlps), "The number of adjacency lists must be equal to the number of edge types."
        from . import autograd as _ag
        from .aggregation import PnaMessageAggregation

        plain_mlp = self.__features_dim == 0 and not any(m.num_hidden_layers != 0 or m.uses_biases for m in mlps)
        default_config = plain_mlp and isinstance(self.__aggregation_fn, str)
        # the native PNA aggregator after a default message MLP: messages from the native message kernel, then the PNA kernel
        # (composed path without gradients, _MlpLayerFunction's PNA mode with them)
        pna_config = plain_mlp and isinstance(self.__aggregation_fn, PnaMessageAggregation)
        grad = _ag.needs_grad(self, node_states)
        bf16_grad = default_config and node_states.dtype == torch.bfloat16 and _mlp_bf16_grad_supported(
            N.lib(), self.__input_state_dim, self.__message_dim, self.__use_target_state_as_message_input)
        if grad and (not (default_config or pna_config) or gather_states is not None or (node_states.dtype != torch.float32 and not bf16_grad)):
            _refuse_autograd(self, node_states)
        if not (default_config or pna_config):
            return self._forward_composed(node_states, adjacency_lists, edge_features, gather_states)
        _check_no_edge_features(edge_features)

        ln: Optional[nn.LayerNorm] = None
        dense: Optional[nn.Linear] = None
        dense_act_module: Optional[nn.Module] = None
        drop_p = 0.0
        for m in self.__state_update:
            if isinstance(m, nn.LayerNorm):
                ln = m
            elif isinstance(m, nn.Linear):
                dense = m
            elif isinstance(m, nn.Dropout):
                drop_p = m.p if self.training else 0.0
            else:
                dense_act_module = m
        # the trailing nn.Dropout of the state update (mlpmessagepassing.py:65) acts on the layer's [N, H_out] output: a torch op on the
        # result (differentiable), never inside the kernels; suppressed when an autograd.Function re-enters the layer
        if drop_p > 0 and not _ag.output_dropout_suppressed():
            apply_dropout = lambda t: torch.nn.functional.dropout(t, drop_p, True)  # noqa: E731
        else:
            apply_dropout = lambda t: t  # noqa: E731
        if grad:   # backward (SURVEY.md §8 f-1): the forward below runs unchanged under no_grad inside the Function
            _check_states(node_states, self.__input_state_dim, "MlpMessagePassingLayer")
            return apply_dropout(_ag.mlp_forward_with_grad(
                self, node_states, adjacency_lists, self.__aggregation_fn, self.__use_target_state_as_message_input,
                self.__message_activation, ln, dense, dense_act_module, [m.single_linear.weight for m in mlps]))
        if pna_config:
            return apply_dropout(self._forward_composed(node_states, adjacency_lists, edge_features, gather_states, dropout_by_caller=True))
        reduce = _reduce_code(self.__aggregation_fn)
        msg_act = _activation_code(self.__message_activation, "message_activation")
        dense_act = N.ACT_NONE if dense_act_module is None else _activation_code(dense_act_module, "dense_activation")

        state_dtype = node_states.dtype if node_states.dtype == torch.bfloat16 else torch.float32
        _check_states(node_states, self.__input_state_dim, "MlpMessagePassingLayer")
        h = N.require_cuda(node_states, "node_states", state_dtype)
        num_nodes, H = h.shape
        D = self.__message_dim
        out_dim = dense.out_features if dense is not None else D
        gsrc = self._gather_source(gather_states, h)
        plan = self._plan(adjacency_lists, num_nodes, None if gsrc is None else gsrc.shape[0])
        weights = [N.require_cuda(m.single_linear.weight, "edge weight", torch.float32) for m in mlps]
        f32 = lambda t, n: None if t is None else N.require_cuda(t, n, torch.float32)  # noqa: E731
        ln_w, ln_b = (f32(ln.weight, "ln.weight"), f32(ln.bias, "ln.bias")) if ln is not None else (None, None)
        d_w = f32(dense.weight, "dense.weight") if dense is not None else None
        d_b = f32(dense.bias, "dense.bias") if dense is not None and dense.bias is not None else None
        ut_i = int(self.__use_target_state_as_message_input)
        for i, w in enumerate(weights):
            _check_shape(w, (D, (1 + ut_i) * H), f"edge weight {i}")
        if ln_w is not None:
            _check_shape(ln_w, (D,), "LayerNorm.weight"); _check_shape(ln_b, (D,), "LayerNorm.bias")
        if d_w is not None:
            _check_shape(d_w, (out_dim, D), "dense.weight")

        lib = N.lib()
        bf16 = state_dtype == torch.bfloat16
        if plan.num_edges > 0 and _use_fused(lib, bf16, H, D):
            ns = num_nodes if gsrc is None else gsrc.shape[0]
            ws_bytes = lib.ptgnn_b200_mlp_fused_workspace_bytes(int(bf16), num_nodes, ns, plan.num_types, H, D, out_dim, ut_i)
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=h.device)
            out = torch.empty(num_nodes, out_dim, dtype=state_dtype, device=h.device)
            bp = plan.block_plan()
            # derived copies of the edge weights (fp16 hi | lo' in the kernel's packed order) and of the dense weight (TF32 hi / lo): once
            # per parameter version, like the gated layer's (fp32 path; the bf16 path converts per call)
            cache_params = weights + ([d_w] if d_w is not None else [])
            cache, valid = self._weight_cache("mlp_f32_fused", 0 if bf16 else lib.ptgnn_b200_mlp_fused_weight_cache_bytes(
                0, plan.num_types, H, D, out_dim, ut_i), cache_params, h.device)
            N.call("ptgnn_b200_mlp_forward_fused", h.device, int(bf16), N.ptr(h), N.ptr(gsrc), num_nodes, ns, H, D, out_dim, plan.num_types,
                   ctypes.byref(bp), N.ptr(plan.row_ptr), N.ptr_table(weights), ut_i, reduce, msg_act, N.ptr(ln_w), N.ptr(ln_b),
                   float(ln.eps) if ln is not None else 0.0, N.ptr(d_w), N.ptr(d_b), dense_act, N.ptr(out), N.ptr(ws), ws_bytes,
                   N.ptr(cache), 0 if cache is None else cache.numel(), int(valid))
            self._weight_cache_filled("mlp_f32_fused", h.device)
            return apply_dropout(out)
        # round-1 three-kernel path; bf16 states: fp32 parameters (converted inside the library), fp32 accumulation
        ws_bytes = lib.ptgnn_b200_mlp_workspace_bytes(int(bf16), num_nodes, plan.num_edges, plan.num_types, H, D, out_dim, ut_i)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=h.device)
        out = torch.empty(num_nodes, out_dim, dtype=state_dtype, device=h.device)
        N.call("ptgnn_b200_mlp_forward", h.device, int(bf16), N.ptr(h), N.ptr(gsrc), num_nodes, H, D, out_dim, plan.num_types, plan.type_off_c,
               N.ptr(plan.row_ptr), N.ptr(plan.pos), N.ptr(plan.src32), N.ptr(plan.tgt32), N.ptr_table(weights), ut_i, reduce, msg_act,
               N.ptr(ln_w), N.ptr(ln_b), float(ln.eps) if ln is not None else 0.0, N.ptr(d_w), N.ptr(d_b), dense_act, N.ptr(out), N.ptr(ws),
               ws_bytes)
        return apply_dropout(out)

    def _forward_composed(self, node_states, adjacency_lists, edge_features, gather_states, dropout_by_caller: bool = False) -> torch.Tensor:
        """Module aggregators (PNA ...), message MLPs with hidden layers / biases, edge features (mlpmessagepassing.py:82-117 in
        full generality): stand-alone native pieces + the module's own tail -- see ptgnn_b200/composed.py.  fp32 states only.
        The native PnaMessageAggregation runs on the layer's own plan.  ``dropout_by_caller``: the caller applies the tail's output
        Dropout to the result (a torch op, as in the default configuration), so it is left out here; otherwise training-mode dropout
        with p > 0 is refused."""
        from . import composed as C
        from .aggregation import PnaMessageAggregation, pna

        native_pna = isinstance(self.__aggregation_fn, PnaMessageAggregation)
        if node_states.dtype != torch.float32:
            raise NotImplementedError("this MlpMessagePassingLayer configuration has no bf16 kernel")
        _check_states(node_states, self.__input_state_dim, "MlpMessagePassingLayer")
        for m in self.__state_update:
            if isinstance(m, nn.Dropout) and self.training and m.p > 0 and not dropout_by_caller:
                raise NotImplementedError("training-mode dropout has no native kernel (forward-only)")
        h = N.require_cuda(node_states, "node_states", torch.float32)
        gsrc = h if gather_states is None else N.require_cuda(gather_states, "gather_states", torch.float32)
        plan = self._plan(adjacency_lists, h.shape[0], None if gather_states is None else gsrc.shape[0])
        mlps = list(self.__edge_message_transformation_layers)
        ut = self.__use_target_state_as_message_input
        state_cols = (2 if ut else 1) * self.__input_state_dim
        feats = C._edge_feature_list(edge_features, plan, self.__features_dim, h.device)
        firsts = [m.linears[0] for m in mlps]
        for i, lin in enumerate(firsts):
            _check_shape(lin.weight, (lin.out_features, state_cols + self.__features_dim), f"message MLP {i} first layer")
        msg = C.first_layer_messages(plan, gsrc, h if ut else None, [l.weight for l in firsts], [l.bias for l in firsts], feats, state_cols)
        depth = len(mlps[0].linears)
        for k in range(1, depth):                       # hidden layers: activation, then one dense GEMM per edge type
            act = mlps[0].activation
            msg = act(msg) if act is not None else msg
            nxt = torch.empty(plan.num_edges, mlps[0].linears[k].out_features, dtype=torch.float32, device=h.device)
            for t, m in enumerate(mlps):
                lo, hi = plan.type_off[t], plan.type_off[t + 1]
                if hi > lo:
                    nxt[lo:hi] = C.linear(msg[lo:hi], m.linears[k].weight, m.linears[k].bias)
            msg = nxt
        if isinstance(self.__aggregation_fn, str):
            agg = C.segment_reduce(msg, plan, _reduce_code(self.__aggregation_fn))
        elif native_pna:    # the messages are in edge order: the layer's plan groups them by target
            agg = pna(msg, plan, self.__aggregation_fn.delta)
        else:   # e.g. the reference's PnaMessageAggregation: messages + concatenated targets, as mlpmessagepassing.py:100-112 passes them
            agg = self.__aggregation_fn(msg, plan.tgt32.to(torch.int64), h.shape[0])
        if self.__message_activation is not None:
            agg = self.__message_activation(agg)
        return self.__state_update[:-1](agg) if dropout_by_caller else self.__state_update(agg)

    @property
    def input_state_dimension(self) -> int:
        return self.__input_state_dim

    @property
    def output_state_dimension(self) -> int:
        return self.__output_state_dim
