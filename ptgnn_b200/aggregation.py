"""Module aggregators for ``MlpMessagePassingLayer(message_aggregation_function=<module>)``.

``PnaMessageAggregation``: Principal Neighbourhood Aggregation (https://arxiv.org/abs/2004.05718) with the reference's conventions
(`/root/reference/ptgnn/neuralmodels/gnn/messagepassing/pna_aggregation.py:13-59`): per target the sum, mean (sum / (degree + 1e-5)),
max, min and a std built from ``relu(m^2 - mean[target]^2) + 1e-10``, concatenated and repeated under the three degree scalers
(identity, ``log(degree + 1) / delta``, its damped inverse) -> ``15 x message_dim`` features.  One native kernel computes all of it
(``ptgnn_b200_pna_forward``, DESIGN.md §3.10) over the target-sorted plan of the message targets; gradients (fp32 messages) come from
``ptgnn_b200_pna_backward_f32`` through ``autograd._PnaFn``.

* Messages: fp32, or bf16 (statistics in fp32, rounded to bf16 before the scalers as the reference's ``.to(msg_dtype)`` does; the
  output is fp32 in both cases, as the reference's ``torch.cat`` promotes it).
* Not supported (``NotImplementedError``): other message dtypes, gradients with bf16 messages, and message widths other than a multiple
  of 4 in [4, 512].
"""
from typing import Optional, Tuple

import torch

from . import _native as N
from .edgeplan import EdgePlan, plan_for
from .messagepassing import AbstractMessageAggregation

_DIMS = "a message dimension that is a multiple of 4 in [4, 512]"


def _messages(messages: torch.Tensor, plan: EdgePlan) -> Tuple[torch.Tensor, bool]:
    """The messages as an aligned contiguous CUDA tensor, and whether they are bf16; checks them against the plan."""
    if messages.dtype not in (torch.float32, torch.bfloat16):
        raise NotImplementedError(f"the PNA kernel takes fp32 or bf16 messages, got {messages.dtype}")
    if messages.dim() != 2 or messages.shape[0] != plan.num_edges:
        raise ValueError(f"messages must be [{plan.num_edges}, D], got {tuple(messages.shape)}")
    if not N.lib().ptgnn_b200_pna_supported(messages.shape[1]):
        raise NotImplementedError(f"the PNA kernel takes {_DIMS}, got D={messages.shape[1]}")
    m = N.require_cuda(messages, "messages", messages.dtype)
    return (m if m.data_ptr() % 16 == 0 else m.clone()), messages.dtype == torch.bfloat16


def native_pna(messages: torch.Tensor, plan: EdgePlan, delta: float, want_arg: bool = False
               ) -> Tuple[torch.Tensor, Optional[torch.Tensor], Optional[torch.Tensor]]:
    """``ptgnn_b200_pna_forward``: (out [N, 15 D] fp32, arg_max, arg_min) for messages [E, D] (fp32 or bf16, edge order) and the plan
    of their targets.  ``want_arg``: also the [N, D] int32 winning edge ids of max and min (E for an empty target), else None."""
    m, bf16 = _messages(messages, plan)
    n, D = plan.num_nodes, m.shape[1]
    out = torch.empty(n, 15 * D, dtype=torch.float32, device=m.device)
    args = torch.empty(2, n, D, dtype=torch.int32, device=m.device) if want_arg else None
    with torch.cuda.device(m.device):
        rc = N.lib().ptgnn_b200_pna_forward(int(bf16), N.ptr(m), plan.num_edges, D, N.ptr(plan.row_ptr),
                                            N.ptr(plan.perm) if plan.num_edges else None, n, float(delta), N.ptr(out),
                                            N.ptr(args[0]) if want_arg else None, N.ptr(args[1]) if want_arg else None,
                                            N.current_stream(m.device))
    N.check(rc, "ptgnn_b200_pna_forward")
    return (out, args[0], args[1]) if want_arg else (out, None, None)


def native_pna_backward(messages: torch.Tensor, plan: EdgePlan, delta: float, out: torch.Tensor, arg_max: torch.Tensor,
                        arg_min: torch.Tensor, d_out: torch.Tensor) -> torch.Tensor:
    """``ptgnn_b200_pna_backward_f32``: d messages [E, D] from d out [N, 15 D] and the forward's fp32 messages, output and arg ids."""
    m, bf16 = _messages(messages, plan)
    if bf16:
        raise NotImplementedError("PNA gradients take fp32 messages")
    n, D = plan.num_nodes, m.shape[1]
    tensors = []
    for t, name, dtype, shape in ((out, "out", torch.float32, (n, 15 * D)), (d_out, "d_out", torch.float32, (n, 15 * D)),
                                  (arg_max, "arg_max", torch.int32, (n, D)), (arg_min, "arg_min", torch.int32, (n, D))):
        t = N.require_cuda(t, name, dtype)
        if tuple(t.shape) != shape:
            raise ValueError(f"{name} must have shape {shape}, got {tuple(t.shape)}")
        tensors.append(t if t.data_ptr() % 16 == 0 else t.clone())
    out, d_out, arg_max, arg_min = tensors
    d_m = torch.empty_like(m)
    with torch.cuda.device(m.device):
        rc = N.lib().ptgnn_b200_pna_backward_f32(N.ptr(m), plan.num_edges, D, N.ptr(plan.row_ptr), N.ptr(plan.perm) if plan.num_edges else None,
                                                 n, float(delta), N.ptr(out), N.ptr(arg_max), N.ptr(arg_min), N.ptr(d_out), N.ptr(d_m),
                                                 N.current_stream(m.device))
    N.check(rc, "ptgnn_b200_pna_backward_f32")
    return d_m


def pna(messages: torch.Tensor, plan: EdgePlan, delta: float) -> torch.Tensor:
    """The aggregation over a given plan: differentiable (``autograd._PnaFn``) when the messages require gradients."""
    if torch.is_grad_enabled() and messages.requires_grad:
        from . import autograd as _ag

        if messages.dtype != torch.float32:
            raise NotImplementedError(f"PNA gradients take fp32 messages, got {messages.dtype}")
        return _ag.pna_with_grad(plan, delta, messages)
    return native_pna(messages.detach(), plan, delta)[0]


class PnaMessageAggregation(AbstractMessageAggregation):
    def __init__(self, delta: float = 1):
        super().__init__()
        self._delta = delta

    @property
    def delta(self) -> float:
        return self._delta

    def forward(self, messages: torch.Tensor, message_targets: torch.Tensor, num_nodes):
        """messages [E, D] (edge order), message_targets [E] int64, num_nodes the target count -> [num_nodes, 15 D] fp32.  The plan of
        the targets comes from ``plan_for`` (cached by tensor identity and version); targets outside [0, num_nodes) raise IndexError
        when its status is polled."""
        targets = N.require_cuda(message_targets, "message_targets", torch.int64)
        if targets.dim() != 1 or messages.dim() != 2 or targets.shape[0] != messages.shape[0]:
            raise ValueError(f"messages [E, D] and message_targets [E] expected, got {tuple(messages.shape)} and {tuple(targets.shape)}")
        plan = plan_for([(targets, targets)], int(num_nodes))
        out = pna(messages, plan, self._delta)
        plan.poll()
        return out

    def output_state_size(self, message_input_size: int) -> int:
        return message_input_size * 5 * 3
