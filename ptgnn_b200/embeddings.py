"""``TokenUnitEmbedder`` and ``SubtokenUnitEmbedder`` with the reference's ``nn.Module`` API, on the native embedding-bag kernels.

Counterpart of `ptgnn/neuralmodels/embeddings/strelementrepresentationmodel.py:16-89` of the reference -- the node embedder that
``GraphNeuralNetwork.forward`` calls before its layer loop.  The reference materialises ``embedded [B, S, D]``, a mask, their product
and the reduction over the S subtoken slots; here ``ptgnn_b200_embedding_bag`` (DESIGN.md §3.12) reads the int64 ids once, adds the
valid slots of a row in slot order in registers and writes the ``[B, D]`` result once.

* Dense output layer (``use_dense_output``): sum and mean are linear, so ``pool(table[ids]) W^T = pool((table W^T)[ids])``.  When the
  vocabulary has no more rows than the minibatch (V <= B) the *table* is transformed with the native ``linear`` operator and the
  bag kernel runs over the transformed table; otherwise, and always for ``"max"``, the rows are pooled first and ``linear`` is applied
  to the ``[B, D]`` result.  The choice depends on V, B and the combination kind only.  In eval mode, when no gradient is asked
  for, the transformed table is kept per parameter version and dropped by ``.to()`` / ``_apply``.
* Gradients (fp32): ``autograd._EmbeddingBagFn`` around the kernels (saves the ids, the lengths and, for max, the ``[B, D]`` uint8
  winning slots); the table gradient is a sorted, atomic-free reduction (the edge plan of the (row, token) pairs and the per-graph
  chunk walk).  The dense layer is the differentiable native ``_LinearFn`` on whichever side of the bag it ran.
* bf16: under ``torch.autocast("cuda", dtype=torch.bfloat16)`` the reference's ``Linear`` returns bf16, so ``SubtokenUnitEmbedder``
  with a dense output returns bf16 rows (accumulated in fp32, rounded once).  ``TokenUnitEmbedder`` returns fp32, as the reference does.
* An id outside ``[0, V)`` is read as row 0 and counted in a pinned status word that every call polls without synchronising: the
  ``IndexError`` is raised by the first call after the kernel ran.  Nothing in the forward synchronises, so it can be captured.

Not supported (``NotImplementedError``): D > 512, more than 64 slots, gradients with a bf16 output, a dense output with D not a
multiple of 4 (the native ``linear`` operator), and ``CharUnitEmbedder`` (stays the reference's).
"""
import math
from typing import Optional, Tuple

import torch
from torch import nn

from . import _native as N
from .edgeplan import EdgePlan

_LIMITS = "an embedding size in [1, 512] and 1 to 64 subtoken slots"


def _aligned(t: torch.Tensor, what: str, dtype: torch.dtype) -> torch.Tensor:
    """A contiguous CUDA tensor of ``dtype`` whose data starts on a 16-byte boundary (the kernels load four columns at once)."""
    t = N.require_cuda(t, what, dtype)
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _bag_args(ids: torch.Tensor, lengths: Optional[torch.Tensor], D: int, mode: str) -> Tuple[torch.Tensor, Optional[torch.Tensor], int, int]:
    if mode not in N.POOL:
        raise ValueError(f'Unrecognized subtoken combination "{mode}".')
    ids = N.require_cuda(ids, "token_idxs", torch.int64)
    if ids.dim() == 1:
        ids = ids.unsqueeze(1)
    if ids.dim() != 2:
        raise ValueError(f"token_idxs must be [B] or [B, S], got {tuple(ids.shape)}")
    B, S = ids.shape
    if not N.lib().ptgnn_b200_embedding_bag_supported(D, max(S, 1)):
        raise NotImplementedError(f"the embedding-bag kernels take {_LIMITS}, got D={D}, S={S}")
    if lengths is not None:
        lengths = N.require_cuda(lengths, "lengths", torch.int64)
        if tuple(lengths.shape) != (B,):
            raise ValueError(f"lengths must be [{B}], got {tuple(lengths.shape)}")
    return ids, lengths, B, S


def new_status() -> torch.Tensor:
    """A pinned int32 word for the kernels' count of out-of-range ids (polled by the host without synchronising)."""
    return torch.zeros(1, dtype=torch.int32).pin_memory()


def poll_status(status: torch.Tensor, vocab: int) -> None:
    bad = int(status[0])
    if bad:
        status[0] = 0
        raise IndexError(f"{bad} token ids outside [0, {vocab}); the kernel read row 0 for them, results are not valid")


def native_embedding_bag(table: torch.Tensor, ids: torch.Tensor, lengths: Optional[torch.Tensor], mode: str,
                         out_dtype: torch.dtype = torch.float32, want_arg: bool = False, status: Optional[torch.Tensor] = None,
                         out: Optional[torch.Tensor] = None):
    """``ptgnn_b200_embedding_bag``: out [B, D] (fp32 or bf16) = pool over the valid slots of table [V, D] fp32 rows, ids [B, S] (or
    [B]) int64, lengths [B] int64 or None (every slot valid).  ``want_arg`` (max): also the [B, D] uint8 winning slots.  ``status``: a
    ``new_status()`` word that receives the number of out-of-range ids.  ``out``: an aligned contiguous [B, D] tensor to write."""
    table = _aligned(table, "embedding table", torch.float32)
    if table.dim() != 2:
        raise ValueError(f"the embedding table must be [V, D], got {tuple(table.shape)}")
    V, D = table.shape
    ids, lengths, B, S = _bag_args(ids, lengths, D, mode)
    if out_dtype not in (torch.float32, torch.bfloat16):
        raise TypeError(f"out_dtype must be float32 or bfloat16, got {out_dtype}")
    if out is None:
        out = torch.empty(B, D, dtype=out_dtype, device=table.device)
    elif out.dtype != out_dtype or tuple(out.shape) != (B, D) or not out.is_contiguous() or out.data_ptr() % 16 != 0:
        raise ValueError(f"out must be an aligned contiguous {(B, D)} {out_dtype} tensor")
    arg = torch.empty(B, D, dtype=torch.uint8, device=table.device) if want_arg and mode == "max" else None
    if B and S:
        with torch.cuda.device(table.device):
            rc = N.lib().ptgnn_b200_embedding_bag(int(out_dtype == torch.bfloat16), N.ptr(table), V, D, N.ptr(ids), N.ptr(lengths), B, S,
                                                  N.POOL[mode], N.ptr(out), N.ptr(arg), N.ptr(status), N.current_stream(table.device))
        N.check(rc, "ptgnn_b200_embedding_bag")
    elif B:
        out.fill_(-math.inf if mode == "max" else 0.0)
    return (out, arg) if want_arg else out


def occurrence_plan(ids: torch.Tensor, lengths: Optional[torch.Tensor], vocab: int) -> EdgePlan:
    """The edge plan of the (row -> token id) pairs of ids [B, S]: its rows are the vocabulary (row ``vocab`` is the sink of the
    padding slots), and its stable order lists a token's occurrences by (row, slot)."""
    B, S = ids.shape
    dev = ids.device
    src, tgt = torch.empty(B * S, dtype=torch.int64, device=dev), torch.empty(B * S, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        rc = N.lib().ptgnn_b200_embedding_bag_pairs(N.ptr(ids), N.ptr(lengths), B, S, vocab, N.ptr(src), N.ptr(tgt), N.current_stream(dev))
    N.check(rc, "ptgnn_b200_embedding_bag_pairs")
    plan = EdgePlan([(src, tgt)], vocab + 1, num_source_nodes=B)
    plan.perm                           # the sorted arrays are built on first access
    return plan


def native_embedding_bag_backward(d_out: torch.Tensor, ids: torch.Tensor, lengths: Optional[torch.Tensor], mode: str, vocab: int,
                                  arg: Optional[torch.Tensor] = None, plan: Optional[EdgePlan] = None) -> torch.Tensor:
    """``ptgnn_b200_embedding_bag_backward_f32``: d table [V, D] from d out [B, D] fp32.  The valid (row, slot) pairs are grouped by
    token id with the edge plan (row V is the sink of the padding slots) and every token's occurrences are added in (row, slot) order
    in chunks: no float atomics, every row written once.  ``plan``: an ``occurrence_plan`` of the same ids and lengths, else built here."""
    d_out = _aligned(d_out, "d_out", torch.float32)
    D = d_out.shape[1]
    ids, lengths, B, S = _bag_args(ids, lengths, D, mode)
    if d_out.shape[0] != B:
        raise ValueError(f"d_out must be [{B}, {D}], got {tuple(d_out.shape)}")
    if mode == "max":
        if arg is None:
            raise ValueError("max needs the forward's arg slots")
        arg = N.require_cuda(arg, "arg", torch.uint8)
    dev = d_out.device
    d_table = torch.empty(vocab, D, dtype=torch.float32, device=dev)
    if B == 0 or S == 0:
        return d_table.zero_()
    lib = N.lib()
    if plan is None:
        plan = occurrence_plan(ids, lengths, vocab)
    elif plan.num_nodes != vocab + 1 or plan.num_edges != B * S:
        raise ValueError("plan does not belong to these ids")
    ws_bytes = lib.ptgnn_b200_embedding_bag_backward_workspace_bytes(B, S, vocab, D)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = lib.ptgnn_b200_embedding_bag_backward_f32(N.ptr(d_out), B, S, D, N.ptr(lengths), N.ptr(arg), N.POOL[mode], N.ptr(plan.row_ptr),
                                                       N.ptr(plan.perm), vocab, N.ptr(d_table), N.ptr(ws), ws_bytes, N.current_stream(dev))
    N.check(rc, "ptgnn_b200_embedding_bag_backward_f32")
    return d_table


def _bf16_autocast(device: torch.device) -> bool:
    return device.type == "cuda" and torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16


def _wants_grad(*params: Optional[torch.Tensor]) -> bool:
    return torch.is_grad_enabled() and any(p is not None and p.requires_grad for p in params)


def _bag(table: torch.Tensor, ids, lengths, mode: str, out_dtype: torch.dtype, status: torch.Tensor) -> torch.Tensor:
    """The bag over ``table``: under autograd when the table needs a gradient."""
    if _wants_grad(table):
        from . import autograd as _ag

        return _ag.embedding_bag_with_grad(table, ids, lengths, mode, status)
    return native_embedding_bag(table.detach(), ids, lengths, mode, out_dtype, status=status)


def _linear(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    from . import autograd as _ag
    from . import composed as C

    if _wants_grad(x, weight):
        return _ag._LinearFn.apply(x, weight, None)
    return C.linear(x.detach(), weight.detach())


class _NativeEmbedder(nn.Module):
    """What both embedders keep besides their parameters: the pinned status word (``_status``) and, for the dense output layer, the
    transformed table of eval mode (``_transformed``).  Both are scratch tied to this process and placement: they are not pickled or
    deep-copied (the reference saves a model by pickling the whole module, abstractneuralmodel.py:155-163, and a restored tensor
    attribute would be pageable or device memory, not the pinned word the kernel and the synchronisation-free poll need)."""

    def __init__(self):
        super().__init__()
        self._status: Optional[torch.Tensor] = None
        self._transformed = None        # eval mode: (key, table W^T)

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_transformed"] = state["_status"] = None
        return state

    def _apply(self, fn, *args, **kwargs):
        self._transformed = None        # .to() / .cuda() / .float(): the table derived for the old placement is dead
        out = super()._apply(fn, *args, **kwargs)
        # the word is pinned when the module reaches the GPU, so that a first forward inside a CUDA-graph capture allocates nothing
        # on the host
        if self._status is None and any(p.is_cuda for p in self.parameters()):
            self._status = new_status()
        return out

    def _status_word(self) -> torch.Tensor:
        if self._status is None:        # built on the GPU directly, or restored from a pickle
            self._status = new_status()
        return self._status


class TokenUnitEmbedder(_NativeEmbedder):
    def __init__(self, vocabulary_size: int, embedding_size: int, dropout_rate: float):
        super().__init__()
        self.__embeddings = nn.Embedding(num_embeddings=vocabulary_size, embedding_dim=embedding_size)
        nn.init.xavier_uniform_(self.__embeddings.weight)
        self.__dropout_layer = nn.Dropout(p=dropout_rate)

    @property
    def embedding_layer(self) -> nn.Embedding:
        return self.__embeddings

    def forward(self, token_idxs: torch.Tensor) -> torch.Tensor:
        """token_idxs [B] int64 -> [B, D] fp32."""
        table = self.__embeddings.weight
        N.require_cuda(table, "embedding table", torch.float32)
        if token_idxs.dim() != 1:
            raise ValueError(f"token_idxs must be [B], got {tuple(token_idxs.shape)}")
        status = self._status_word()
        poll_status(status, table.shape[0])
        out = _bag(table, token_idxs, None, "sum", torch.float32, status)
        poll_status(status, table.shape[0])
        return self.__dropout_layer(out)


class SubtokenUnitEmbedder(_NativeEmbedder):
    def __init__(self, vocabulary_size: int, embedding_size: int, dropout_rate: float, subtoken_combination_kind: str,
                 use_dense_output: bool = True):
        super().__init__()
        assert subtoken_combination_kind in {"mean", "max", "sum"}
        self.__subtoken_combination_kind = subtoken_combination_kind
        self.__embeddings = nn.Embedding(num_embeddings=vocabulary_size, embedding_dim=embedding_size)
        nn.init.uniform_(self.__embeddings.weight)
        if use_dense_output:
            self.__out_layer = nn.Linear(embedding_size, embedding_size, bias=False)
            nn.init.xavier_uniform_(self.__out_layer.weight)
        else:
            self.__out_layer = None
        self.__dropout_layer = nn.Dropout(p=dropout_rate)

    @property
    def embedding_layer(self) -> nn.Embedding:
        return self.__embeddings

    def _transformed_table(self, table: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
        """table W^T [V, D].  Kept in eval mode while neither parameter was modified in place, re-assigned or moved (in training mode
        edits through ``.data`` are common and do not move the version counter: it is derived on every call)."""
        if self.training or _wants_grad(table, weight):
            return _linear(table, weight)
        key = tuple((p.data_ptr(), p._version, p.device, p.dtype) for p in (table, weight))
        if self._transformed is None or self._transformed[0] != key:
            self._transformed = (key, _linear(table, weight))
        return self._transformed[1]

    def forward(self, token_idxs: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
        """
        :param token_idxs: The subtoken ids in a [B, max_num_subtokens] matrix.
        :param lengths: A [B]-sized vector containing the lengths
        :return: a [B, D] matrix of D-sized representations, one per input example.
        """
        kind = self.__subtoken_combination_kind
        table = self.__embeddings.weight
        weight = None if self.__out_layer is None else self.__out_layer.weight
        N.require_cuda(table, "embedding table", torch.float32)
        if token_idxs.dim() != 2:
            raise ValueError(f"token_idxs must be [B, max_num_subtokens], got {tuple(token_idxs.shape)}")
        V, D = table.shape
        B = token_idxs.shape[0]
        bf16 = weight is not None and _bf16_autocast(table.device)
        if bf16 and _wants_grad(table, weight):
            raise NotImplementedError("SubtokenUnitEmbedder: gradients with a bf16 output have no native kernel; train in fp32")
        if weight is not None and D % 4 != 0:
            raise NotImplementedError(f"SubtokenUnitEmbedder: the native linear operator takes dimensions that are multiples of 4, got D={D}; "
                                      "use use_dense_output=False")
        out_dtype = torch.bfloat16 if bf16 else torch.float32
        status = self._status_word()
        poll_status(status, V)
        if weight is None:
            out = _bag(table, token_idxs, lengths, kind, out_dtype, status)
        elif kind != "max" and V <= B:
            out = _bag(self._transformed_table(table, weight), token_idxs, lengths, kind, out_dtype, status)
        else:
            out = _linear(_bag(table, token_idxs, lengths, kind, torch.float32, status), weight).to(out_dtype)
        poll_status(status, V)
        return self.__dropout_layer(out)
