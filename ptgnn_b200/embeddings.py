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

Not supported (``NotImplementedError``): D > 512, more than 64 slots, gradients with a bf16 output, and a dense output with D not a
multiple of 4 (the native ``linear`` operator).

``CharUnitEmbedder`` (strelementrepresentationmodel.py:100-142) runs its three convolutions and the max over positions as one native
kernel, ``ptgnn_b200_char_cnn_forward`` (DESIGN.md §3.13): the one-hot input and the [B, F, L] conv outputs never exist.  Its derived
weights (W1 as a gather table, W2 / W3 split and pre-swizzled) are kept per parameter version in eval mode, like the transformed table
above.  Gradients (fp32) are ``autograd._CharCnnFn``: token chunks, each re-running the kernel in its "materialise" mode.

``LinearFeatureEmbedder`` (linearmapembedding.py:13-29, the node embedder of the PPI model) is ``act(features W^T)`` on one persistent
kernel, ``ptgnn_b200_feature_embed_forward`` (DESIGN.md §3.15): the activation is applied in its epilogue, and inside a container's layer
loop it also writes the packed (hi | lo') rows of its fp32 output for the first fused layer.  Its prepared weights are kept per parameter
version in eval mode.  Gradients (fp32) are ``autograd._FeatureEmbedFn``.  Not supported (``NotImplementedError``): an embedding size
that is not a multiple of 8 in [8, 256], an input size outside [1, 512], activations other than None, ReLU, Tanh and GELU(erf), and
gradients with a bf16 output.
"""
import math
from typing import NamedTuple, Optional, Tuple

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


def new_status(words: int = 1) -> torch.Tensor:
    """A pinned int32 word for the kernels' count of out-of-range ids (polled by the host without synchronising); the char CNN uses a
    second word for its fp16-range flag."""
    return torch.zeros(words, dtype=torch.int32).pin_memory()


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
        N.call("ptgnn_b200_embedding_bag", table.device, int(out_dtype == torch.bfloat16), N.ptr(table), V, D, N.ptr(ids), N.ptr(lengths), B,
               S, N.POOL[mode], N.ptr(out), N.ptr(arg), N.ptr(status))
    elif B:
        out.fill_(-math.inf if mode == "max" else 0.0)
    return (out, arg) if want_arg else out


def occurrence_plan(ids: torch.Tensor, lengths: Optional[torch.Tensor], vocab: int) -> EdgePlan:
    """The edge plan of the (row -> token id) pairs of ids [B, S]: its rows are the vocabulary (row ``vocab`` is the sink of the
    padding slots), and its stable order lists a token's occurrences by (row, slot)."""
    B, S = ids.shape
    dev = ids.device
    src, tgt = torch.empty(B * S, dtype=torch.int64, device=dev), torch.empty(B * S, dtype=torch.int64, device=dev)
    N.call("ptgnn_b200_embedding_bag_pairs", dev, N.ptr(ids), N.ptr(lengths), B, S, vocab, N.ptr(src), N.ptr(tgt))
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
    N.call("ptgnn_b200_embedding_bag_backward_f32", dev, N.ptr(d_out), B, S, D, N.ptr(lengths), N.ptr(arg), N.POOL[mode], N.ptr(plan.row_ptr),
           N.ptr(plan.perm), vocab, N.ptr(d_table), N.ptr(ws), ws_bytes)
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

    _STATUS_WORDS = 1

    def __init__(self):
        super().__init__()
        self._status: Optional[torch.Tensor] = None
        self._transformed = None        # eval mode: (key, table W^T) or the char CNN's (key, prepared weights)

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
            self._status = new_status(self._STATUS_WORDS)
        return out

    def _status_word(self) -> torch.Tensor:
        if self._status is None:        # built on the GPU directly, or restored from a pickle
            self._status = new_status(self._STATUS_WORDS)
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


# ---------------------------------------------------------------------------------------------------------------------------------
# CharUnitEmbedder
# ---------------------------------------------------------------------------------------------------------------------------------
class CnnConfig(NamedTuple):
    """The reference's ``CnnConfig`` (strelementrepresentationmodel.py:92-97); any object with these five fields is accepted."""
    l1_filters: int
    l1_window_size: int
    l2_filters: int
    l2_window_size: int
    lout_window_size: int


def char_cnn_shape(conv1: nn.Conv1d, conv2: nn.Conv1d, conv3: nn.Conv1d) -> Tuple[int, int, int, int, int, int, int]:
    """(C, F1, w1, F2, w2, D, w3) of the three convolutions."""
    return (conv1.in_channels, conv1.out_channels, conv1.kernel_size[0], conv2.out_channels, conv2.kernel_size[0], conv3.out_channels,
            conv3.kernel_size[0])


def char_cnn_check(shape, L: int) -> None:
    C, F1, w1, F2, w2, D, w3 = shape
    if L < w1 + w2 + w3 - 2:
        raise RuntimeError(f"CharUnitEmbedder: {L} characters per token are fewer than the {w1 + w2 + w3 - 2} the three windows need")
    if not N.lib().ptgnn_b200_char_cnn_supported(C, F1, w1, F2, w2, D, w3, L):
        raise NotImplementedError(f"the char CNN kernel takes l1 / l2 filters in {{64, 128, 256}}, windows in [1, 5], an embedding size in "
                                  f"[1, 256] and up to 32 characters per token; got C={C}, F1={F1}, w1={w1}, F2={F2}, w2={w2}, D={D}, "
                                  f"w3={w3}, L={L}")


def char_cnn_prepare(shape, w1, b1, w2, b2, w3, bf16: bool, status: Optional[torch.Tensor]) -> torch.Tensor:
    """``ptgnn_b200_char_cnn_prepare``: the derived weights (gather table, biases, split and pre-swizzled W2 / W3) as a uint8 tensor."""
    lib = N.lib()
    nbytes = lib.ptgnn_b200_char_cnn_workspace_bytes(int(bf16), *shape)
    dev = w1.device
    buf = torch.empty(nbytes + 1024, dtype=torch.uint8, device=dev)
    off = (-buf.data_ptr()) % 1024
    prepared = buf[off:off + nbytes]
    ws = [N.require_cuda(t.detach(), name, torch.float32) for t, name in ((w1, "W1"), (b1, "b1"), (w2, "W2"), (b2, "b2"), (w3, "W3"))]
    N.call("ptgnn_b200_char_cnn_prepare", dev, int(bf16), *[N.ptr(t) for t in ws], *shape, N.ptr(prepared), nbytes, N.ptr(status))
    return prepared


def native_char_cnn(chars: torch.Tensor, shape, prepared: torch.Tensor, bf16: bool = False, want_arg: bool = False,
                    status: Optional[torch.Tensor] = None):
    """``ptgnn_b200_char_cnn_forward``: out [B, D] (fp32, or bf16 with ``bf16``) from chars [B, L] int64 and ``char_cnn_prepare``d
    weights of the same ``bf16`` flag.  ``want_arg``: also the [B, D] uint8 winning positions."""
    chars = N.require_cuda(chars, "chars", torch.int64)
    if chars.dim() != 2:
        raise ValueError(f"chars must be [B, max_num_chars], got {tuple(chars.shape)}")
    B, L = chars.shape
    char_cnn_check(shape, L)
    D = shape[5]
    out = torch.empty(B, D, dtype=torch.bfloat16 if bf16 else torch.float32, device=chars.device)
    arg = torch.empty(B, D, dtype=torch.uint8, device=chars.device) if want_arg else None
    if B:
        N.call("ptgnn_b200_char_cnn_forward", chars.device, int(bf16), N.ptr(chars), B, L, *shape, N.ptr(prepared), prepared.numel(),
               N.ptr(out), N.ptr(arg), N.ptr(status))
    return (out, arg) if want_arg else out


def native_char_cnn_materialise(chars: torch.Tensor, shape, prepared: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``ptgnn_b200_char_cnn_materialise_f32``: the post-ReLU a1 [B (L - w1 + 1), F1] and a2 [B (L - w1 - w2 + 2), F2] of fp32
    ``prepared`` weights."""
    B, L = chars.shape
    C, F1, w1, F2, w2, D, w3 = shape
    L1, L2 = L - w1 + 1, L - w1 - w2 + 2
    a1 = torch.empty(B * L1, F1, dtype=torch.float32, device=chars.device)
    a2 = torch.empty(B * L2, F2, dtype=torch.float32, device=chars.device)
    if B:
        N.call("ptgnn_b200_char_cnn_materialise_f32", chars.device, N.ptr(chars), B, L, *shape, N.ptr(prepared), prepared.numel(), N.ptr(a1),
               N.ptr(a2), None)
    return a1, a2


def poll_char_status(status: torch.Tensor, vocab: int) -> None:
    poll_status(status, vocab)
    if int(status[1]):
        status[1] = 0
        raise FloatingPointError("CharUnitEmbedder: an fp32 weight or activation is outside the fp16 range (|x| >= 65504) of the "
                                 "kernel's split products; results are not valid")


class CharUnitEmbedder(_NativeEmbedder):
    _STATUS_WORDS = 2

    def __init__(self, num_chars: int, embedding_size: int, config: CnnConfig, dropout_rate: float = 0.0):
        super().__init__()
        self.__num_chars_in_vocabulary = num_chars
        self.__conv_l1 = nn.Conv1d(in_channels=num_chars, out_channels=config.l1_filters, kernel_size=config.l1_window_size)
        self.__conv_l2 = nn.Conv1d(in_channels=config.l1_filters, out_channels=config.l2_filters, kernel_size=config.l2_window_size)
        self.__conv_l3 = nn.Conv1d(in_channels=config.l2_filters, out_channels=embedding_size, kernel_size=config.lout_window_size,
                                   bias=False)
        self.__dropout = nn.Dropout(p=dropout_rate)

    def _params(self):
        return (self.__conv_l1.weight, self.__conv_l1.bias, self.__conv_l2.weight, self.__conv_l2.bias, self.__conv_l3.weight)

    def _prepared(self, shape, bf16: bool, status: torch.Tensor) -> torch.Tensor:
        """The derived weights.  Kept in eval mode while no parameter was modified in place, re-assigned or moved; derived on every
        call in training mode (edits through ``.data`` do not move the version counter)."""
        params = self._params()
        if self.training:
            return char_cnn_prepare(shape, *params, bf16, status)
        key = (bf16,) + tuple((p.data_ptr(), p._version, p.device, p.dtype) for p in params)
        if self._transformed is None or self._transformed[0] != key:
            self._transformed = (key, char_cnn_prepare(shape, *params, bf16, status))
        return self._transformed[1]

    def forward(self, chars: torch.Tensor) -> torch.Tensor:
        """
        :param chars: [B, max_num_chars] int64
        :return: [B, D] (fp32; bf16 under ``torch.autocast("cuda", bfloat16)``)
        """
        params = self._params()
        N.require_cuda(params[0], "conv_l1 weight", torch.float32)
        if chars.dim() != 2:
            raise ValueError(f"chars must be [B, max_num_chars], got {tuple(chars.shape)}")
        shape = char_cnn_shape(self.__conv_l1, self.__conv_l2, self.__conv_l3)
        char_cnn_check(shape, chars.shape[1])
        bf16 = _bf16_autocast(params[0].device)
        grad = _wants_grad(*params)
        if bf16 and grad:
            raise NotImplementedError("CharUnitEmbedder: gradients with a bf16 output have no native kernel; train in fp32")
        status = self._status_word()
        poll_char_status(status, self.__num_chars_in_vocabulary)
        prepared = self._prepared(shape, bf16, status)
        if grad:
            from . import autograd as _ag

            out = _ag.char_cnn_with_grad(chars, shape, prepared, status, *params)
        else:
            out = native_char_cnn(chars, shape, prepared, bf16, status=status)
        poll_char_status(status, self.__num_chars_in_vocabulary)
        return self.__dropout(out)


# ---------------------------------------------------------------------------------------------------------------------------------
# LinearFeatureEmbedder
# ---------------------------------------------------------------------------------------------------------------------------------
def feature_embed_check(F: int, D: int) -> None:
    if not N.lib().ptgnn_b200_feature_embed_supported(F, D):
        raise NotImplementedError(f"the feature-embedding kernel takes an input size in [1, 512] and an embedding size that is a multiple "
                                  f"of 8 in [8, 256]; got input_element_size={F}, output_embedding_size={D}")


def feature_embed_prepare(weight: torch.Tensor, bf16: bool, status: Optional[torch.Tensor]) -> torch.Tensor:
    """``ptgnn_b200_feature_embed_prepare``: W [D, F] split (fp32) or rounded (bf16), padded and pre-swizzled, as a uint8 tensor."""
    D, F = weight.shape
    w = N.require_cuda(weight.detach(), "weight", torch.float32)
    nbytes = N.lib().ptgnn_b200_feature_embed_workspace_bytes(int(bf16), F, D)
    prepared = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
    N.call("ptgnn_b200_feature_embed_prepare", w.device, int(bf16), N.ptr(w), F, D, N.ptr(prepared), nbytes, N.ptr(status))
    return prepared


def native_feature_embed(x: torch.Tensor, prepared: torch.Tensor, D: int, activation: int, bf16: bool = False, want_packed: bool = False,
                         want_pre: bool = False, status: Optional[torch.Tensor] = None):
    """``ptgnn_b200_feature_embed_forward``: (out [N, D], packed or None, pre or None) from x [N, F] fp32 and ``feature_embed_prepare``d
    weights of the same ``bf16`` flag.  out is fp32, or bf16 with ``bf16``.  ``want_packed`` (fp32): also the packed (hi | lo') rows the
    fused layers take as their packed input; ``want_pre`` (fp32): also the pre-activation [N, D]."""
    x = N.require_cuda(x, "features", torch.float32)
    if x.dim() != 2:
        raise ValueError(f"features must be [N, F], got {tuple(x.shape)}")
    rows, F = x.shape
    feature_embed_check(F, D)
    dev = x.device
    out = torch.empty(rows, D, dtype=torch.bfloat16 if bf16 else torch.float32, device=dev)
    packed = pre = None
    if want_packed and not bf16:
        packed = torch.empty(max(N.lib().ptgnn_b200_packed_state_bytes(rows, D), 1), dtype=torch.uint8, device=dev)
    if want_pre and not bf16:
        pre = torch.empty(rows, D, dtype=torch.float32, device=dev)
    if rows:
        N.call("ptgnn_b200_feature_embed_forward", dev, int(bf16), N.ptr(x), rows, F, D, activation, N.ptr(prepared), prepared.numel(),
               N.ptr(out), N.ptr(packed), N.ptr(pre), N.ptr(status))
    return out, packed, pre


def native_activation_grad(activation: int, grad_out: torch.Tensor, saved: torch.Tensor) -> torch.Tensor:
    """``ptgnn_b200_activation_grad_f32``: grad_out act'(pre), with ``saved`` the output (ReLU, Tanh) or the pre-activation (GELU)."""
    grad_out = N.require_cuda(grad_out, "grad_out", torch.float32)
    saved = N.require_cuda(saved, "saved", torch.float32)
    d_pre = torch.empty_like(grad_out)
    N.call("ptgnn_b200_activation_grad_f32", grad_out.device, activation, N.ptr(grad_out), N.ptr(saved), grad_out.numel(), N.ptr(d_pre))
    return d_pre


def poll_feature_status(status: torch.Tensor) -> None:
    if int(status[0]):
        status[0] = 0
        raise FloatingPointError("LinearFeatureEmbedder: an fp32 feature, weight or output is outside the fp16 range (|x| >= 65504) of "
                                 "the kernel's split products; results are not valid")


class LinearFeatureEmbedder(_NativeEmbedder):
    """``activation(features W^T)`` on one native kernel (DESIGN.md §3.15).  Inside a container's layer loop (``edgeplan.state_chain``)
    the fp32 forward also writes the packed form of its output, so that a first fused layer skips its packing pass."""

    def __init__(self, input_element_size: int, output_embedding_size: int, activation: Optional[nn.Module] = None):
        super().__init__()
        self.__linear_map = nn.Linear(input_element_size, output_embedding_size, bias=False)
        nn.init.xavier_uniform_(self.__linear_map.weight)
        self.__activation = activation

    def _prepared(self, weight: torch.Tensor, bf16: bool, status: torch.Tensor) -> torch.Tensor:
        """The prepared weights.  Kept in eval mode while the weight was not modified in place, re-assigned or moved; derived on every
        call in training mode (edits through ``.data`` do not move the version counter)."""
        if self.training:
            return feature_embed_prepare(weight, bf16, status)
        key = (bf16, weight.data_ptr(), weight._version, weight.device, weight.dtype)
        if self._transformed is None or self._transformed[0] != key:
            self._transformed = (key, feature_embed_prepare(weight, bf16, status))
        return self._transformed[1]

    def forward(self, features: torch.Tensor) -> torch.Tensor:
        """
        :param features: [N, input_element_size] fp32
        :return: [N, output_embedding_size] (fp32; bf16 under ``torch.autocast("cuda", bfloat16)``)
        """
        from .edgeplan import current_state_chain
        from .messagepassing import _activation_code

        weight = self.__linear_map.weight
        D, F = weight.shape
        feature_embed_check(F, D)
        act = _activation_code(self.__activation, "LinearFeatureEmbedder activation")
        if features.dim() != 2 or features.shape[1] != F:
            raise ValueError(f"features must be [N, {F}], got {tuple(features.shape)}")
        bf16 = _bf16_autocast(weight.device)
        grad = _wants_grad(weight, features)
        if bf16 and grad:
            raise NotImplementedError("LinearFeatureEmbedder: gradients with a bf16 output have no native kernel; train in fp32")
        N.require_cuda(weight, "weight", torch.float32)
        if bf16 and features.dtype in (torch.bfloat16, torch.float16):
            features = features.float()          # exact; the kernel rounds to bf16 as autocast's Linear would
        x = N.require_cuda(features, "features", torch.float32)
        status = self._status_word()
        poll_feature_status(status)
        prepared = self._prepared(weight, bf16, status)
        if grad:
            from . import autograd as _ag

            out = _ag.feature_embed_with_grad(x, weight, prepared, act, status)
        else:
            chain = None if bf16 else current_state_chain()
            out, packed, _ = native_feature_embed(x, prepared, D, act, bf16, want_packed=chain is not None and chain.want_output,
                                                  status=status)
            if chain is not None:
                chain.store(out, packed)
        poll_feature_status(status)
        return out
