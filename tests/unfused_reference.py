"""Float64 references of the unfused layer kernels with an error bound for every output element, and a graph built to drive
them through their tile edges.

The kernels: the 3xTF32 tensor-core pipeline (csrc/tc_pipeline.cuh with the message, GRU and dense policies of
csrc/layers_tc.cu), its bf16 version (csrc/tc_pipeline_bf16.cuh, same policies), the FFMA kernels (csrc/layers.cu,
csrc/gemm_simt.cuh) and the two segmented reduces (csrc/reduce.cuh).  u = 2^-24 throughout; the sequential fp32 sum, the
bf16 message model and the bf16 rounding window come from ``fused_reference``.  The float64 products run on whatever device
the inputs are on (a float64 GEMM errs by ~2^-50 of the mass, far below every bound here).

3xTF32 GEMM.  Each fp32 operand x is split into hi = tf32_hi(x), rounded to nearest on 10 mantissa bits, so
|x - hi| <= 2^-11 |x|, and lo = x - hi, exact in fp32.  We assume the tensor cores truncate lo to TF32 (the larger of the
two possible errors): |lo - lo'| <= 2^-10 |lo| <= 2^-21 |x| = 8u |x|.  The kernel adds hi*hi into the main accumulator and
hi*lo' + lo'*hi into a correction accumulator and drops lo*lo (<= 2^-22 |x w| = 4u |x w|).  Per product that is
(8 + 8 + 4) u |x w| to first order, 21u with the second-order terms.  Each 8-wide k-step adds one block of exact products
into an fp32 accumulator; we allow 2u of the mass per step (one ulp: truncating alignment), as ``fused_reference`` does per
16-wide step.  The correction accumulator holds 2^-11 of the mass: 1u for all of its steps.  Adding the two accumulators
costs 1u.  So with S = sum over the GEMM's K segments of ceil(K / 8) steps

    |y~ - y| <= C * mass + 2^-100 K,   C = (21 + 2 S + 1 + 1) u,   mass = sum_k |w_k x_k|.

K is H for a message (2H with target states: S counts both halves), D for the dense layer, D + H for the GRU's r and z
gates.  A kernel that runs hi*hi alone errs by ~2^-11 / sqrt(K) of the mass and fails this (``test_unfused_reference_cpu``).

FFMA kernels: a plain fp32 fma chain over K terms and the bias: gamma_{K+1} (mass + |b|), gamma_n = n u / (1 - n u).

bf16 tensor cores: bf16 operands, exact products, fp32 accumulation per 16-wide k-step: (4 S + 4) u of the mass with
S = sum ceil(K / 16) (``fused_reference.bf16_window_constant``).

3xFP16 (mode '3xfp16': the weights-stationary GRU, csrc/gru_ws.cu, on fp32 states).  The aggregate arrives as the fused
write-out's fp16 (hi | lo') split, the states as ``pack_states`` rows and the weights as ``pack_gru_ws_kernel`` packs them, all
with the same split: hi = fl16(x), lo' = fl16(2^11 (x - hi)).  The kernel adds hi*hi into the main accumulator and hi*lo' then
lo'*hi into the correction accumulator, 16-wide k-steps each, and combines them as fmaf(corr, 2^-11, main).  That is the
arithmetic of ``fused_reference``'s messages, so per gate group the constant is the same, (14 + 2 S) u of the mass, plus
2^-36 (sum_k |x_k| + sum_k |w_k|) for operands whose lo' is an fp16 subnormal; here S = (H + D) / 16 for r and z (state and
aggregate chunks share their accumulator), D / 16 for i_n and H / 16 for h_n.  S reaches 28 at H = 448 in the state-only
instance, past the 2^-18 that ``fused_reference.fp32_message_constant`` asserts for messages, so this constant has its own
function (``f16x3_constant``).  Messages follow ``fused_reference.messages``; every
other bf16 output (aggregate, LayerNorm output, dense output, GRU output) is the bf16 rounding of an fp32 value within its
fp32 bound e of the reference, so it lies within e + 1 bf16 ulp of the rounded reference.

Reduces.  For given fp32 messages the sum is bit-exact on both kernels: a sequential fp32 sum in edge order from 0.  The
mean is that sum divided by the count in one IEEE fp32 division: bit-exact too.  Max / min values and args are exact:
strict compares, so ties go to the first occurrence; empty rows hold 0 and arg = E.

Epilogues.  An activation propagates a bound through its Lipschitz constant (GELU 1.13, ReLU 1; tanh: its largest slope
within the bound, so that a saturated row keeps a tight bound) and adds its fp32 evaluation error, 8u (|x| + |act(x)|) (erff and tanhf are within 2 ulp).  LayerNorm over a row x with input bound b_i:
the mean moves by mean(b) plus gamma_D of mean(|x| + b); each centred value d_i by eta_i = b_i + that + u |d_i|; by
Minkowski's inequality sqrt(mean(d^2) + eps) moves by at most ||eta||_2 / sqrt(D), and its fp32 evaluation (a sum of D
squares, a division, the eps add, rsqrtf within 2 ulp) adds gamma_D / 2 + 5u relative.  With rho the total relative change
of the reciprocal standard deviation r, |y~_i - y_i| <= |w_i| r (eta_i + (|d_i| + eta_i) rho / (1 - rho)) + 3u |w_i d_i r|
+ u |y_i|.

GRU (nn.GRUCell).  The gate pre-activations carry their GEMM bound plus the rounding of each bias add.  sigma' <= 1/4 and
tanh' <= 1 carry them through the gates; then each approximate function adds its own error:
  * sigmoid_fast(x) = rcp.approx(1 + __expf(-x)) (fp32 tensor-core GRU): __expf is within 2 + 1.2 |x| ulp, which moves
    1 + e^-x by (1 - s)(2 + 1.2 |x|) 2u relative; the add and rcp.approx (1 ulp) add 3u: err <= s ((1 - s)(2 + 1.2|x|) 2u + 3u).
  * tanh_fast(x) = 1 - 2 rcp.approx(__expf(2x) + 1): the same with s = sigma(-2x) and 2x, doubled, plus 4u (|t| + 1) for
    the final subtraction.  This also covers the FFMA kernel's expf / tanhf (within 2 ulp).
  * tanh.approx.f32 (bf16 GRU, and sigmoid as 0.5 tanh(x / 2) + 0.5): relative error <= 2^-10.98; we use 2^-10.9 |t| + 2^-20.
Then h' = (1 - z) n + z h moves by |1 - z| dn + dz (|n - h| + dn) plus 3u (|(1 - z) n| + |z h|) + u |h'|.  The bf16 kernels
blend as fmaf(z, h - n, n) instead: the rounding of h - n, scaled by z, adds u z |h - n|, which the terms above do not hold when
z -> 1 and |n| >> |h| (then |(1 - z) n| and |z h| are both small while |z (h - n)| is about |n|).
Every GRU and LayerNorm bound is widened by 2 % for the second-order terms dropped above.

State-only GRU (``gru_table``: GruGlobalStateUpdate, the TABLE instance of csrc/gru_ws.cu).  The input side gi = g W_ih^T + b_ih
is an fp32 table from ``ptgnn_b200_linear_f32`` (``dense`` in ``fp32_dense_mode``, with its own bound), also when the states are
bf16, so the bf16 form mixes an fp32 gi with bf16 W_hh and h; the kernel's bias vector holds b_hr, b_hz, b_hn only (b_ih is in
the table).  Its order of adds: r = sigma((h W_hr + b_hr) + gi_r), z likewise, n = tanh(gi_n + r (h W_hn + b_hn)); each of
those adds rounds once (u of its result), and gi's bound passes through the gates like the GEMM bound.
"""
import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

import fused_reference as FR

U = FR.U
ABS_TF32 = 2.0 ** -100
SM_COUNT = 132                      # H100 SXM: the persistent pipelines launch one CTA per SM
TILE_M = 128                        # edges / rows per tile of the tensor-core pipelines
WARP_ROWS = 16                      # target rows per warp of the streaming reduce


def gamma(n) -> float:
    return n * U / (1 - n * U)


def tf32_constant(*Ks: int) -> float:
    S = sum(math.ceil(K / 8) for K in Ks)
    return (21 + 2 * S + 1 + 1) * U


def ffma_constant(*Ks: int) -> float:
    return gamma(sum(Ks) + 1)


def bf16_constant(*Ks: int) -> float:
    return (4 * sum(math.ceil(K / 16) for K in Ks) + 4) * U


def f16x3_constant(*Ks: int) -> float:
    return (14 + 2 * sum(math.ceil(K / 16) for K in Ks)) * U


def gemm_constant(mode: str, *Ks: int) -> float:
    return {"tc": tf32_constant, "ffma": ffma_constant, "bf16": bf16_constant, "3xfp16": f16x3_constant}[mode](*Ks)


def _abs_term(mode: str, xa: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """The absolute part of a GEMM bound, [rows or 1, out]: 3xFP16 2^-36 (sum_k |x_k| + sum_k |w_k|) (xa = |x|), else 2^-100 K."""
    if mode == "3xfp16":
        return FR.ABS_F16 * (xa.sum(1, keepdim=True) + W.abs().sum(1)[None, :])
    return torch.full((1, W.shape[0]), ABS_TF32 * W.shape[1], dtype=torch.float64, device=W.device)


def fp32_message_mode(H: int, D: int) -> str:
    """Which kernel computes fp32 messages (layers.cu edge_messages; tc::supported_message)."""
    return "tc" if H % 4 == 0 and D % 16 == 0 and H >= 32 and D >= 16 else "ffma"


def fp32_gru_mode(H: int, D: int) -> str:
    return "tc" if H % 32 == 0 and D % 4 == 0 and D >= 32 else "ffma"


def fp32_dense_mode(D: int, Hout: int) -> str:
    return "tc" if D % 4 == 0 and Hout % 16 == 0 and D >= 32 else "ffma"


_bf16 = FR._bf16


def round_bf16(ref: torch.Tensor, bnd: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    ref_b = _bf16(ref)
    return ref_b, bnd + FR._bf16_ulp(ref_b.abs() + bnd)


# ---- messages ---------------------------------------------------------------------------------------------------------
def fp32_messages(h: torch.Tensor, adj, weights: Sequence[torch.Tensor], use_target: bool, mode: Optional[str] = None,
                  device=None, chunk: int = 16384):
    """-> (tgt [E] int64, m [E, D] float64, err [E, D] float64) in concatenated (type-major) edge order, on the CPU.  ``mode``
    'tc' (3xTF32) or 'ffma'; default: the kernel the library picks for these dims."""
    dev = device or h.device
    H, D = h.shape[1], weights[0].shape[0]
    mode = mode or fp32_message_mode(H, D)
    c = gemm_constant(mode, *((H, H) if use_target else (H,)))
    h64 = h.to(dev).double()
    tgts, ms, errs = [], [], []
    for (s, t), w in zip(adj, weights):
        W = w.to(dev).double()
        Wa = W.abs()
        s, t = s.to(dev), t.to(dev)
        for a in range(0, s.shape[0], chunk):
            X = torch.cat([h64[s[a:a + chunk]], h64[t[a:a + chunk]]], 1) if use_target else h64[s[a:a + chunk]]
            ms.append((X @ W.T).cpu())
            errs.append((c * (X.abs() @ Wa.T) + ABS_TF32 * W.shape[1]).cpu())
        tgts.append(t.cpu())
    if not ms:
        return torch.cat(tgts), torch.zeros(0, D, dtype=torch.float64), torch.zeros(0, D, dtype=torch.float64)
    return torch.cat(tgts), torch.cat(ms), torch.cat(errs)


# ---- reductions -------------------------------------------------------------------------------------------------------
def reduce_exact(tgt: torch.Tensor, m32: torch.Tensor, num_nodes: int, reduce: str):
    """The segmented reduce of fp32 rows ``m32`` (edge order) as the kernels compute it -> (out [N, D] float32, arg [N, D]
    int64 or None).  sum / mean: sequential fp32 sum, one fp32 division.  max / min: first occurrence wins, empty -> 0 / E."""
    E, D = m32.shape
    m = m32.float().cpu()
    cnt = torch.bincount(tgt, minlength=num_nodes)
    if reduce in ("sum", "mean"):
        s = torch.from_numpy(FR._seq_sum_f32(tgt, m.numpy(), num_nodes))
        if reduce == "mean":
            s = torch.from_numpy(s.numpy() / cnt.clamp(min=1).numpy().astype(np.float32)[:, None])
        return s, None
    op = "amax" if reduce == "max" else "amin"
    idx = tgt[:, None].expand(E, D)
    init = -math.inf if reduce == "max" else math.inf
    val = torch.full((num_nodes, D), init, dtype=torch.float32).scatter_reduce_(0, idx, m, op)
    win = m == val[tgt]
    eid = torch.where(win, torch.arange(E)[:, None].expand(E, D), torch.full((E, D), E, dtype=torch.int64))
    arg = torch.full((num_nodes, D), E, dtype=torch.int64).scatter_reduce_(0, idx, eid, "amin")
    val = torch.where(arg == E, torch.zeros_like(val), val)
    return val, arg


def layer_norm(x: torch.Tensor, bx: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float):
    """LayerNorm of the float64 rows x whose fp32 version in the kernel lies within bx -> (ref, bound)."""
    D = x.shape[1]
    w, b = w.double()[None, :], b.double()[None, :]
    mu = x.mean(1, keepdim=True)
    d = x - mu
    sig = torch.sqrt((d * d).mean(1, keepdim=True) + eps)
    r = 1.0 / sig
    y = d * r * w + b
    dmu = bx.mean(1, keepdim=True) + gamma(D) * (x.abs() + bx).mean(1, keepdim=True) + U * mu.abs()
    eta = bx + dmu + U * (d.abs() + bx + dmu)
    rho = eta.norm(dim=1, keepdim=True) / (math.sqrt(D) * sig) + gamma(D) / 2 + 5 * U
    assert float(rho.max()) < 0.5, "LayerNorm input bound too wide to linearise"
    rho = rho / (1 - rho)
    bnd = w.abs() * r * (eta + (d.abs() + eta) * rho) + 3 * U * (w * d * r).abs() + U * y.abs()
    return y, 1.02 * bnd


# ---- dense layer ------------------------------------------------------------------------------------------------------
def dense(y: torch.Tensor, ey: Optional[torch.Tensor], W: torch.Tensor, bias: Optional[torch.Tensor], act: Optional[str], mode: str):
    """act(y W^T + b) for float64 rows y (their kernel version within ey) -> (ref, bound), on y's device.  mode 'tc' /
    'ffma' (fp32) or 'bf16' (bf16 weights and output)."""
    dev = y.device
    W = (_bf16(W) if mode == "bf16" else W.double()).to(dev)
    Wa = W.abs()
    pre = y @ W.T
    mass = y.abs() @ Wa.T
    b = torch.zeros(W.shape[0], dtype=torch.float64, device=dev) if bias is None else bias.double().to(dev)
    pre = pre + b
    e = gemm_constant(mode, y.shape[1]) * (mass + b.abs()) + ABS_TF32 * y.shape[1] + U * pre.abs()
    if ey is not None:
        e = e + (ey @ Wa.T) * (1 + 2.0 ** -10)
    ref, e = FR.activation_bound(pre, e, act)
    if mode == "bf16":
        ref, e = round_bf16(ref, e)
    return ref, e


# ---- GRU --------------------------------------------------------------------------------------------------------------
def _sigmoid_err_fast(a: torch.Tensor) -> torch.Tensor:
    s = torch.sigmoid(a)
    return 1.05 * s * ((1 - s) * (2 + 1.2 * a.abs()) * 2 * U + 3 * U) + 2.0 ** -120


def _tanh_err_fast(c: torch.Tensor) -> torch.Tensor:
    s = torch.sigmoid(-2 * c)
    return 1.05 * 2 * s * ((1 - s) * (2 + 2.4 * c.abs()) * 2 * U + 3 * U) + 4 * U * (torch.tanh(c).abs() + 1)


def _tanh_err_mufu(c: torch.Tensor) -> torch.Tensor:
    return 2.0 ** -10.9 * torch.tanh(c).abs() + 2.0 ** -20


def _sigmoid_err_mufu(a: torch.Tensor) -> torch.Tensor:
    return 0.5 * _tanh_err_mufu(0.5 * a) + U


def _gate_errors(mode: str):
    return (_sigmoid_err_mufu, _tanh_err_mufu) if mode == "bf16" else (_sigmoid_err_fast, _tanh_err_fast)


def _sigmoid_gate(a: torch.Tensor, e: torch.Tensor, mode: str):
    return torch.sigmoid(a), 0.25 * e + _gate_errors(mode)[0](a.abs() + e)


def _gru_blend(z, dz, c, dc, h, mode: str):
    """n = tanh(c), h' = (1 - z) n + z h from the gates and their bounds -> (ref, bound); bf16: fmaf(z, h - n, n), rounded."""
    n = torch.tanh(c)
    dn = dc + _gate_errors(mode)[1](c.abs() + dc)
    out = (1 - z) * n + z * h
    e = (1 - z) * dn + dz * ((n - h).abs() + dn) + 3 * U * (((1 - z) * n).abs() + (z * h).abs()) + U * out.abs()
    if mode == "bf16":
        e = e + U * z * (h - n).abs()
    e = 1.02 * e
    if mode == "bf16":
        return round_bf16(out, e)
    return out, e


def gru(x: torch.Tensor, ex: Optional[torch.Tensor], h: torch.Tensor, w_ih, w_hh, b_ih, b_hh, mode: str):
    """nn.GRUCell(x, h) in float64 -> (ref, bound), on x's device.  x's kernel version lies within ex (None: exact input); h
    is exact.  mode 'tc' / 'ffma' / '3xfp16' (fp32) or 'bf16' (bf16 x, h, weights and output)."""
    dev = x.device
    H, D = h.shape[1], x.shape[1]
    cast = _bf16 if mode == "bf16" else (lambda t: t.double())
    Wi, Wh = cast(w_ih).to(dev), cast(w_hh).to(dev)
    bi, bh = b_ih.double().to(dev), b_hh.double().to(dev)
    x, h = x.double(), h.double().to(dev)
    gi, gh = x @ Wi.T, h @ Wh.T
    mi, mh = x.abs() @ Wi.abs().T, h.abs() @ Wh.abs().T
    pe = torch.zeros_like(gi) if ex is None else (ex @ Wi.abs().T) * (1 + 2.0 ** -10)
    ai = _abs_term(mode, x.abs() if ex is None else x.abs() + ex, Wi)
    ah = _abs_term(mode, h.abs(), Wh)
    c_rz, c_i, c_h = gemm_constant(mode, D, H), gemm_constant(mode, D), gemm_constant(mode, H)
    g = lambda t, k: t[:, k * H:(k + 1) * H]
    gate = []
    for k in (0, 1):                                            # r, z
        bsum = bi[k * H:(k + 1) * H] + bh[k * H:(k + 1) * H]
        a = g(gi, k) + g(gh, k) + bsum
        e = c_rz * (g(mi, k) + g(mh, k)) + g(pe, k) + U * (bsum.abs() + a.abs()) + g(ai, k) + g(ah, k)
        gate.append(_sigmoid_gate(a, e, mode))
    (r, dr), (z, dz) = gate
    gn = g(gi, 2) + bi[2 * H:]
    en = c_i * g(mi, 2) + g(pe, 2) + U * gn.abs() + g(ai, 2)
    gh_n = g(gh, 2) + bh[2 * H:]
    ehn = c_h * g(mh, 2) + U * gh_n.abs() + g(ah, 2)
    c = gn + r * gh_n
    dc = en + r * ehn + dr * (gh_n.abs() + ehn) + U * ((r * gh_n).abs() + c.abs())
    return _gru_blend(z, dz, c, dc, h, mode)


def gru_table(gi: torch.Tensor, e_gi: torch.Tensor, h: torch.Tensor, w_hh, b_hh, mode: str):
    """The state-only GRU: GRUCell with the input-side pre-activations given per row -> (ref, bound), on gi's device.  gi [N, 3H]
    (gates r, z, n; b_ih included) is the float64 table row of each node's graph and its fp32 version lies within e_gi; h is
    exact.  mode '3xfp16' (fp32 states) or 'bf16' (bf16 h, W_hh and output; gi stays fp32)."""
    dev = gi.device
    H = h.shape[1]
    Wh = (_bf16(w_hh) if mode == "bf16" else w_hh.double()).to(dev)
    bh = b_hh.double().to(dev)
    h = h.double().to(dev)
    gh, mh = h @ Wh.T, h.abs() @ Wh.abs().T
    ah = _abs_term(mode, h.abs(), Wh)
    c_h = gemm_constant(mode, H)
    g = lambda t, k: t[:, k * H:(k + 1) * H]
    hb = [g(gh, k) + bh[k * H:(k + 1) * H] for k in range(3)]         # h W_h + b_h, one rounding each
    eh = [c_h * g(mh, k) + g(ah, k) + U * hb[k].abs() for k in range(3)]
    gate = []
    for k in (0, 1):                                            # r, z: (h W_h + b_h) + gi
        a = hb[k] + g(gi, k)
        gate.append(_sigmoid_gate(a, eh[k] + g(e_gi, k) + U * a.abs(), mode))
    (r, dr), (z, dz) = gate
    c = g(gi, 2) + r * hb[2]
    dc = g(e_gi, 2) + r * eh[2] + dr * (hb[2].abs() + eh[2]) + U * ((r * hb[2]).abs() + c.abs())
    return _gru_blend(z, dz, c, dc, h, mode)


# ---- structured graphs ------------------------------------------------------------------------------------------------
TYPE_COUNTS = (0, 1, 127, 128, 129, 255, 256, 257)   # per-type edge counts around the 128-edge tile boundary
EMPTY_RUNS = (1, 15, 16, 17, 33)                     # zero in-degree runs, at the start, middle and end of a 16-row warp block
HUB_DEGREE = 2100


def structured_graph(num_nodes: int, big: int = 20_000, seed: int = 0):
    """Deterministic graph for the unfused kernels -> (adjacency list, empty-run starts {(length, where): row}).

    Edge types: three large ones (big, big, big / 2 edges) with every count of TYPE_COUNTS between them, so tile runs cross
    type boundaries and empty types; at the default size that is >= 3 waves of 128-edge tiles on 132 SMs.  Type 0 holds a hub
    target with HUB_DEGREE in-edges and duplicated edges (exact ties).  Rows without in-edges: every run length of EMPTY_RUNS
    starting on a 16-row warp block, starting 5 rows into one and ending on one's last row, plus the last three rows.  List
    order is not target order.  ``structure_facts`` recomputes all of it."""
    rng = np.random.RandomState(seed)
    N = num_nodes
    empty = np.zeros(N, dtype=bool)
    runs = {}
    blk = 2
    for L in EMPTY_RUNS:
        for where in ("start", "middle", "end"):
            base = WARP_ROWS * blk
            start = {"start": base, "middle": base + 5, "end": base + 3 * WARP_ROWS - L}[where]
            assert start + L < N - 4, "graph too small for its empty runs"
            empty[start:start + L] = True
            runs[(L, where)] = start
            blk += (L + 5) // WARP_ROWS + 5
    empty[N - 3:] = True
    live = np.flatnonzero(~empty)
    hub = int(live[len(live) // 2])
    counts = [big] + list(TYPE_COUNTS[:5]) + [big] + list(TYPE_COUNTS[5:]) + [big // 2]
    adj = []
    for t, n in enumerate(counts):
        src = rng.randint(0, N, n)
        tgt = live[rng.randint(0, len(live), n)]
        if t == 6:                                                  # every other row gets an edge: the runs stay as designed
            assert n >= len(live), "graph too small to cover its rows"
            tgt[:len(live)] = live
        if t == 0:
            tgt[:HUB_DEGREE] = hub
            dup = rng.randint(HUB_DEGREE, n, 64)                   # duplicated edges: same source, target and type
            src[dup[:32]], tgt[dup[:32]] = src[dup[32:]], tgt[dup[32:]]
            src[:4] = src[HUB_DEGREE - 4:HUB_DEGREE]                # and duplicated hub edges
        perm = rng.permutation(n)
        adj.append((torch.from_numpy(src[perm].astype(np.int64)), torch.from_numpy(tgt[perm].astype(np.int64))))
    return adj, runs


def structure_facts(adj, num_nodes: int) -> Dict[str, object]:
    counts = [int(s.shape[0]) for s, _ in adj]
    src = torch.cat([s for s, _ in adj]).numpy()
    tgt = torch.cat([t for _, t in adj]).numpy()
    et = np.repeat(np.arange(len(adj)), counts)
    deg = np.bincount(tgt, minlength=num_nodes)
    runs = set()
    zero = np.r_[False, deg == 0, False]
    starts = np.flatnonzero(~zero[:-1] & zero[1:])
    ends = np.flatnonzero(zero[:-1] & ~zero[1:])
    for s, e in zip(starts, ends):
        L = int(e - s)
        if s % WARP_ROWS == 0:
            runs.add((L, "start"))
        if e % WARP_ROWS == 0:
            runs.add((L, "end"))
        if s % WARP_ROWS != 0 and e % WARP_ROWS != 0:
            runs.add((L, "middle"))
    keys = np.unique(np.stack([src, tgt, et]), axis=1)
    ties = 0
    for t in range(len(adj)):
        sel = et == t
        ties += int(sel.sum() - np.unique(np.stack([src[sel], tgt[sel]]), axis=1).shape[1])
    return dict(
        type_counts=counts,
        tiles=sum((c + TILE_M - 1) // TILE_M for c in counts),
        max_in_degree=int(deg.max()),
        empty_runs=runs,
        trailing_empty=int(np.argmax(deg[::-1] != 0)),
        duplicates=int(src.shape[0] - keys.shape[1]),
        same_type_duplicates=ties,
        mod16=num_nodes % 16,
        mod128=num_nodes % 128,
    )
