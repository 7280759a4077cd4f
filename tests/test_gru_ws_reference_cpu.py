"""CPU checks of the weights-stationary GRU references (``unfused_reference.gru`` in mode '3xfp16' and 'bf16', and
``unfused_reference.gru_table``): an emulation of csrc/gru_ws.cu's arithmetic stays inside the per-element bound, and the same
bound rejects the kernel mistakes it exists to catch.

The emulation follows the kernel step by step: every operand split into fp16 (hi, lo') exactly as the fused write-out,
``pack_states`` and ``pack_gru_ws_kernel`` split it; exact products; one fp32 rounding per 16-wide k-step and accumulator (hi*hi
into the main one, hi*lo' then lo'*hi into the correction one); state chunks before aggregate chunks; fmaf(corr, 2^-11, main);
fp32 gate math in the kernel's order of adds.  bf16: bf16 operands, one fp32 accumulator, the fmaf blend, a bf16 store."""
import pytest
import torch

import fused_reference as FR
import unfused_reference as R
from helpers import split_f16

WORST = {}


def _split(x: torch.Tensor):
    hi, lo = split_f16(x)
    return hi.double(), lo.double()


def _accumulate(main, corr, x, w, bf16: bool, correction: bool = True):
    """Adds x [N, K] times w [M, K]^T into the fp32 accumulators in 16-wide k-steps."""
    if bf16:
        xh, wh = x.to(torch.bfloat16).double(), w.to(torch.bfloat16).double()
        xl = wl = None
    else:
        (xh, xl), (wh, wl) = _split(x), _split(w)
    for k in range(0, x.shape[1], 16):
        s = slice(k, k + 16)
        main = (main.double() + xh[:, s] @ wh[:, s].T).float()
        if not bf16 and correction:
            corr = (corr.double() + xh[:, s] @ wl[:, s].T).float()
            corr = (corr.double() + xl[:, s] @ wh[:, s].T).float()
    return main, corr


def _combine(main, corr):
    return (corr.double() * 2.0 ** -11 + main.double()).float()       # one fmaf


def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _emulate(h, w_hh, b_hh, bf16, x=None, w_ih=None, b_ih=None, gi=None, mutant=None):
    """The kernel's output rows (fp32, or bf16 as float) for the layer (x, w_ih, b_ih) or the state-only instance (gi, an fp32
    [N, 3H] table).  ``mutant``: 'hi_only', 'no_state_correction', 'swap_rz', 'b_ir_twice', 'wrong_row'."""
    N, H = h.shape
    z2 = lambda n: torch.zeros(N, n)
    rz, rz_c = z2(2 * H), z2(2 * H)
    hn, hn_c = z2(H), z2(H)
    corr = mutant != "hi_only"
    state_corr = corr and mutant != "no_state_correction"
    rz, rz_c = _accumulate(rz, rz_c, h, w_hh[:2 * H], bf16, state_corr)             # state chunks first
    hn, hn_c = _accumulate(hn, hn_c, h, w_hh[2 * H:], bf16, state_corr)
    if gi is None:
        rz, rz_c = _accumulate(rz, rz_c, x, w_ih[:2 * H], bf16, corr)               # then the aggregate chunks
        i_n, i_c = _accumulate(z2(H), z2(H), x, w_ih[2 * H:], bf16, corr)
        a_in = i_n if bf16 else _combine(i_n, i_c)
    a_rz = rz if bf16 else _combine(rz, rz_c)
    a_hn = hn if bf16 else _combine(hn, hn_c)
    a_r, a_z = a_rz[:, :H], a_rz[:, H:]
    if mutant == "swap_rz":
        a_r, a_z = a_z, a_r
    bh = b_hh.float()
    if gi is None:
        bi = b_ih.float()
        br, bz = bi[:H] + bh[:H], bi[H:2 * H] + bh[H:2 * H]                        # the packed bias vector
        r, z = torch.sigmoid(a_r + br), torch.sigmoid(a_z + bz)
        pre_n = a_in + bi[2 * H:]
    else:
        gr = gi[:, :H] + (b_ih[:H].float() if mutant == "b_ir_twice" else 0.0)
        r, z = torch.sigmoid((a_r + bh[:H]) + gr), torch.sigmoid((a_z + bh[H:2 * H]) + gi[:, H:2 * H])
        pre_n = gi[:, 2 * H:]
    hb = a_hn + bh[2 * H:]
    hv = torch.roll(h, 1, 0) if mutant == "wrong_row" else h
    if bf16:
        n = torch.tanh(_fma(r, hb, pre_n))
        return _fma(z, hv - n, n).to(torch.bfloat16).float()
    n = torch.tanh(pre_n + r * hb)
    return (1.0 - z) * n + z * hv


def _inputs(H, D, S, seed, rows=320):
    gen = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    cell = torch.nn.GRUCell(S or D, H)
    p = [t.detach() for t in (cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh)]
    h = torch.randn(rows, H, generator=gen) * 0.5
    h[:, :3] *= 2.0 ** -20                                      # lo' an fp16 subnormal
    h[5] = 0
    return gen, p, h


def _layer_case(H, D, bf16, seed=3):
    gen, (w_ih, w_hh, b_ih, b_hh), h = _inputs(H, D, None, seed)
    x = torch.randn(h.shape[0], D, generator=gen) * 4
    x[:, 7] *= 2.0 ** -18
    x[9] = 0
    if bf16:
        h, x = h.to(torch.bfloat16).float(), x.to(torch.bfloat16).float()
    ref, bound = R.gru(x.double(), None, h, w_ih, w_hh, b_ih, b_hh, "bf16" if bf16 else "3xfp16")
    return (lambda m=None: _emulate(h, w_hh, b_hh, bf16, x=x, w_ih=w_ih, b_ih=b_ih, mutant=m)), ref, bound


def _table_case(H, bf16, seed=4, S=96):
    gen, (w_ih, w_hh, b_ih, b_hh), h = _inputs(H, None, S, seed)
    G = 7
    g = (torch.randn(G, S, generator=gen) * 6).clamp(-30, 30)
    g[2] = 0
    gid = torch.randint(0, G, (h.shape[0],), generator=gen)
    gi64, e_gi = R.dense(g.double(), None, w_ih, b_ih, None, R.fp32_dense_mode(S, 3 * H))
    gi = torch.nn.functional.linear(g, w_ih, b_ih)                  # an fp32 table within e_gi
    FR.check_bound(gi, gi64, e_gi, "fp32 gi table")
    if bf16:
        h = h.to(torch.bfloat16).float()
    ref, bound = R.gru_table(gi64[gid], e_gi[gid], h, w_hh, b_hh, "bf16" if bf16 else "3xfp16")
    return (lambda m=None: _emulate(h, w_hh, b_hh, bf16, gi=gi[gid], b_ih=b_ih, mutant=m)), ref, bound


CASES = [("layer", H, False) for H in (64, 128)] + [("table", H, False) for H in (64, 192, 448)] + \
        [("layer", 128, True), ("table", 64, True), ("table", 448, True)]


@pytest.mark.parametrize("kind,H,bf16", CASES, ids=[f"{k}-H{H}-{'bf16' if b else 'fp32'}" for k, H, b in CASES])
def test_emulation_inside_the_bound_and_mutants_outside(kind, H, bf16):
    run, ref, bound = _layer_case(H, 128, bf16) if kind == "layer" else _table_case(H, bf16)
    what = f"{kind} H={H} {'bf16' if bf16 else 'fp32'}"
    ratio = FR.check_bound(run(), ref, bound, what)
    WORST[what] = ratio
    print(f"worst error/bound {what}: {ratio:.3f}")
    assert ratio > 1e-3, "the emulation is so far inside the bound that the bound says little"
    mutants = ["swap_rz", "wrong_row"] + ([] if bf16 else ["hi_only", "no_state_correction"]) + (["b_ir_twice"] if kind == "table" else [])
    for m in mutants:
        with pytest.raises(AssertionError):
            FR.check_bound(run(m), ref, bound, f"{what} mutant {m}")
    if bf16:     # one element 2 bf16 ulps off: pick the one with the tightest bound relative to its ulp
        got = run()
        ulp = FR._bf16_ulp(ref)
        i = int(torch.argmin(bound / ulp))
        moved = got.clone().reshape(-1)
        moved[i] += 2 * float(ulp.reshape(-1)[i])
        with pytest.raises(AssertionError):
            FR.check_bound(moved.reshape(got.shape), ref, bound, f"{what} 2 ulps")


def test_constants():
    assert R.gemm_constant("3xfp16", 128, 128) == FR.fp32_message_constant(128, 2)     # the messages' constant, S = 16
    assert R.gemm_constant("3xfp16", 448) == (14 + 56) * R.U                            # S = 28: past 2^-18
    assert R.gemm_constant("3xfp16", 448) > 2.0 ** -18


def test_bf16_blend_term_covers_a_saturated_z():
    """z -> 1 with |n| >> |h|: fmaf(z, h - n, n) rounds h - n at the size of n, which |(1 - z) n| and |z h| do not hold."""
    z = torch.tensor([[1 - 2.0 ** -9]], dtype=torch.float64)
    n = torch.tensor([[0.75]], dtype=torch.float64)
    h = torch.tensor([[2.0 ** -12]], dtype=torch.float64)
    zero = torch.zeros_like(z)
    c = torch.atanh(n)
    _, with_fma = R._gru_blend(z, zero, c, zero, h, "bf16")
    _, plain = R._gru_blend(z, zero, c, zero, h, "3xfp16")
    assert float(with_fma - FR._bf16_ulp(FR._bf16((1 - z) * n + z * h))) >= 1.02 * R.U * float(z * (h - n).abs())
    assert float(plain) < R.U * float(z * (h - n).abs())
