"""Float restatements of the reference's PnaMessageAggregation (pna_aggregation.py:27-56), the native kernel's float32 operation order,
the backward formula, and the bound for the log-scaled blocks (DESIGN.md §3.10).

``emulate_forward`` repeats the forward kernel's float32 operations: sums in edge order from 0 (``scatter_add_``, one rounding per
edge, as the kernel adds), ``den = fl(k) + fl(1e-5)``, strict-compare max / min with the first occurrence winning, the std terms
``relu(m * m - mean * mean) + 1e-10`` summed in edge order, a correctly rounded sqrt.  Every one of these is a correctly rounded IEEE
operation on both sides, so the kernel must match the ``S = [sum | mean | max | min | std]`` columns bit for bit.  (torch's float32
CPU sqrt is not always correctly rounded: the reference's own std can be one ulp away.)  ``p1`` uses ``log``,
which torch's CPU and CUDA's ``logf`` may round differently by an ulp: the scaled blocks are compared under ``scaled_bound``.

``layer_forward`` is the reference's forward as differentiable torch ops in the dtype of its input (float32: the reference's own
numbers; float64: the accuracy reference), and ``emulate_backward`` states the kernel's gradient formula in its order.
"""
import torch

U = 2.0 ** -24          # unit roundoff of fp32
FLT_MAX = torch.finfo(torch.float32).max
MUTANTS = ("clamped_count", "fmaxf_relu", "last_tie")


def plan(targets: torch.Tensor, n: int):
    """(stable target order = the kernel's walk order, in-degree per target)."""
    return torch.argsort(targets, stable=True), torch.bincount(targets, minlength=n)


def extreme(x: torch.Tensor, targets: torch.Tensor, n: int, is_max: bool, last_tie: bool = False):
    """torch_scatter's max / min over dim 0: strict compare from -FLT_MAX / FLT_MAX, first occurrence wins ties (``last_tie``: the
    last one, a mutant), NaN never wins, 0 and arg E where nothing won.  (values, arg int64)."""
    E, D = x.shape
    init = -FLT_MAX if is_max else FLT_MAX
    idx = targets[:, None].expand(E, D)
    eligible = ~torch.isnan(x) & ((x > init) if is_max else (x < init))
    clean = torch.where(eligible, x, torch.full_like(x, init))
    best = torch.full((n, D), init, dtype=x.dtype).scatter_reduce(0, idx, clean, "amax" if is_max else "amin", include_self=True)
    winners = eligible & (clean == best.gather(0, idx))
    ids = torch.arange(E, dtype=torch.int64)[:, None].expand(E, D)
    if last_tie:
        arg = torch.full((n, D), -1, dtype=torch.int64).scatter_reduce(0, idx, torch.where(winners, ids, -1), "amax", include_self=True)
        arg = torch.where(arg < 0, torch.full_like(arg, E), arg)
    else:
        arg = torch.full((n, D), E, dtype=torch.int64).scatter_reduce(0, idx, torch.where(winners, ids, E), "amin", include_self=True)
    return torch.where(arg == E, torch.zeros_like(best), best), arg


def scalers(counts: torch.Tensor, delta: float, dtype=torch.float32):
    """(den, p1, m1) [n, 1]: fl(k) + fl(1e-5), log(fl(k) + 1) / fl(delta), 1 / (p1 + fl(1e-3)) in ``dtype``."""
    k = counts.to(dtype)[:, None]
    den = k + torch.tensor(1e-5, dtype=dtype)
    p1 = torch.log(k + 1) / torch.tensor(delta, dtype=dtype)
    return den, p1, 1.0 / (p1 + torch.tensor(1e-3, dtype=dtype))


def emulate_forward(messages: torch.Tensor, targets: torch.Tensor, n: int, delta: float, mutant: str = None):
    """(out [n, 15 D] fp32, arg_max, arg_min [n, D] int64) by the forward kernel's float32 operations.  ``messages``: fp32 or bf16.
    ``mutant``: one of MUTANTS -- the mean over a clamped count, an fmaxf relu (NaN lost), the last occurrence winning ties."""
    x = messages.float()
    E, D = x.shape
    _, counts = plan(targets, n)
    idx = targets[:, None].expand(E, D)
    total = torch.zeros(n, D).scatter_add_(0, idx, x)
    den, p1, m1 = scalers(counts, delta)
    if mutant == "clamped_count":
        den = counts.clamp(min=1).float()[:, None]
    mean = total / den
    mx, amx = extreme(x, targets, n, True, mutant == "last_tie")
    mn, amn = extreme(x, targets, n, False, mutant == "last_tie")
    d = x * x - (mean * mean)[targets]
    r = torch.where(d > 0, d, torch.zeros_like(d)) if mutant == "fmaxf_relu" else torch.relu(d)
    comp = r + torch.tensor(1e-10, dtype=torch.float32)
    # through float64 the square root is correctly rounded (53 >= 2 * 24 + 2 bits), as the kernel's __fsqrt_rn
    std = torch.sqrt(torch.zeros(n, D).scatter_add_(0, idx, comp).double()).float()
    S = torch.cat([total, mean, mx, mn, std], dim=1).to(messages.dtype).float()
    return torch.cat([S, S * p1, S * m1], dim=1), amx, amn


def layer_forward(messages: torch.Tensor, targets: torch.Tensor, n: int, delta: float) -> torch.Tensor:
    """The reference's forward as differentiable torch ops in ``messages.dtype`` (fp32 or fp64); max / min route their gradient to
    the first winning edge, as torch_scatter's arg does."""
    x = messages
    E, D = x.shape
    dt = x.dtype
    _, counts = plan(targets, n)
    idx = targets[:, None].expand(E, D)
    total = torch.zeros(n, D, dtype=dt).scatter_add(0, idx, x)
    den, p1, m1 = scalers(counts, delta, dt)
    mean = total / den
    stats = [total, mean]
    for is_max in (True, False):
        _, arg = extreme(x.detach().float() if dt == torch.float32 else x.detach(), targets, n, is_max)
        padded = torch.cat([x, torch.zeros(1, D, dtype=dt)], dim=0)
        stats.append(padded.gather(0, arg))
    comp = torch.relu(x.pow(2) - mean[targets].pow(2)) + torch.tensor(1e-10, dtype=dt)
    stats.append(torch.sqrt(torch.zeros(n, D, dtype=dt).scatter_add(0, idx, comp)))
    S = torch.cat(stats, dim=1)
    return torch.cat([S, S * p1, S * m1], dim=1)


def emulate_backward(messages: torch.Tensor, targets: torch.Tensor, n: int, delta: float, out: torch.Tensor, arg_max: torch.Tensor,
                     arg_min: torch.Tensor, d_out: torch.Tensor, drop_mean_term: bool = False) -> torch.Tensor:
    """d messages [E, D] by the backward kernel's formula and float32 order (DESIGN.md §3.10):
        dS = (G0 + G1 p1) + G2 m1,  dQ = dS_std / (2 std),  C_v = #{e -> v : fl(m_e^2) - fl(mean^2) > 0} per column,
        d m_e = ((((dS_sum + (dS_mean - ((2 mean) dQ) C_v) / den) + [e = argmax] dS_max) + [e = argmin] dS_min) + [m_e on the positive
                side] (2 m_e) dQ)
    ``drop_mean_term``: without the ``(2 mean) dQ C_v`` term (a mutant: the std's dependence on the mean forgotten)."""
    x = messages.float()
    E, D = x.shape
    _, counts = plan(targets, n)
    den, p1, m1 = scalers(counts, delta)
    G = d_out.float()
    dS = [(G[:, b * D:(b + 1) * D] + G[:, (5 + b) * D:(6 + b) * D] * p1) + G[:, (10 + b) * D:(11 + b) * D] * m1 for b in range(5)]
    mu, std = out[:, D:2 * D], out[:, 4 * D:5 * D]
    dQ = dS[4] / (2.0 * std)
    q = (x * x - (mu * mu)[targets]) > 0
    C = torch.zeros(n, D).index_add_(0, targets, q.float())
    t = ((2.0 * mu) * dQ) * C
    base = dS[0] + ((dS[1] if drop_mean_term else dS[1] - t) / den)
    e = torch.arange(E)[:, None]
    g = base[targets]
    g = torch.where(e == arg_max[targets], g + dS[2][targets], g)
    g = torch.where(e == arg_min[targets], g + dS[3][targets], g)
    return torch.where(q, g + (2.0 * x) * dQ[targets], g)


def scaled_bound(S_ref: torch.Tensor, D: int) -> torch.Tensor:
    """Per-element bound on |out_kernel - out_ref| for out [n, 15 D] from the reference's fp32 output (0 on the S columns): p1 differs
    by the two logs' roundings (<= 1 ulp each, 4u relative), the divisions by delta and the products (u each): 16 u |out| covers p1,
    m1 = 1 / (p1 + 1e-3) (at most p1's relative error plus two roundings), the scaled blocks, and the reference's std being one ulp
    (2u) away."""
    b = 16 * U * S_ref.double().abs()
    b[:, :5 * D] = 0.0
    return b
