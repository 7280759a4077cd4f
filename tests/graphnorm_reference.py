"""Float restatement of the reference's GraphNorm (graphnorm.py:9-54), written from its semantics, the per-element error bound of the
native forward (DESIGN.md §3.9 / §4), and a float32 emulation of the kernels' order.

``layer_forward`` runs in the dtype of its inputs: in float32 it reproduces the reference's outputs and autograd gradients bit for bit
(the ops of the reference and of the ``torch_scatter`` stub's ``scatter_mean``, in the same order), in float64 it is the accuracy
reference.  ``emulate_forward`` repeats the kernels' float32 operations one by one (every kernel operation is an explicit
round-to-nearest intrinsic, and torch's float32 CPU ops round the same way), so the kernels must match it bit for bit.
"""
import torch

CHUNK = 32              # readout::CHUNK: rows per warp-chunk
U = 2.0 ** -24          # unit roundoff of fp32


def scatter_mean(src: torch.Tensor, index: torch.Tensor, G: int) -> torch.Tensor:
    """torch_scatter's scatter_mean over dim 0 as the stub computes it: a scatter_add into zeros, divided by the count clamped to 1."""
    out = torch.zeros(G, src.shape[1], dtype=src.dtype).scatter_add(0, index[:, None].expand_as(src), src)
    count = torch.zeros(G, dtype=src.dtype).scatter_add(0, index, torch.ones(index.shape[0], dtype=src.dtype))
    count = torch.where(count < 1, torch.ones_like(count), count)
    return out / count[:, None]


def layer_forward(x, n2g, gamma, alpha, bias, eps=1e-10, G=None):
    """The layer's forward: gamma, alpha, bias [1, D]; G (default max + 1) the graph count."""
    G = int(n2g.max()) + 1 if G is None else G
    mean = scatter_mean(x, n2g, G)
    shifted = x - alpha * mean[n2g]
    sigma_2 = scatter_mean(torch.pow(shifted, 2), n2g, G) + eps
    return gamma * shifted / torch.sqrt(sigma_2[n2g]) + bias


def chunks(n2g: torch.Tensor, G: int):
    """(order, counts, chunk start, length, graph, index within the graph): the plan's stable node order and its 32-row chunks."""
    order = torch.argsort(n2g, stable=True)
    counts = torch.bincount(n2g, minlength=G)
    row_ptr = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(counts, 0)])
    cs, cl, cg, cj = [], [], [], []
    for b in range(G):
        c = int(counts[b])
        for j, s in enumerate(range(0, c, CHUNK)):
            cs.append(int(row_ptr[b]) + s), cl.append(min(CHUNK, c - s)), cg.append(b), cj.append(j)
    t = lambda v: torch.tensor(v, dtype=torch.int64)  # noqa: E731
    return order, counts, t(cs), t(cl), t(cg), t(cj)


def emulate_forward(x, n2g, gamma, alpha, bias, eps=1e-10, G=None, drop_alpha=False):
    """(y in x's dtype, mean [G, D], rstd [G, D]) by the kernels' float32 operations in their order (DESIGN.md §3.9).
    ``drop_alpha``: sum s^2 without the (1 - alpha) factor (a mutant the bound must reject)."""
    G = int(n2g.max()) + 1 if G is None else G
    x32 = x.float()
    D = x32.shape[1]
    gamma, alpha, bias = (p.float().reshape(1, D) for p in (gamma, alpha, bias))
    order, counts, cs, cl, cg, cj = chunks(n2g, G)
    xs = x32[order]
    C = cs.numel()
    acc = torch.zeros(C, D)
    for t in range(CHUNK):
        m = cl > t
        acc[m] = acc[m] + xs[cs[m] + t]
    mc = acc / cl.float()[:, None]
    m2c = torch.zeros(C, D)
    for t in range(CHUNK):
        m = cl > t
        d = xs[cs[m] + t] - mc[m]
        m2c[m] = m2c[m] + d * d
    mu, m2 = torch.zeros(G, D), torch.zeros(G, D)
    na = torch.zeros(G, dtype=torch.int64)
    for j in range(int(cj.max()) + 1 if C else 0):
        sel = cj == j
        g, nb = cg[sel], cl[sel]
        if j == 0:
            mu[g], m2[g] = mc[sel], m2c[sel]
        else:
            n, fa, fb = (na[g] + nb).float()[:, None], na[g].float()[:, None], nb.float()[:, None]
            delta = mc[sel] - mu[g]
            mu[g] = mu[g] + delta * (fb / n)
            m2[g] = (m2[g] + m2c[sel]) + (delta * delta) * ((fa * fb) / n)
        na[g] += nb
    var = torch.where(counts[:, None] > 0, m2 / counts.float().clamp(min=1)[:, None], torch.zeros(()))
    t = mu if drop_alpha else (1.0 - alpha) * mu
    sigma2 = (var + t * t) + torch.tensor(eps, dtype=torch.float32)
    # torch's float32 CPU sqrt is not always correctly rounded; through float64 both roundings are (53 >= 2 * 24 + 2 bits)
    rstd = (1.0 / torch.sqrt(sigma2.double()).float().double()).float()
    s = (x32 - mu[n2g]) + t[n2g]
    y = s * (gamma * rstd[n2g]) + bias
    return y.to(x.dtype), mu, rstd


def bound(x, n2g, gamma, alpha, bias, eps=1e-10, G=None):
    """Per-element bound on |y_kernel - y_exact| for the fp32 forward (DESIGN.md §4), in float64.  Per graph and column, with
    M = max |x|, n nodes and k chunks:
        mean   E = (33 + 7k) u M        (the chunk's sequential sum of <= 32 rows and its division; each of the k - 1 Chan steps adds
                                          at most 3 roundings of |m_b - m_a| <= 2M and one of |mu| <= M)
        sigma2 |d| <= (40 + 3k) u sigma2 + 16 M E + 9 E^2 + 2|t| dt + dt^2,   t = (1 - alpha) mu,  dt = |1 - alpha| (E + 2u|mu|)
               (every M2 term is a sum of non-negative terms: n_c + 3 roundings in the chunk, 3 per Chan step; the between-chunk term
               delta^2 n_a n_b / n with |delta| <= 2M, n_b <= 32 and delta off by <= 2E; var, t^2 and the two additions)
        rstd   relative  er = |d| / (2 sigma2) + 2u   (sqrt and division)
        y      |dy| <= (|gamma| r (|alpha| E + u(|x - mu| + |s| + 2|t|) + |s| er) + 2u |gamma s r| + u |y|) * 1.01 + 1e-30
               (s = (x - mu) + t: mu enters with weight -1 + (1 - alpha) = -alpha)
    where s, r = 1 / sqrt(sigma2) and y are exact (float64)."""
    G = int(n2g.max()) + 1 if G is None else G
    x = x.double()
    D = x.shape[1]
    gamma, alpha, bias = (p.double().reshape(1, D) for p in (gamma, alpha, bias))
    counts = torch.bincount(n2g, minlength=G)
    k = ((counts + CHUNK - 1) // CHUNK).double()[:, None]
    M = torch.zeros(G, D, dtype=torch.float64).scatter_reduce(0, n2g[:, None].expand_as(x), x.abs(), "amax", include_self=True)
    mu = torch.zeros(G, D, dtype=torch.float64).index_add(0, n2g, x) / counts.clamp(min=1).double()[:, None]
    s = x - alpha * mu[n2g]
    var = torch.zeros(G, D, dtype=torch.float64).index_add(0, n2g, (x - mu[n2g]) ** 2) / counts.clamp(min=1).double()[:, None]
    t = (1.0 - alpha) * mu
    sigma2 = var + t * t + eps
    E = (33 + 7 * k) * U * M
    dt = (1.0 - alpha).abs() * (E + 2 * U * mu.abs())
    d_sigma2 = (40 + 3 * k) * U * sigma2 + 16 * M * E + 9 * E * E + 2 * t.abs() * dt + dt * dt
    er = d_sigma2 / (2 * sigma2) + 2 * U
    r = 1.0 / torch.sqrt(sigma2)
    y = gamma * s * r[n2g] + bias
    g_r = gamma.abs() * r[n2g]
    out = g_r * (alpha.abs() * E[n2g] + U * ((x - mu[n2g]).abs() + s.abs() + 2 * t[n2g].abs()) + s.abs() * er[n2g]) + 2 * U * (g_r * s).abs() + U * y.abs()
    return out * 1.01 + 1e-30
