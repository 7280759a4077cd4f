"""Float restatement of the reference's GraphNorm (graphnorm.py:9-54), written from its semantics, the per-element error bound of the
native forward (DESIGN.md §3.9 / §4), and a float32 emulation of the kernels' order.

``layer_forward`` runs in the dtype of its inputs: in float32 it reproduces the reference's outputs and autograd gradients bit for bit
(the ops of the reference and of the ``torch_scatter`` stub's ``scatter_mean``, in the same order), in float64 it is the accuracy
reference.  ``emulate_forward`` repeats the kernels' float32 operations one by one (every kernel operation is an explicit
round-to-nearest intrinsic, and torch's float32 CPU ops round the same way), so the kernels must match it bit for bit.
"""
import torch

CHUNK = 32              # pergraph::CHUNK: rows per warp-chunk
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


def gamma_n(n):
    """gamma_n = n u / (1 - n u): the relative error bound of n roundings (tensor or number)."""
    return n * U / (1 - n * U)


def _bwd_inputs(x, dy, n2g, mean, rstd, gamma, alpha, eps, G):
    G = int(n2g.max()) + 1 if G is None else G
    x, dy = x.double(), dy.double()
    D = x.shape[1]
    gamma, alpha = (p.double().reshape(1, D) for p in (gamma, alpha))
    counts = torch.bincount(n2g, minlength=G)
    return x, dy, mean.double(), rstd.double(), gamma, alpha, float(torch.tensor(eps, dtype=torch.float32)), counts, G, D


def backward_formula(x, dy, n2g, mean, rstd, gamma, alpha, eps=1e-10, G=None):
    """(dx [N, D], d gamma [D], d alpha [D], d beta [D]) in float64 from exactly the kernels' inputs: x, dy, the forward's mean and
    rstd [G, D], gamma, alpha and eps as float32 (the kernel receives eps as a float).  Per graph and column, with x^ = s rstd,
    s = (x - mu) + (1 - alpha) mu, k = gamma rstd, A = sum dy, B = sum dy x^ and n rows:
        dL/ds_i = k (dy_i - x^_i B / n),   S = sum_i dL/ds_i = k (A - (1 - alpha) mu rstd B),   dx_i = dL/ds_i - alpha S / n
    and for a one-node graph, where 1 - x^2 = eps rstd^2 exactly: dL/ds = k eps rstd^2 dy, S = k eps rstd^2 A, dx = (1 - alpha) dL/ds.
    d gamma = sum_g B, d beta = sum_g A, d alpha = -sum_g mu S.  With the exact float64 mean and rstd this is the gradient."""
    x, dy, mu, r, gamma, alpha, eps, counts, G, D = _bwd_inputs(x, dy, n2g, mean, rstd, gamma, alpha, eps, G)
    s = (x - mu[n2g]) + (1.0 - alpha) * mu[n2g]
    xh = s * r[n2g]
    A = torch.zeros(G, D, dtype=torch.float64).index_add(0, n2g, dy)
    B = torch.zeros(G, D, dtype=torch.float64).index_add(0, n2g, dy * xh)
    n = counts.double().clamp(min=1)[:, None]
    k = gamma * r
    one = (counts == 1)[:, None]
    ke = k * eps * r * r
    S = torch.where(one, ke * A, k * (A - (1.0 - alpha) * mu * r * B))
    dls = torch.where(one[n2g], ke[n2g] * dy, k[n2g] * (dy - xh * (B / n)[n2g]))
    dx = dls - (alpha * S / n)[n2g]
    return dx, B.sum(0), -(mu * S).sum(0), A.sum(0)


def backward_bound(x, dy, n2g, mean, rstd, gamma, alpha, eps=1e-10, G=None):
    """Per-element bounds (dx [N, D], d gamma, d alpha, d beta [D]) on |kernel - backward_formula| for the fp32 backward (DESIGN.md
    §4), in float64, from the §3.9 order.  Every term is a sum of absolute values, so cancellation in dy - x^ c1, in A - P B or in
    1 - x^2 is covered.  With u = 2^-24, gamma_n = n u / (1 - n u), k chunks in the graph and t = (1 - alpha) mu, P = t rstd:
        x^     e_x = rstd (u |x - mu| + u |s| + 3u |t|) + u |x^|           (x - mu, t's two roundings, + t, * rstd)
        A      e_A = gamma_{32+k} sum |dy|                                 (the chunk's chain of <= 32 rows, then k chunk additions)
        B      e_B = sum |dy| e_x + gamma_{33+k} sum |dy x^|               (the product, then the same chains)
        S      e_S = |k| (e_A + |P| e_B + 4u |P B| + u (|A| + |P B|)) + 2u |k (A - P B)|   (P: 3 roundings, P B and the difference
                                                                                  one each; k = gamma rstd and k (A - P B) one each)
        c1     e_1 = (e_B + u |B|) / n,   c2  e_2 = (|alpha| e_S + 2u |alpha S|) / n
        dx     |d| <= |k| (|x^| e_1 + |c1| e_x + u |x^ c1| + u (|dy| + |x^ c1|)) + u |k| |dy - x^ c1| + u |k (dy - x^ c1)| + e_2
                      + u (|k (dy - x^ c1)| + |c2|)
    A one-node graph (1 - x^2 = eps rstd^2, no c1 or c2): k' = k eps rstd^2 (1 - alpha) carries 6 roundings, so
        dx  |d| <= 7u |k' dy|,   S  e_S = |k eps rstd^2| (e_A + 5u |A|)
    The parameter sums over G graphs in order: d beta  sum_g e_A + gamma_G sum_g |A|,  d gamma  sum_g e_B + gamma_G sum_g |B|,
    d alpha  sum_g (|mu| e_S + u |mu S|) + gamma_G sum_g |mu S|.  Second-order terms: 1 % slack, plus 1e-37 absolute."""
    x, dy, mu, r, gamma, alpha, eps, counts, G, D = _bwd_inputs(x, dy, n2g, mean, rstd, gamma, alpha, eps, G)
    mun, rn = mu[n2g], r[n2g]
    t = (1.0 - alpha) * mu
    s = (x - mun) + t[n2g]
    xh = s * rn
    e_x = rn * (U * (x - mun).abs() + U * s.abs() + 3 * U * t[n2g].abs()) + U * xh.abs()
    chunks = ((counts + CHUNK - 1) // CHUNK).double()[:, None]
    gsum = lambda v: torch.zeros(G, D, dtype=torch.float64).index_add(0, n2g, v)  # noqa: E731
    A, B = gsum(dy), gsum(dy * xh)
    e_A = gamma_n(32 + chunks) * gsum(dy.abs())
    e_B = gsum(dy.abs() * e_x) + gamma_n(33 + chunks) * gsum((dy * xh).abs())
    k = gamma * r
    P = t * r
    W = A - P * B
    e_S = k.abs() * (e_A + P.abs() * e_B + 4 * U * (P * B).abs() + U * (A.abs() + (P * B).abs())) + 2 * U * (k * W).abs()
    S = k * W
    n = counts.double().clamp(min=1)[:, None]
    c1 = B / n
    e_1 = (e_B + U * B.abs()) / n
    e_2 = (alpha.abs() * e_S + 2 * U * (alpha * S).abs()) / n
    kn, c1n = k[n2g], c1[n2g]
    d1 = dy - xh * c1n
    b_dx = (kn.abs() * (xh.abs() * e_1[n2g] + c1n.abs() * e_x + U * (xh * c1n).abs() + U * (dy.abs() + (xh * c1n).abs()))
            + 2 * U * (kn * d1).abs() + e_2[n2g] + U * ((kn * d1).abs() + (alpha * S / n)[n2g].abs()))
    one = (counts == 1)[:, None]
    ke = k * eps * r * r
    b_dx = torch.where(one[n2g], 7 * U * ((ke * (1.0 - alpha))[n2g] * dy).abs(), b_dx)
    e_S = torch.where(one, ke.abs() * (e_A + 5 * U * A.abs()), e_S)
    S = torch.where(one, ke * A, S)
    gG = gamma_n(G)
    b_gamma = e_B.sum(0) + gG * B.abs().sum(0)
    b_beta = e_A.sum(0) + gG * A.abs().sum(0)
    b_alpha = (mu.abs() * e_S + U * (mu * S).abs()).sum(0) + gG * (mu * S).abs().sum(0)
    return tuple(b * 1.01 + 1e-37 for b in (b_dx, b_gamma, b_alpha, b_beta))


def emulate_backward(x, dy, n2g, mean, rstd, gamma, alpha, eps=1e-10, G=None, mutant=None):
    """(dx [N, D], d gamma [D], d alpha [D], d beta [D]) by the backward kernels' float32 operations in their order (DESIGN.md §3.9),
    bit for bit: A_c, B_c over each chunk's rows in node order, the chunk sums in chunk order from 0, k, c1, c2 and S per graph (the
    one-node branch included), dx, and the parameter sums over the graphs in order from 0.  ``mutant`` (the bound must reject each):
    "no_one_node_branch" runs the general formula on one-node graphs, "c2_without_alpha" drops alpha from c2."""
    G = int(n2g.max()) + 1 if G is None else G
    x32, dy32 = x.float(), dy.float()
    D = x32.shape[1]
    gamma, alpha = (p.float().reshape(1, D) for p in (gamma, alpha))
    mu, r = mean.float(), rstd.float()
    eps32 = torch.tensor(eps, dtype=torch.float32)
    order, counts, cs, cl, cg, cj = chunks(n2g, G)
    t = (1.0 - alpha) * mu
    xh = ((x32 - mu[n2g]) + t[n2g]) * r[n2g]
    xs, gs, hs = x32[order], dy32[order], xh[order]
    C = cs.numel()
    Ac, Bc = torch.zeros(C, D), torch.zeros(C, D)
    for i in range(CHUNK):
        m = cl > i
        Ac[m] = Ac[m] + gs[cs[m] + i]
        Bc[m] = Bc[m] + gs[cs[m] + i] * hs[cs[m] + i]
    A, B = torch.zeros(G, D), torch.zeros(G, D)
    for j in range(int(cj.max()) + 1 if C else 0):
        sel = cj == j
        A[cg[sel]] = A[cg[sel]] + Ac[sel]
        B[cg[sel]] = B[cg[sel]] + Bc[sel]
    k = gamma * r
    S = k * (A - (t * r) * B)
    n = counts.float()[:, None]
    has = counts[:, None] > 0
    c1 = torch.where(has, B / n.clamp(min=1), torch.zeros(()))
    aS = S if mutant == "c2_without_alpha" else alpha * S
    c2 = torch.where(has, aS / n.clamp(min=1), torch.zeros(()))
    coef_k = k
    if mutant != "no_one_node_branch":
        one = (counts == 1)[:, None]
        ke = k * (eps32 * (r * r))
        coef_k = torch.where(one, ke * (1.0 - alpha), k)
        c1 = torch.where(one, torch.zeros(()), c1)
        c2 = torch.where(one, torch.zeros(()), c2)
        S = torch.where(one, ke * A, S)
    dx = coef_k[n2g] * (dy32 - xh * c1[n2g]) - c2[n2g]
    sg, sb, sa = torch.zeros(D), torch.zeros(D), torch.zeros(D)
    for b in range(G):
        sb = sb + A[b]
        sg = sg + B[b]
        sa = sa + mu[b] * S[b]
    return dx, sg, -sa, sb
