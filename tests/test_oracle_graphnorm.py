"""GraphNorm on the CPU: the float restatement (graphnorm_reference.py) against the reference's own outputs and gradients
(tests/golden/graphnorm_*.npz, written by tests/golden/generate_graphnorm_golden.py), the kernel's error bound against the float32
emulation of the kernel order, the native class's signature and state_dict keys, and the overlay's opt-in binding."""
import inspect
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import graphnorm_reference as GR
from oracle.refimport import reference_available

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["graphnorm_d32", "graphnorm_d64", "graphnorm_d128", "graphnorm_d256"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    f = {k: torch.from_numpy(z[k]) for k in z.files}
    f["sd"] = {k[4:]: v for k, v in f.items() if k.startswith("sd::")}
    return f


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_reference_graphnorm_and_its_gradients(name):
    f = load(name)
    x = f["x"].clone().requires_grad_(True)
    params = {n: f["sd"][n].clone().requires_grad_(True) for n in ("gamma", "alpha", "bias")}
    out = GR.layer_forward(x, f["n2g"], params["gamma"], params["alpha"], params["bias"])
    assert torch.equal(out.detach(), f["out"]), f"{name}: restatement differs from the reference's output"
    out.backward(f["dy"])
    assert torch.equal(x.grad, f["d_x"]), f"{name}: d x"
    for n, p in params.items():
        assert torch.equal(p.grad, f["d_" + n]), f"{name}: d {n}"


def test_restatement_reproduces_reference_on_bf16_rounded_states():
    f = load("graphnorm_d128_bf16")
    sd = f["sd"]
    assert torch.equal(GR.layer_forward(f["x"], f["n2g"], sd["gamma"], sd["alpha"], sd["bias"]), f["out_fp32_rounded_inputs"])
    assert torch.equal(f["x"].to(torch.bfloat16).float(), f["x"]), "the states are bf16 values"


def test_fixture_graph_maps_have_the_intended_structure():
    for name in NAMES:
        f = load(name)
        counts = torch.bincount(f["n2g"])
        assert (counts == 0).any() and (counts == 1).any() and bool((counts > 2 * GR.CHUNK).any()), name
        assert not bool((f["n2g"][1:] >= f["n2g"][:-1]).all()), f"{name}: unsorted"
        sd = f["sd"]
        assert not torch.equal(sd["gamma"], torch.ones_like(sd["gamma"])) and not torch.equal(sd["alpha"], torch.ones_like(sd["alpha"]))
        assert bool((sd["bias"] != 0).all())


@pytest.mark.parametrize("name", NAMES)
def test_kernel_order_emulation_is_inside_the_bound_and_a_dropped_alpha_is_not(name):
    f = load(name)
    sd, n2g = f["sd"], f["n2g"]
    exact = GR.layer_forward(f["x"].double(), n2g, sd["gamma"].double(), sd["alpha"].double(), sd["bias"].double())
    bnd = GR.bound(f["x"], n2g, sd["gamma"], sd["alpha"], sd["bias"])
    y, _, _ = GR.emulate_forward(f["x"], n2g, sd["gamma"], sd["alpha"], sd["bias"])
    err = (y.double() - exact).abs()
    assert bool((err <= bnd).all()), f"{name}: emulated kernel order exceeds the bound (worst ratio {float((err / bnd).max()):.2f})"
    mutant, _, _ = GR.emulate_forward(f["x"], n2g, sd["gamma"], sd["alpha"], sd["bias"], drop_alpha=True)
    assert bool(((mutant.double() - exact).abs() > bnd).any()), f"{name}: the bound does not catch a dropped alpha"


def test_emulation_gives_bias_exactly_for_one_node_graphs_with_alpha_one():
    gen = torch.Generator().manual_seed(1)
    n2g = torch.tensor([0, 1, 1, 2, 3, 3, 3])
    x = torch.randn(7, 32, generator=gen) * 10
    bias = torch.randn(1, 32, generator=gen)
    y, mu, _ = GR.emulate_forward(x, n2g, torch.randn(1, 32, generator=gen), torch.ones(1, 32), bias)
    assert torch.equal(y[0], bias[0]) and torch.equal(y[3], bias[0]) and torch.equal(mu[0], x[0])


def test_native_class_has_reference_signature_parameters_and_keys():
    import ptgnn_b200 as P

    torch.manual_seed(0)
    m = P.GraphNorm(64)
    assert [n for n, _ in m.named_parameters()] == ["gamma", "alpha", "bias"]
    assert m.input_state_dimension == 64 and m.output_state_dimension == 64
    assert [tuple(p.shape) for p in m.parameters()] == [(1, 64)] * 3
    if not reference_available():
        pytest.skip("reference package not available")
    from oracle.refimport import import_reference

    import_reference()
    from ptgnn.neuralmodels.gnn.messagepassing.graphnorm import GraphNorm as Ref

    assert inspect.signature(Ref.__init__) == inspect.signature(P.GraphNorm.__init__)
    torch.manual_seed(0)
    ref = Ref(64)
    assert list(ref.state_dict()) == list(m.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(ref.state_dict().values(), m.state_dict().values())), "same seed, same values"
    m.load_state_dict(ref.state_dict(), strict=True)


@pytest.mark.skipif(not reference_available(), reason="reference package not available")
def test_overlay_binds_the_native_graphnorm_only_when_asked():
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from oracle.refimport import import_reference\nimport_reference()\n"
        "import ptgnn_b200 as P, ptgnn_b200.overlay as ov\n"
        "MOD = 'ptgnn.neuralmodels.gnn.messagepassing.graphnorm'\n"
        "import importlib\nref = importlib.import_module(MOD).GraphNorm\n"
        "r = ov.install(force_torch_scatter=True)\n"
        "assert r['graphnorm'] is False and importlib.import_module(MOD).GraphNorm is ref\n"
        "ov.uninstall()\n"
        "r = ov.install(force_torch_scatter=True, native_graphnorm=True)\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.graphnorm import GraphNorm as M\n"
        "assert r['graphnorm'] is True and M is P.GraphNorm\n"
        "ov.uninstall()\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.graphnorm import GraphNorm as M2\n"
        "assert M2 is ref\nprint('GRAPHNORM-OVERLAY-OK')\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "GRAPHNORM-OVERLAY-OK" in r.stdout, r.stdout + r.stderr[-3000:]


def test_overlay_pre_seeds_the_native_graphnorm_before_the_reference_module_is_imported():
    if not reference_available():
        pytest.skip("reference package not available")
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from oracle.refimport import import_reference\nimport_reference()\n"
        "import ptgnn_b200 as P, ptgnn_b200.overlay as ov\n"
        "assert 'ptgnn.neuralmodels.gnn.messagepassing.graphnorm' not in sys.modules\n"
        "ov.install(force_torch_scatter=True, native_graphnorm=True)\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.graphnorm import GraphNorm as M\n"
        "assert M is P.GraphNorm\nprint('GRAPHNORM-PRESEED-OK')\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "GRAPHNORM-PRESEED-OK" in r.stdout, r.stdout + r.stderr[-3000:]


# ---- backward ---------------------------------------------------------------------------------------------------------------
EPS32 = float(torch.tensor(1e-10, dtype=torch.float32))     # the eps the kernels receive (a float)


def _bwd_case(counts, D, alpha_value, seed, equal_rows=()):
    """(x, dy, n2g, G, gamma, alpha) on a shuffled map with the given graph sizes; the graphs in ``equal_rows`` have all rows equal."""
    gen = torch.Generator().manual_seed(seed)
    n2g = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    n2g = n2g[torch.randperm(n2g.numel(), generator=gen)]
    G = len(counts)
    x = torch.randn(n2g.numel(), D, generator=gen) * 2.0 + torch.randn(G, D, generator=gen)[n2g] * 3.0
    for g in equal_rows:
        x[n2g == g] = torch.randn(D, generator=gen) * 3.0
    dy = torch.randn(n2g.numel(), D, generator=gen)
    gamma = 1.0 + 0.5 * torch.randn(1, D, generator=gen)
    alpha = torch.full((1, D), alpha_value) if alpha_value is not None else torch.rand(1, D, generator=gen) * 1.5
    return x, dy, n2g, G, gamma, alpha


def _exact_stats(x64, n2g, alpha64, eps, G):
    mean = GR.scatter_mean(x64, n2g, G)
    sigma2 = GR.scatter_mean((x64 - alpha64 * mean[n2g]) ** 2, n2g, G) + eps
    return mean, 1.0 / torch.sqrt(sigma2)


BWD_CASES = {"sizes_alpha_rand": ([1, 31, 32, 33, 0, 1, 64, 65, 200], None, ()), "alpha0": ([1, 5, 33, 0, 70], 0.0, ()),
             "alpha_half": ([1, 5, 33, 0, 70], 0.5, (1,)), "alpha1": ([1, 5, 33, 0, 70], 1.0, (2,)),
             "alpha1.7": ([1, 5, 33, 0, 70], 1.7, (1, 4))}


@pytest.mark.parametrize("eps", [EPS32, 0.25])
@pytest.mark.parametrize("case", list(BWD_CASES))
def test_backward_formula_equals_autograd_through_the_float64_forward(case, eps):
    """With the exact float64 mean and rstd, backward_formula is the gradient of layer_forward (one-node graphs and graphs of equal
    rows included).  Relative to each gradient's largest element: autograd itself cancels in 1 - x^2 on a one-node graph, where the
    formula does not.  eps = 0.25 makes the one-node gradient large enough to be pinned too."""
    counts, a, equal = BWD_CASES[case]
    x, dy, n2g, G, gamma, alpha = _bwd_case(counts, 64, a, len(counts) + int(10 * (a or 0)), equal)
    x64, g64, a64, b64 = (t.double().requires_grad_(True) for t in (x, gamma, alpha, torch.zeros(1, 64)))
    GR.layer_forward(x64, n2g, g64, a64, b64, eps=eps, G=G).backward(dy.double())
    mean, rstd = _exact_stats(x64.detach(), n2g, alpha.double(), eps, G)
    got = GR.backward_formula(x, dy, n2g, mean, rstd, gamma, alpha, eps=eps, G=G)
    for name, g, ref in zip(("dx", "d gamma", "d alpha", "d beta"), got, (x64.grad, g64.grad[0], a64.grad[0], b64.grad[0])):
        err = float((g - ref).abs().max() / ref.abs().max())
        assert err <= 1e-12, f"{case} eps={eps} {name}: {err:.2e}"
    one = torch.bincount(n2g, minlength=G) == 1
    rows = one[n2g]
    if eps == 0.25 and a != 1.0:
        rel = ((got[0][rows] - x64.grad[rows]).abs() / x64.grad[rows].abs()).max()
        assert float(rel) <= 1e-12, f"{case}: one-node rows {float(rel):.2e}"


def _emulated_pair(counts, D, a, seed, equal=()):
    x, dy, n2g, G, gamma, alpha = _bwd_case(counts, D, a, seed, equal)
    _, mean, rstd = GR.emulate_forward(x, n2g, gamma, alpha, torch.zeros(1, D), G=G)
    return x, dy, n2g, G, gamma, alpha, mean, rstd


@pytest.mark.parametrize("case", list(BWD_CASES))
def test_backward_emulation_is_inside_the_bound_and_the_mutants_are_not(case):
    """The float32 emulation of the backward kernels' order against backward_formula on the forward's float32 statistics, under
    backward_bound; the one-node branch removed (the general formula on count 1) and c2 without alpha fall outside it."""
    counts, a, equal = BWD_CASES[case]
    args = _emulated_pair(counts, 64, a, 3 * len(counts), equal)
    x, dy, n2g, G, gamma, alpha, mean, rstd = args
    ref = GR.backward_formula(*args[:2], n2g, mean, rstd, gamma, alpha, eps=1e-10, G=G)
    bnd = GR.backward_bound(*args[:2], n2g, mean, rstd, gamma, alpha, eps=1e-10, G=G)

    def over(got):
        return [float(((g.double() - r).abs() / b).max()) for g, r, b in zip(got, ref, bnd)]

    worst = over(GR.emulate_backward(x, dy, n2g, mean, rstd, gamma, alpha, G=G))
    assert max(worst) <= 1.0, f"{case}: emulated kernel order exceeds the bound (dx, dgamma, dalpha, dbeta ratios {worst})"
    if a != 1.0:            # alpha = 1: s = 0 on a one-node graph, where both branches give exactly 0
        assert over(GR.emulate_backward(x, dy, n2g, mean, rstd, gamma, alpha, G=G, mutant="no_one_node_branch"))[0] > 1.0, case
    if a not in (0.0, 1.0):  # alpha S = S at alpha = 1, and c2 = 0 at alpha = 0
        assert max(over(GR.emulate_backward(x, dy, n2g, mean, rstd, gamma, alpha, G=G, mutant="c2_without_alpha"))) > 1.0, case
