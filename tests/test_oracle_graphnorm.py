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
