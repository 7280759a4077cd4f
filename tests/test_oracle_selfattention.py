"""MultiHeadSelfAttentionMessagePassing on the CPU: the float restatement (selfattention_reference.py) against the reference's own
outputs (tests/golden/selfatt_*.npz, written by tests/golden/generate_selfattention_golden.py), the kernel's error bound against a
float32 emulation of the kernel order, the native class's signature and state_dict keys, and the overlay's opt-in binding."""
import inspect
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import selfattention_reference as SR
from oracle.refimport import reference_available

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["selfatt_h1_d16", "selfatt_h3_d32", "selfatt_h8_d16", "selfatt_h4_dk64_dv32", "selfatt_h2_dk128_dv64"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    f = {k: int(z[k]) if z[k].ndim == 0 else torch.from_numpy(z[k]) for k in z.files}
    f["sd"] = {k[4:]: v for k, v in f.items() if k.startswith("sd::")}
    return f


def restated(f, x=None):
    return SR.layer_forward(f["x"] if x is None else x, f["n2g"], f["sd"], f["heads"], f["dk"], f["max_num_nodes"])


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_reference_selfattention(name):
    f = load(name)
    assert torch.equal(restated(f), f["out"]), f"{name}: restatement differs from the reference's output"


def test_restatement_reproduces_reference_autocast():
    f = load("selfatt_h8_d16_bf16ac")
    with torch.autocast("cpu", dtype=torch.bfloat16):
        out = restated(f)
    # CPU bf16 GEMMs round differently from one instruction set to another: the autocast output is pinned at bf16 resolution
    ref = f["out_autocast"]
    assert float(((out.float() - ref).abs() / ref.abs().clamp(min=1)).max()) <= 2 ** -6
    assert torch.equal(restated(f), f["out_fp32_rounded_inputs"])


def test_fixture_graph_maps_have_the_intended_structure():
    f = load("selfatt_h1_d16")
    counts = torch.bincount(f["n2g"])
    assert counts.tolist() == [1, 16, 17, 0, 64, 65, 249, 250, 251], "every tile / chunk edge and a graph without nodes"
    assert not bool((f["n2g"][1:] >= f["n2g"][:-1]).all()), "unsorted"
    assert [e - s for s, e in SR.chunks(load("selfatt_h3_d32")["n2g"], 64)] == [64, 1, 1, 64, 64, 64, 58, 17, 64]


@pytest.mark.parametrize("name", NAMES)
def test_kernel_order_emulation_is_inside_the_bound_and_hi_only_is_not(name):
    f = load(name)
    heads, dk, L = f["heads"], f["dk"], f["max_num_nodes"]
    t = torch.nn.functional.linear(f["x"].double(), f["sd"][SR.PREFIX + "selfatt_head_transforms.weight"].double())
    exact = SR.attention(t, f["n2g"], heads, dk, L)
    bnd = SR.bound(t, f["n2g"], heads, dk, L)
    emu = SR.emulate_kernel(t.float(), f["n2g"], heads, dk, L)
    assert bool(((emu.double() - exact).abs() <= bnd).all()), f"{name}: emulated kernel order exceeds the bound"
    hi_only = SR.emulate_kernel(t.float(), f["n2g"], heads, dk, L, corrections=False)
    assert bool(((hi_only.double() - exact).abs() > bnd).any()), f"{name}: the bound does not catch the missing correction products"


def test_native_class_has_reference_signature_parameters_and_keys():
    import ptgnn_b200 as P

    torch.manual_seed(0)
    m = P.MultiHeadSelfAttentionMessagePassing(32, 16, 16, 32, 64, 4, max_num_nodes=64)
    assert [n for n, _ in m.named_parameters()] == [SR.PREFIX + n for n in (
        "selfatt_head_transforms.weight", "summarization_layer.weight", "intermediate_layer.weight", "intermediate_layer.bias",
        "output_layer.weight", "output_layer.bias", "layer_norm1.weight", "layer_norm1.bias", "layer_norm2.weight", "layer_norm2.bias")]
    assert m.input_state_dimension == 32 and m.output_state_dimension == 32
    if not reference_available():
        pytest.skip("reference package not available")
    from oracle.refimport import import_reference

    import_reference()
    from ptgnn.neuralmodels.gnn.messagepassing.selfattmessagepassing import MultiHeadSelfAttentionMessagePassing as Ref

    assert inspect.signature(Ref.__init__) == inspect.signature(P.MultiHeadSelfAttentionMessagePassing.__init__)
    torch.manual_seed(0)
    ref = Ref(32, 16, 16, 32, 64, 4, max_num_nodes=64)
    assert list(ref.state_dict()) == list(m.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(ref.state_dict().values(), m.state_dict().values())), "same seed, same values"
    m.load_state_dict(ref.state_dict(), strict=True)


@pytest.mark.skipif(not reference_available(), reason="reference package not available")
def test_overlay_binds_the_native_layer_only_when_asked():
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from oracle.refimport import import_reference\nimport_reference()\n"
        "import ptgnn_b200 as P, ptgnn_b200.overlay as ov\n"
        "MOD = 'ptgnn.neuralmodels.gnn.messagepassing.selfattmessagepassing'\n"
        "import importlib\nref = importlib.import_module(MOD).MultiHeadSelfAttentionMessagePassing\n"
        "r = ov.install(force_torch_scatter=True)\n"
        "assert r['selfattention'] is False and importlib.import_module(MOD).MultiHeadSelfAttentionMessagePassing is ref\n"
        "ov.uninstall()\n"
        "r = ov.install(force_torch_scatter=True, native_selfattention=True)\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.selfattmessagepassing import MultiHeadSelfAttentionMessagePassing as M\n"
        "assert r['selfattention'] is True and M is P.MultiHeadSelfAttentionMessagePassing\n"
        "ov.uninstall()\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.selfattmessagepassing import MultiHeadSelfAttentionMessagePassing as M2\n"
        "assert M2 is ref\nprint('SELFATT-OVERLAY-OK')\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "SELFATT-OVERLAY-OK" in r.stdout, r.stdout + r.stderr[-3000:]


def test_overlay_pre_seeds_the_native_layer_before_the_reference_module_is_imported():
    if not reference_available():
        pytest.skip("reference package not available")
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from oracle.refimport import import_reference\nimport_reference()\n"
        "import ptgnn_b200 as P, ptgnn_b200.overlay as ov\n"
        "assert 'ptgnn.neuralmodels.gnn.messagepassing.selfattmessagepassing' not in sys.modules\n"
        "ov.install(force_torch_scatter=True, native_selfattention=True)\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.selfattmessagepassing import MultiHeadSelfAttentionMessagePassing as M\n"
        "assert M is P.MultiHeadSelfAttentionMessagePassing\nprint('SELFATT-PRESEED-OK')\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "SELFATT-PRESEED-OK" in r.stdout, r.stdout + r.stderr[-3000:]


# ---- backward ---------------------------------------------------------------------------------------------------------------
def _exact_forward(t64, n2g, heads, dk, L):
    """float64 (o, lse) of the attention."""
    a, b, _ = SR.split_heads(t64, heads, dk)
    lse = torch.cat([torch.logsumexp(torch.einsum("khd,vhd->khv", a[s:e], b[s:e]) / dk ** 0.5, dim=-1) for s, e in SR.chunks(n2g, L)])
    return SR.attention(t64, n2g, heads, dk, L), lse


def _bwd_inputs(counts, heads, dk, dv, seed):
    gen = torch.Generator().manual_seed(seed)
    n2g = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    n2g = n2g[torch.randperm(n2g.numel(), generator=gen)]
    t = torch.randn(n2g.numel(), heads * (2 * dk + dv), generator=gen)
    return n2g, t, torch.randn(n2g.numel(), heads * dv, generator=gen)


BWD_COUNTS = [1, 16, 17, 0, 64, 65, 130]


@pytest.mark.parametrize("dk,dv,L", [(16, 32, 70), (32, 16, 1000), (64, 64, 1)])
def test_backward_formula_equals_autograd_through_the_float64_forward(dk, dv, L):
    heads = 2
    n2g, t, d_o = _bwd_inputs(BWD_COUNTS, heads, dk, dv, dk + dv + L)
    t64 = t.double().requires_grad_(True)
    SR.attention(t64, n2g, heads, dk, L).backward(d_o.double())
    o, lse = _exact_forward(t64.detach(), n2g, heads, dk, L)
    got = SR.backward_formula(t64.detach(), o, lse, d_o, n2g, heads, dk, L)
    err = float((got - t64.grad).abs().max() / t64.grad.abs().max())
    assert err <= 1e-12, f"dk={dk} dv={dv} L={L}: {err:.2e}"


MUTANTS = ["no_delta", "db_unscaled", "kv_own_tile", "q_short"]


@pytest.mark.parametrize("dk,dv", [(16, 16), (32, 64)])
def test_backward_emulation_is_inside_the_bound_and_the_mutants_are_not(dk, dv):
    """The float32 emulation of the backward kernels' order, on the float32-rounded exact o and lse, against backward_formula under
    backward_bound; each named mutant falls outside it (L = 100: chunks of 1 to 100 rows, two of them longer than a 64-row tile)."""
    heads, L = 2, 100
    n2g, t, d_o = _bwd_inputs(BWD_COUNTS, heads, dk, dv, 5 + dk)
    o, lse = (z.float() for z in _exact_forward(t.double(), n2g, heads, dk, L))
    ref = SR.backward_formula(t, o, lse, d_o, n2g, heads, dk, L)
    bnd = SR.backward_bound(t, o, lse, d_o, n2g, heads, dk, L)
    ratio = float(((SR.emulate_backward(t, o, lse, d_o, n2g, heads, dk, L).double() - ref).abs() / bnd).max())
    assert ratio <= 1.0, f"emulated kernel order exceeds the bound ({ratio:.2f})"
    for m in MUTANTS:
        mut = SR.emulate_backward(t, o, lse, d_o, n2g, heads, dk, L, mutant=m).double()
        assert bool(((mut - ref).abs() > bnd).any()), f"the bound does not reject {m}"
