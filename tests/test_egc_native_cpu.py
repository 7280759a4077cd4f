"""CPU: the float64 restatement of EGCMessagePassingLayer (tests/egc_reference.py) against the reference's fixtures, the teeth of its
error bound, the bf16 emulation against the reference under autocast, and the ``overlay.install(native_egc=True)`` binding."""
import os
import subprocess
import sys

import pytest
import torch

import egc_reference as E
from helpers import golden_adjacency, golden_state_dict, load_golden
from oracle.refimport import reference_available

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P_ = "_EGCMessagePassingLayer__"


def _fixture(name):
    g = load_golden(name)
    adj = golden_adjacency(g)
    W, cw, cb = E.params_of(golden_state_dict(g), len(adj))
    return g, adj, W, cw, cb


@pytest.mark.parametrize("agg", ["sum", "mean", "max", "min"])
def test_restatement_reproduces_the_reference_forward_and_gradients(agg):
    g, adj, W, cw, cb = _fixture(f"egc_grad_{agg}")
    heads, bases = int(g["heads"]), int(g["bases"])
    h = torch.from_numpy(g["h"]).double().requires_grad_(True)
    params = [w.double().requires_grad_(True) for w in W] + [cw.double().requires_grad_(True), cb.double().requires_grad_(True)]
    out = E.forward_torch(h, adj, params[:-2], params[-2], params[-1], agg, heads, bases)
    # relative L2: the fixture is the reference's fp32 arithmetic, whose elementwise error near cancellations exceeds 1e-6
    assert E.rel_l2(out, torch.from_numpy(g["out"])) <= 1e-6
    grads = torch.autograd.grad(out, [h] + params, torch.from_numpy(g["d_out"]).double())
    assert E.rel_l2(grads[0], torch.from_numpy(g["d_h"])) <= 1e-5
    keys = [f"{P_}bases.{t}.weight" for t in range(len(W))] + [P_ + "weight_coeffs.weight", P_ + "weight_coeffs.bias"]
    for k, d in zip(keys, grads[1:]):
        ref = torch.from_numpy(g["grad::" + k])
        assert E.rel_l2(d, ref) <= 1e-5 if bool(ref.any()) else bool((d == 0).all()), k
    # the fixture has what the GPU tests rely on: an empty type, targets without in-edges, and no ties among a target's messages
    assert any(s.numel() == 0 for s, _ in adj)
    tgt = torch.cat([t for _, t in adj])
    assert int((torch.bincount(tgt, minlength=h.shape[0]) == 0).sum()) > 0
    if agg in ("max", "min"):
        keys_e = torch.cat([s * h.shape[0] + t + i * h.shape[0] ** 2 for i, (s, t) in enumerate(adj)])
        assert keys_e.unique().numel() == keys_e.numel()


def _random_case(seed, n=400, H=64, out=64, heads=8, bases=4, counts=(1500, 0, 700)):
    gen = torch.Generator().manual_seed(seed)
    adj = [(torch.randint(0, n, (c,), generator=gen), torch.randint(0, n - 30, (c,), generator=gen)) for c in counts]
    W = [torch.randn(bases * out, H, generator=gen) * 0.1 for _ in counts]
    cw, cb = torch.randn(heads * bases, H, generator=gen) * 0.1, torch.randn(heads * bases, generator=gen) * 0.1
    return torch.randn(n, H, generator=gen), adj, W, cw, cb


@pytest.mark.parametrize("agg", ["sum", "mean", "max", "min"])
@pytest.mark.parametrize("heads,bases,out", [(8, 4, 64), (4, 8, 64), (2, 1, 128), (8, 2, 64)])
def test_bound_holds_for_the_kernels_arithmetic_and_has_teeth(agg, heads, bases, out):
    h, adj, W, cw, cb = _random_case(5, out=out, heads=heads, bases=bases)
    ref, bnd = E.forward64(h, adj, W, cw, cb, agg, heads, bases)
    R = E.R
    R.check_bound(E.emulate_f32(h, adj, W, cw, cb, agg, heads, bases), ref, bnd, f"{agg} 3xFP16 emulation")
    with pytest.raises(AssertionError):
        R.check_bound(E.emulate_f32(h, adj, W, cw, cb, agg, heads, bases, correction=False), ref, bnd, "no correction products")
    if agg == "mean":
        with pytest.raises(AssertionError):
            R.check_bound(E.emulate_f32(h, adj, W, cw, cb, agg, heads, bases, mean_division=False), ref, bnd, "no mean division")
    empty = torch.ones(h.shape[0], dtype=torch.bool)
    empty[torch.cat([t for _, t in adj])] = False
    assert bool((bnd[empty] == 0).all()) and bool((ref[empty] == 0).all())


def test_slab_rows_are_a_permutation_in_the_documented_order():
    out, heads, bases = 128, 8, 4
    rows = torch.cat([E.slab_rows(s, out, heads, bases) for s in range(bases * out // 128)])
    assert torch.equal(rows.sort().values, torch.arange(bases * out))
    dh = out // heads
    # slab 1, position p = j * 4 + b: column o = 32 + j, head o // dh, base b
    j, b = 5, 3
    o = 32 + j
    assert int(E.slab_rows(1, out, heads, bases)[j * 4 + b]) == ((o // dh) * bases + b) * dh + o % dh


@pytest.mark.parametrize("agg", ["sum", "max"])
def test_bf16_emulation_reproduces_the_reference_under_autocast(agg):
    """Exact except where an fp32 sum of the reference (the coefficient Linear, the message GEMM, the sum over the bases) lands
    within its accumulation-order difference of a bf16 midpoint: such a value is one bf16 ulp apart, and where it is a product in a
    sum over the bases that cancels, the output moves by that ulp of the product.  1 of 24576 elements of egc_sum_bf16ac differs,
    none of egc_max_bf16ac."""
    g, adj, W, cw, cb = _fixture(f"egc_{agg}_bf16ac")
    got = E.emulate_bf16(torch.from_numpy(g["h"]), adj, W, cw, cb, agg, 8, 4)
    ref = torch.from_numpy(g["out_autocast"]).double()
    diff = (got - ref).abs()
    assert float((diff > 0).double().mean()) <= 1e-3, f"{int((diff > 0).sum())} elements differ"
    assert E.rel_l2(got, ref) <= 1e-5
    assert E.n2_bars(got, ref, torch.from_numpy(g["out_fp32_rounded_inputs"])) == {"rel_l2": True, "mean": True, "within": True}


@pytest.mark.skipif(not reference_available(), reason="reference package not available")
def test_overlay_binds_the_native_egc_only_when_asked():
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from oracle.refimport import import_reference\nimport_reference()\n"
        "import ptgnn_b200 as P, ptgnn_b200.overlay as ov, importlib\n"
        "MOD = 'ptgnn.neuralmodels.gnn.messagepassing.egcmessagepassing'\n"
        "early = importlib.import_module(MOD)\nref = early.EGCMessagePassingLayer\n"
        "r = ov.install(force_torch_scatter=True)\n"
        "assert r['egc'] is False and importlib.import_module(MOD).EGCMessagePassingLayer is ref\n"
        "ov.uninstall()\n"
        "holder = type(sys)('holder'); holder.__name__ = 'ptgnn.holder'; holder.EGC = ref; sys.modules['ptgnn.holder'] = holder\n"
        "r = ov.install(force_torch_scatter=True, native_egc=True)\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.egcmessagepassing import EGCMessagePassingLayer as M\n"
        "assert r['egc'] is True and M is P.EGCMessagePassingLayer\n"
        "assert holder.EGC is M, 'a reference module imported before install is re-bound'\n"
        "m = M(64, 64, 3, 'sum')\nassert m.output_state_dimension == 64\n"
        "ov.uninstall()\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.egcmessagepassing import EGCMessagePassingLayer as M2\n"
        "assert M2 is ref and holder.EGC is ref\nprint('EGC-OVERLAY-OK')\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "EGC-OVERLAY-OK" in r.stdout, r.stdout + r.stderr[-3000:]


def test_refusals_before_any_kernel():
    import ptgnn_b200 as P

    layer = P.EGCMessagePassingLayer(64, 64, 1, "sum", dropout_rate=0.1).train()
    adj = [(torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.int64))]
    with pytest.raises(NotImplementedError):
        layer(torch.zeros(4, 64), adj)


@pytest.mark.parametrize("agg", ["sum", "mean", "max", "min"])
@pytest.mark.parametrize("heads,bases,out", [(8, 4, 64), (4, 8, 64), (2, 1, 128), (8, 2, 64)])
def test_bf16_per_element_bound_rejects_dropped_roundings(agg, heads, bases, out):
    """The bf16 bar of the GPU tests is per element: exact wherever no fp32 accumulation lands near a bf16 midpoint.  Kernels that
    skip the bf16 rounding of A and of the products, or of the coefficients, fail it."""
    h, adj, W, cw, cb = _random_case(6, out=out, heads=heads, bases=bases)
    ref, bnd = E.bf16_kernel_reference(h, adj, W, cw, cb, agg, heads, bases)
    assert float((bnd > 0).double().mean()) <= 0.25, "the bound should be 0 for most elements"
    for mutant in ("no_round_ap", "no_round_coef"):
        if mutant == "no_round_ap" and bases == 1 and agg in ("max", "min"):
            continue        # A is already a bf16 message and the single product is exact in fp32: those roundings change nothing
        got, _ = E.bf16_kernel_reference(h, adj, W, cw, cb, agg, heads, bases, mutant=mutant)
        with pytest.raises(AssertionError):
            E.R.check_bound(got, ref, bnd, mutant)
    # the reference's autocast arithmetic (emulate_bf16) rounds at the same points: it agrees wherever the bound is 0
    emu = E.emulate_bf16(h, adj, W, cw, cb, agg, heads, bases)
    exact = bnd == 0
    assert float((emu[exact] != ref[exact]).double().mean()) <= 1e-3
