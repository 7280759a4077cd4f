"""CPU checks of the native VarMisuse head (DESIGN.md §3.16): the float64 restatement (tests/heads_reference.py) against fixtures generated
from the reference class, the teeth of its error bounds, the native class's interface against the reference's, the refusals (raised
before any kernel runs) and the ``overlay.install(native_heads=True)`` binding."""
import inspect
import os
import subprocess
import sys

import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import heads_reference as R  # noqa: E402
from helpers import load_golden  # noqa: E402

from oracle.refimport import import_reference, reference_available  # noqa: E402

import ptgnn_b200  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODULE = "ptgnn.implementations.varmisuse.varmisuse"
KEY = "_VarMisuseGraphModel__candidate_scores.weight"
FIXTURES = ("heads_varmisuse", "heads_varmisuse_crossed")
needs_reference = pytest.mark.skipif(not reference_available(), reason="the reference tree is not present")


def golden(name):
    g = load_golden(name)
    t = {k: torch.from_numpy(v) for k, v in g.items()}
    return t, (t["h"], t["cand"], t["slot_of"], t["slot_nodes"], t["correct"], t["w"])


@pytest.mark.parametrize("name", FIXTURES)
def test_restatement_reproduces_the_reference(name):
    t, args = golden(name)
    ref = R.varmisuse(*args)
    assert abs(float(ref["loss"]) - float(t["loss"])) <= R.loss_bound(*args)
    assert ref["hits"] / args[3].shape[0] == float(t["accuracy"])
    d_h, d_w = R.varmisuse_gradients(*args)
    for got, key in ((d_h, "grad_h"), (d_w, "grad_w")):
        want = t[key].double()
        assert float((got - want).abs().max()) <= 1e-5 * max(1.0, float(want.abs().max())), key


def test_fixtures_cover_the_slot_shapes():
    t, (h, cand, slot_of, slot_nodes, correct, w) = golden("heads_varmisuse")
    counts = torch.bincount(slot_of, minlength=slot_nodes.shape[0])
    assert sorted(counts.tolist()) == [1, 2, 31, 32, 33, 300]
    assert not bool((slot_of[1:] >= slot_of[:-1]).all()), "slot ids are not sorted"
    ref = R.varmisuse(h, cand, slot_of, slot_nodes, correct, w)
    tied = [j for j in range(slot_nodes.shape[0]) if int((ref["score"][slot_of == j] == ref["score"][ref["argmax"][j]]).sum()) > 1]
    assert tied, "some slot's best score is tied"
    crossed, _ = golden("heads_varmisuse_crossed")
    assert bool((slot_of[crossed["correct"]] != torch.arange(slot_nodes.shape[0])).any())


@pytest.mark.parametrize("name", FIXTURES)
def test_bounds_have_teeth(name):
    """The fp32 reference sits inside the bounds; a 2^-12 error in the weight does not."""
    t, args = golden(name)
    exact = R.varmisuse(*args)
    h, cand, slot_of, slot_nodes, correct, w = args
    assert bool(((exact["score"] - R.varmisuse(*args[:5], w * (1 + 2.0 ** -12))["score"]).abs() > R.score_bound(*args[:4], w)).any())
    assert abs(float(exact["loss"]) - float(t["loss"])) <= R.loss_bound(*args)


def test_constructor_signature_and_keys():
    cls = ptgnn_b200.VarMisuseGraphModel
    assert list(inspect.signature(cls.__init__).parameters) == ["self", "gnn"]
    assert list(inspect.signature(cls.forward).parameters) == ["self", "graph_data", "correct_candidate_idxs"]
    gnn = nn.Module()
    gnn.output_node_state_dim = 64
    m = cls(gnn)
    assert list(m.state_dict()) == [KEY] and tuple(m.state_dict()[KEY].shape) == (1, 128)
    with pytest.raises(ZeroDivisionError):
        m.report_metrics()          # as the reference: no sample seen yet


def _reference_module():
    import_reference()
    from ptgnn.neuralmodels.gnn import structs

    structs.GraphData.__class_getitem__ = classmethod(lambda cls, params: cls)   # see tests/golden/generate_heads_golden.py
    return __import__(MODULE, fromlist=["x"])


@needs_reference
def test_seeded_parameters_and_state_dicts_match_the_reference():
    ref = _reference_module()
    for H in (4, 64, 256):
        gnn = nn.Linear(3, 3)
        gnn.output_node_state_dim = H
        torch.manual_seed(5)
        r = ref.VarMisuseGraphModel(gnn)
        torch.manual_seed(5)
        n = ptgnn_b200.VarMisuseGraphModel(gnn)
        assert list(r.state_dict()) == list(n.state_dict())
        assert all(torch.equal(a, b) for a, b in zip(r.state_dict().values(), n.state_dict().values()))
        n.load_state_dict(r.state_dict(), strict=True)
        r.load_state_dict(n.state_dict(), strict=True)


def test_supported_state_sizes():
    lib = N.lib()
    for H, ok in ((4, True), (64, True), (1024, True), (6, False), (0, False), (1028, False), (2, False)):
        assert bool(lib.ptgnn_b200_varmisuse_supported(H)) == ok, H
        assert (lib.ptgnn_b200_varmisuse_workspace_bytes(10, 3, H) > 0) == ok, H


def test_refusals_before_any_kernel():
    launches = N.launch_count()
    gnn = nn.Module()
    gnn.output_node_state_dim = 6
    m = ptgnn_b200.VarMisuseGraphModel(gnn)
    h = torch.zeros(5, 6)
    from ptgnn_b200.gnn import GnnOutput

    out = GnnOutput(h, h, torch.zeros(5, dtype=torch.int64), {"candidate_nodes": torch.tensor([0, 1]), "slot_node_idx": torch.tensor([2])},
                    {"candidate_nodes": torch.tensor([0, 0])}, 1)
    gnn.forward = lambda **kw: out
    with pytest.raises(NotImplementedError, match="multiple of 4"):
        m({}, torch.tensor([0]))
    assert N.launch_count() == launches


@needs_reference
def test_overlay_binds_the_native_head_only_when_asked():
    code = (
        "import sys, warnings; sys.path.insert(0, %r)\n"
        "from oracle.refimport import import_reference\nimport_reference()\n"
        "from ptgnn.neuralmodels.gnn import structs\n"
        "structs.GraphData.__class_getitem__ = classmethod(lambda cls, params: cls)\n"
        "import ptgnn_b200 as P, ptgnn_b200.overlay as ov, importlib\n"
        "r = ov.install(force_torch_scatter=True)\n"
        "mod = importlib.import_module(%r)\nref = mod.VarMisuseGraphModel\n"
        "from ptgnn.baseneuralmodel import ModuleWithMetrics\n"
        "class StubModel:\n"
        "    def build_neural_module(self):\n"
        "        g = __import__('torch').nn.Module()\n"
        "        g.output_node_state_dim = 16\n"
        "        return g\n"
        "def build():\n"
        "    model = mod.VarMisuseModel(StubModel())\n"
        "    return model.build_neural_module()\n"
        "assert r['heads'] is False and type(build()) is ref\n"
        "ov.uninstall()\n"
        "holder = type(sys)('holder'); holder.__name__ = 'ptgnn.holder'; holder.VM = ref; sys.modules['ptgnn.holder'] = holder\n"
        "r = ov.install(force_torch_scatter=True, native_heads=True)\n"
        "assert r['heads'] is True and mod.VarMisuseGraphModel is P.VarMisuseGraphModel\n"
        "assert holder.VM is P.VarMisuseGraphModel, 'a reference module imported before install is re-bound'\n"
        "m = build()\nassert type(m) is P.VarMisuseGraphModel and isinstance(m, ModuleWithMetrics)\n"
        "assert list(m.state_dict()) == [%r]\n"
        "ov.uninstall()\n"
        "assert mod.VarMisuseGraphModel is ref and holder.VM is ref and type(build()) is ref\nprint('HEADS-OVERLAY-OK')\n"
        % (ROOT, MODULE, KEY))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "HEADS-OVERLAY-OK" in r.stdout, r.stdout + r.stderr[-3000:]


@needs_reference
def test_overlay_changes_nothing_when_the_head_module_cannot_be_imported():
    """Unpatched, the reference's varmisuse module fails to import on Pythons whose typing rejects GraphData[Tuple[str, bool]]; then
    install(native_heads=True) raises ImportError before any step is applied.  Where it imports, the overlay is simply installed."""
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "sys.path[:0] = [%r, %r]\n"
        "import ptgnn_b200.overlay as ov\n"
        "before = set(sys.modules)\n"
        "try:\n"
        "    r = ov.install(force_torch_scatter=True, native_heads=True)\n"
        "except ImportError as e:\n"
        "    assert 'nothing was installed' in str(e)\n"
        "    changed = {m for m in set(sys.modules) ^ before if not m.startswith('ptgnn_b200')}   # the library's own imports aside\n"
        "    assert not changed and sys.modules.get('torch_scatter') is None, sorted(changed)\n"
        "    assert not ov._saved\n"
        "    print('REFUSED-CLEANLY')\n"
        "else:\n"
        "    assert r['heads'] is True\n"
        "    print('INSTALLED')\n"
        % (ROOT, os.path.join(ROOT, "oracle", "refstubs"), os.environ.get("PTGNN_REFERENCE_ROOT", "/root/reference")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and ("REFUSED-CLEANLY" in r.stdout or "INSTALLED" in r.stdout), r.stdout + r.stderr[-3000:]
