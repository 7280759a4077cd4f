"""CPU checks of the native classification heads (DESIGN.md §3.17): the float64 restatement (tests/classification_heads_reference.py)
against fixtures generated from the reference classes, the teeth of its error bounds, the native classes' interface, state_dict keys and
seeded initialisation against the reference's, the metrics protocol, and the ``overlay.install(native_graph2class_head=True,
native_ppi_head=True)`` binding and refusal."""
import inspect
import os
import subprocess
import sys

import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import classification_heads_reference as R  # noqa: E402
from helpers import load_golden  # noqa: E402

from oracle.refimport import import_reference, reference_available  # noqa: E402

import ptgnn_b200  # noqa: E402
from ptgnn_b200 import _native as N  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G2C_MODULE = "ptgnn.implementations.typilus.graph2class"
PPI_MODULE = "ptgnn.implementations.ppi.ppi"
needs_reference = pytest.mark.skipif(not reference_available(), reason="the reference tree is not present")


def golden(name):
    return {k: torch.from_numpy(v) for k, v in load_golden(name).items()}


def test_restatement_reproduces_graph2class():
    t = golden("heads_graph2class")
    h, idx, target, w, b = t["h"], t["idx"], t["target"], t["w"], t["b"]
    z, zb = R.logits(h, idx, w, b), R.logit_bound(h, idx, w, b)
    loss, lb, lse, arg, hits, n = R.ce(z, zb, target)
    assert abs(loss - float(t["loss"])) <= lb
    assert hits / target.shape[0] == float(t["accuracy"])
    assert int(arg[0]) == 0 and bool((z[0] == z[0, 0]).all()), "row 0 ties across every class; the first index wins"
    assert bool((target == R.IGNORE_INDEX).any()) and idx.unique().shape[0] < idx.shape[0], "ignored targets and repeated supernodes"
    for got, key in zip(R.param_grads(h, idx, w, R.ce_grad(z, target)), ("grad_h", "grad_w", "grad_b")):
        assert R.rel_err(got, t[key]) <= 1e-5, key


def test_restatement_reproduces_graph2class_under_bf16_autocast():
    t = golden("heads_graph2class_bf16ac")
    h, idx, target, w, b = t["h"], t["idx"], t["target"], t["w"], t["b"]
    z, zb = R.logits(h, idx, w, b, bf16=True), R.logit_bound(h, idx, w, b, bf16=True)
    assert bool(((t["logits"].double() - z).abs() <= zb).all()), "the reference's bf16 logits lie within the bf16 bound"
    loss, lb, *_ = R.ce(t["logits"].double(), zb, target)
    assert abs(loss - float(t["loss"])) <= lb


def test_restatement_reproduces_ppi():
    t = golden("heads_ppi")
    h, targets, w, b = t["h"], t["targets"], t["w"], t["b"]
    z, zb = R.logits(h, None, w, b), R.logit_bound(h, None, w, b)
    loss, lb, tp, fp, fn = R.bce(z, zb, targets)
    assert abs(loss - float(t["loss"])) <= lb
    assert R.bce_counts_decidable(z, zb)
    precision, recall, fscore = R.ppi_metrics(tp, fp, fn)
    R_ = h.shape[0]
    assert float(fscore) * R_ / R_ == float(t["f1_score"])
    assert float(precision) * R_ / R_ == float(t["pr_score"])
    assert float(recall) * R_ / R_ == float(t["re_score"])
    d_logits = (torch.sigmoid(z) - targets.double()) / R_
    for got, key in zip(R.param_grads(h, None, w, d_logits), ("grad_h", "grad_w", "grad_b")):
        assert R.rel_err(got, t[key]) <= 1e-5, key


@pytest.mark.parametrize("name", ["heads_graph2class", "heads_ppi"])
def test_bounds_have_teeth(name):
    t = golden(name)
    idx = t.get("idx")
    mutants = R.mutants_exceed(t["h"], idx, t["w"], t["b"])
    assert mutants == {"weight_2^-12": True, "no_correction": True}, mutants
    ref, zb = R.logits(t["h"], idx, t["w"], t["b"]), R.logit_bound(t["h"], idx, t["w"], t["b"])
    assert bool(((R.emulate_logits(t["h"], idx, t["w"], t["b"]) - ref).abs() <= zb).all()), "the kernel's own arithmetic passes"


def _classes():
    import_reference()
    from ptgnn.neuralmodels.gnn import graphneuralnetwork, structs

    for cls in (structs.GraphData, structs.TensorizedGraphData, graphneuralnetwork.GraphNeuralNetworkModel):
        cls.__class_getitem__ = classmethod(lambda cls, params: cls)
    import importlib

    return importlib.import_module(G2C_MODULE).Graph2ClassModule, importlib.import_module(PPI_MODULE).PPIClassification


class Stub(nn.Module):
    output_node_state_dim = 64


@needs_reference
def test_interface_keys_and_seeded_initialisation_match_the_reference():
    ref_g2c, ref_ppi = _classes()
    for ref, nat, C in ((ref_g2c, ptgnn_b200.Graph2ClassModule, 101), (ref_ppi, ptgnn_b200.PPIClassification, 121)):
        assert nat.__name__ == ref.__name__
        assert list(inspect.signature(nat.__init__).parameters) == list(inspect.signature(ref.__init__).parameters)
        assert list(inspect.signature(nat.forward).parameters) == list(inspect.signature(ref.forward).parameters)
        torch.manual_seed(5)
        r = ref(Stub(), C)
        torch.manual_seed(5)
        n = nat(Stub(), C)
        assert list(r.state_dict()) == list(n.state_dict())
        assert all(torch.equal(a, b) for a, b in zip(r.state_dict().values(), n.state_dict().values()))
        n.load_state_dict(r.state_dict(), strict=True)
    assert list(inspect.signature(ptgnn_b200.Graph2ClassModule.predict).parameters) == list(inspect.signature(ref_g2c.predict).parameters)
    assert list(inspect.signature(ptgnn_b200.Graph2ClassModule._logits).parameters) == list(inspect.signature(ref_g2c._logits).parameters)


def test_state_dict_keys():
    assert list(ptgnn_b200.Graph2ClassModule(Stub(), 3).state_dict()) == [
        "_Graph2ClassModule__node_to_class.weight", "_Graph2ClassModule__node_to_class.bias"]
    assert list(ptgnn_b200.PPIClassification(Stub(), 3).state_dict()) == [
        "_PPIClassification__output_representation_to_logits.weight", "_PPIClassification__output_representation_to_logits.bias"]


def test_metrics_before_any_sample_raise_zero_division_as_the_reference():
    for m in (ptgnn_b200.Graph2ClassModule(Stub(), 3), ptgnn_b200.PPIClassification(Stub(), 3)):
        with pytest.raises(ZeroDivisionError):
            m.report_metrics()
        m.train()
        m.eval()


def test_supported_shapes_and_sizes():
    lib = N.lib()
    for H, C, ok in ((8, 1, 1), (64, 101, 1), (256, 256, 1), (256, 121, 1), (12, 10, 0), (264, 10, 0), (64, 257, 0), (64, 0, 0)):
        assert lib.ptgnn_b200_classify_supported(H, C) == ok, (H, C)
    # the feature embedder's prepared format, columns padded to 16: fp32 (hi, lo') at 128 bytes per 64-wide K block and column
    assert lib.ptgnn_b200_classify_prepared_bytes(0, 64, 101) == 2 * 1 * 112 * 128
    assert lib.ptgnn_b200_classify_prepared_bytes(1, 256, 121) == 1 * 4 * 128 * 128
    assert lib.ptgnn_b200_classify_prepared_bytes(0, 256, 256) == 2 * 2 * 4 * 128 * 128
    # per-row partials (one float4 per row and column block) and one float4 per 1024 rows, each slice rounded up to 256 bytes
    assert lib.ptgnn_b200_classify_workspace_bytes(0, 3000, 256, 121) == 48128 + 256
    assert lib.ptgnn_b200_classify_workspace_bytes(0, 1000, 64, 129) == 2 * 1000 * 16 + 256


class FixedGnn(nn.Module):
    output_node_state_dim = 64

    def forward(self, **kwargs):
        return type("GnnOutput", (), {"output_node_representations": torch.zeros(2, 64)})()


def test_cpu_tensors_raise():
    with torch.no_grad(), pytest.raises(N.NativeLibraryError):
        ptgnn_b200.PPIClassification(FixedGnn(), 3)({}, torch.zeros(2, 3, dtype=torch.bool))


@needs_reference
def test_overlay_binds_the_native_graph2class_head_only_when_asked():
    code = (
        "import sys, warnings; sys.path.insert(0, %r)\n"
        "warnings.simplefilter('ignore', FutureWarning)\n"
        "from oracle.refimport import import_reference\nimport_reference()\n"
        "import ptgnn_b200 as P, ptgnn_b200.overlay as ov, importlib\n"
        "from ptgnn.baseneuralmodel import ModuleWithMetrics\n"
        "r = ov.install(force_torch_scatter=True)\n"
        "assert r['graph2class_head'] is False and r['ppi_head'] is False\n"
        "mod = importlib.import_module(%r)\nref = mod.Graph2ClassModule\n"
        "from ptgnn.implementations.typilus.train import create_graph2class_gnn_model\n"
        "class StubGnnModel:\n"
        "    def build_neural_module(self):\n"
        "        g = __import__('torch').nn.Module()\n"
        "        g.output_node_state_dim = 64\n"
        "        return g\n"
        "def build():\n"
        "    model = create_graph2class_gnn_model()\n"
        "    model._Graph2Class__gnn_model = StubGnnModel()\n"
        "    model._Graph2Class__target_vocab = ['t%%d' %% i for i in range(101)]\n"
        "    return model.build_neural_module()\n"
        "assert type(build()) is ref\n"
        "ov.uninstall()\n"
        "holder = type(sys)('holder'); holder.__name__ = 'ptgnn.holder'; holder.G2C = ref; sys.modules['ptgnn.holder'] = holder\n"
        "r = ov.install(force_torch_scatter=True, native_graph2class_head=True)\n"
        "assert r['graph2class_head'] is True and r['heads'] is False and mod.Graph2ClassModule is P.Graph2ClassModule\n"
        "assert holder.G2C is P.Graph2ClassModule, 'a reference module imported before install is re-bound'\n"
        "m = build()\nassert type(m) is P.Graph2ClassModule and isinstance(m, ModuleWithMetrics)\n"
        "assert list(m.state_dict()) == ['_Graph2ClassModule__node_to_class.weight', '_Graph2ClassModule__node_to_class.bias']\n"
        "ov.uninstall()\n"
        "assert mod.Graph2ClassModule is ref and holder.G2C is ref and type(build()) is ref\nprint('G2C-OVERLAY-OK')\n"
        % (ROOT, G2C_MODULE))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "G2C-OVERLAY-OK" in r.stdout, r.stdout + r.stderr[-3000:]


@needs_reference
def test_overlay_refuses_the_ppi_head_cleanly_when_its_module_cannot_be_imported():
    """Unpatched, the reference's ppi module fails to import on Pythons whose typing rejects TensorizedGraphData[np.ndarray]; then
    install(native_ppi_head=True) raises ImportError before any step is applied.  Where it imports, the overlay is simply installed."""
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "sys.path[:0] = [%r, %r]\n"
        "import ptgnn_b200.overlay as ov\n"
        "before = set(sys.modules)\n"
        "try:\n"
        "    r = ov.install(force_torch_scatter=True, native_ppi_head=True)\n"
        "except ImportError as e:\n"
        "    assert 'native_ppi_head=True' in str(e) and 'nothing was installed' in str(e), str(e)\n"
        "    changed = {m for m in set(sys.modules) ^ before if not m.startswith('ptgnn_b200')}\n"
        "    assert not changed and sys.modules.get('torch_scatter') is None, sorted(changed)\n"
        "    assert not ov._saved\n"
        "    print('REFUSED-CLEANLY')\n"
        "else:\n"
        "    assert r['ppi_head'] is True\n"
        "    print('INSTALLED')\n"
        % (ROOT, os.path.join(ROOT, "oracle", "refstubs"), os.environ.get("PTGNN_REFERENCE_ROOT", "/root/reference")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and ("REFUSED-CLEANLY" in r.stdout or "INSTALLED" in r.stdout), r.stdout + r.stderr[-3000:]
    if sys.version_info >= (3, 12):
        assert "REFUSED-CLEANLY" in r.stdout
