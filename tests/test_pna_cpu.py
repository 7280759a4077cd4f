"""CPU: what an MlpMessagePassingLayer with the native PnaMessageAggregation refuses before it reaches a kernel, and the
``overlay.install(native_pna=True)`` binding of the class into the reference."""
import os
import subprocess
import sys

import pytest
import torch

import ptgnn_b200 as P
from oracle.refimport import reference_available
from ptgnn_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADJ = [(torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.int64))]


@pytest.mark.parametrize("kw", [dict(mlp_hidden_layers=1), dict(features_dimension=4)])
def test_training_dropout_still_refused_outside_the_native_pna_configuration(kw):
    # a message MLP that is not one bias-free Linear per type takes the composed path, where nothing applies the output dropout
    layer = P.MlpMessagePassingLayer(32, 32, 32, 1, P.PnaMessageAggregation(), dropout_rate=0.5, **kw).train()
    with torch.no_grad(), pytest.raises(NotImplementedError, match="dropout"):
        layer(torch.zeros(4, 32), ADJ, edge_features=[torch.zeros(3, 4)] if "features_dimension" in kw else None)
    for p in layer.parameters():             # gradients enabled, frozen parameters: the same path
        p.requires_grad_(False)
    with pytest.raises(NotImplementedError, match="dropout"):
        layer(torch.zeros(4, 32), ADJ, edge_features=[torch.zeros(3, 4)] if "features_dimension" in kw else None)


def test_training_dropout_runs_with_the_native_pna_and_a_default_message_mlp():
    # the layer applies the dropout to its result: the call gets past every refusal and stops only at the CPU tensors
    layer = P.MlpMessagePassingLayer(32, 32, 32, 1, P.PnaMessageAggregation(), dropout_rate=0.5).train()
    with torch.no_grad(), pytest.raises(N.NativeLibraryError):
        layer(torch.zeros(4, 32), ADJ)
    with pytest.raises(N.NativeLibraryError):
        layer(torch.zeros(4, 32), ADJ)


def test_gradients_still_refused_for_hidden_layer_mlps_with_the_native_pna():
    layer = P.MlpMessagePassingLayer(32, 32, 32, 1, P.PnaMessageAggregation(), mlp_hidden_layers=1)
    with pytest.raises(NotImplementedError):
        layer(torch.zeros(4, 32), ADJ)


@pytest.mark.skipif(not reference_available(), reason="reference package not available")
def test_overlay_binds_the_native_pna_only_when_asked():
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from oracle.refimport import import_reference\nimport_reference()\n"
        "import ptgnn_b200 as P, ptgnn_b200.overlay as ov\n"
        "MOD = 'ptgnn.neuralmodels.gnn.messagepassing.pna_aggregation'\n"
        "import importlib\nref = importlib.import_module(MOD).PnaMessageAggregation\n"
        "r = ov.install(force_torch_scatter=True)\n"
        "assert r['pna'] is False and importlib.import_module(MOD).PnaMessageAggregation is ref\n"
        "ov.uninstall()\n"
        "r = ov.install(force_torch_scatter=True, native_pna=True)\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.pna_aggregation import PnaMessageAggregation as M\n"
        "import ptgnn.neuralmodels.gnn.messagepassing as pkg\n"
        "assert r['pna'] is True and M is P.PnaMessageAggregation and pkg.PnaMessageAggregation is M\n"
        "m = M(delta=2.3)\nassert m.delta == 2.3 and m.output_state_size(8) == 120\n"
        "ov.uninstall()\n"
        "from ptgnn.neuralmodels.gnn.messagepassing.pna_aggregation import PnaMessageAggregation as M2\n"
        "assert M2 is ref and pkg.PnaMessageAggregation is ref\nprint('PNA-OVERLAY-OK')\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "PNA-OVERLAY-OK" in r.stdout, r.stdout + r.stderr[-3000:]
