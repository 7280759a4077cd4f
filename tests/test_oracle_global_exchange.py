"""GruGlobalStateUpdate on the CPU: the float restatement (global_exchange_reference.py) against the reference's own outputs (tests/golden/global_*.npz, written by
tests/golden/generate_global_exchange_golden.py), and the overlay's class mapping and state_dict keys."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import global_exchange_reference as GX
from oracle.refimport import reference_available

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PREFIX_R = "sd::_AbstractGlobalGraphExchange__global_graph_representation_module."
PREFIX_G = "sd::_GruGlobalStateUpdate__gru_cell."


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: str(z[k]) if z[k].dtype.kind == "U" else torch.from_numpy(z[k]) for k in z.files}


def oracle_out(f):
    w = f.get(PREFIX_R + "_WeightedSumVarSizedElementReduce__weights_layer.weight")
    return GX.global_gru_update_forward(f["h"], f["n2g"], f["kind"], w, *(f[PREFIX_G + k] for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")))


@pytest.mark.parametrize("name", ["global_weighted", "global_sum", "global_mean", "global_max"])
def test_oracle_reproduces_reference_global_exchange(name):
    f = load(name)
    w = f.get(PREFIX_R + "_WeightedSumVarSizedElementReduce__weights_layer.weight")
    g = GX.graph_readout(f["h"], f["n2g"], int(f["n2g"].max()) + 1, f["kind"], w)
    assert torch.equal(g, f["g"]), f"{name}: oracle readout differs from the reference's"
    assert torch.equal(oracle_out(f), f["out"]), f"{name}: oracle layer output differs from the reference's"


def test_oracle_reproduces_reference_global_exchange_autocast():
    f = load("global_weighted_bf16ac")
    with torch.autocast("cpu", dtype=torch.bfloat16):
        out = oracle_out(f)
    assert torch.equal(out.float(), f["out_autocast"])
    assert torch.equal(oracle_out(f), f["out_fp32_rounded_inputs"])


def test_fixture_graph_map_has_the_intended_structure():
    n2g = load("global_sum")["n2g"]
    counts = torch.bincount(n2g)
    assert counts[3] == 0 and counts[0] == 1 and counts[5] == 1, "a gap and two 1-node graphs"
    assert not bool((n2g[1:] >= n2g[:-1]).all()), "unsorted"


@pytest.mark.skipif(not reference_available(), reason="the reference tree is not available")
def test_overlay_maps_reference_global_exchange_to_native_class():
    code = f"""
import sys
sys.path.insert(0, {ROOT!r})
from oracle.refimport import import_reference
import_reference()
from ptgnn.neuralmodels.gnn.messagepassing.globalgraphexchange import GruGlobalStateUpdate as Ref
from ptgnn.neuralmodels.reduceops.varsizedsummary import WeightedSumVarSizedElementReduce, SimpleVarSizedElementReduce
ref_keys = [sorted(Ref(r, 64, 64).state_dict()) for r in (WeightedSumVarSizedElementReduce(64), SimpleVarSizedElementReduce("sum"))]
import ptgnn_b200.overlay as ov
ov.install()
import importlib
mod = importlib.import_module("ptgnn.neuralmodels.gnn.messagepassing.globalgraphexchange")
import ptgnn_b200 as P
assert mod.GruGlobalStateUpdate is P.GruGlobalStateUpdate, mod.GruGlobalStateUpdate
assert mod.AbstractGlobalGraphExchange is P.AbstractGlobalGraphExchange
nat_keys = [sorted(mod.GruGlobalStateUpdate(r, 64, 64).state_dict()) for r in (WeightedSumVarSizedElementReduce(64), SimpleVarSizedElementReduce("sum"))]
assert nat_keys == ref_keys, (nat_keys, ref_keys)
own = [sorted(P.GruGlobalStateUpdate(r, 64, 64).state_dict()) for r in (P.WeightedSumVarSizedElementReduce(64), P.SimpleVarSizedElementReduce("sum"))]
assert own == ref_keys, (own, ref_keys)
print("ok", ref_keys[0])
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr
