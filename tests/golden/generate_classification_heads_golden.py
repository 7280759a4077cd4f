"""Generates the classification-head fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_classification_heads_golden.py       # writes tests/golden/heads_graph2class*.npz, heads_ppi.npz

The reference's ``Graph2ClassModule`` (``implementations/typilus/graph2class.py:63-102``) and ``PPIClassification``
(``implementations/ppi/ppi.py:13-62``) are imported read-only through ``oracle/refimport.py`` and run on the CPU with a stub GNN that
returns a fixed ``GnnOutput``; their parameters are the reference's seeded initialisation.

* ``heads_graph2class``: N = 500 node states h [N, 64], S = 300 supernode ids drawn with repeats, C = 101, every 9th target -100
  (ignored) and supernode row 0 all zeros (with the zero bias every logit of that row ties).  The loss, the accuracy and the autograd
  gradients ``grad_h``, ``grad_w``, ``grad_b``.
* ``heads_graph2class_bf16ac``: the same inputs under CPU autocast bf16: the loss, the accuracy and the bf16 logits.
* ``heads_ppi``: N = 120 node states h [N, 256], C = 121, bool targets, drawn so that no logit lies within 2e-4 of the threshold 0 (the
  counts are then decided by the kernel's error bound): the loss, the three metrics and the autograd gradients.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.gnn import graphneuralnetwork, structs  # noqa: E402

# ppi.py subscripts TensorizedGraphData[np.ndarray] and GraphData[np.ndarray] and the model class GraphNeuralNetworkModel with fewer
# parameters than their Generic takes, which this Python's typing rejects at class creation.  The subscriptions are only annotations,
# so they are let through for the import.
for cls in (structs.GraphData, structs.TensorizedGraphData, graphneuralnetwork.GraphNeuralNetworkModel):
    cls.__class_getitem__ = classmethod(lambda cls, params: cls)
from ptgnn.implementations.ppi.ppi import PPIClassification  # noqa: E402
from ptgnn.implementations.typilus.graph2class import Graph2ClassModule  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


class StubGnn(torch.nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.output_node_state_dim = dim
        self.output = None

    def forward(self, **kwargs):
        return self.output


def graph2class(bf16: bool):
    gen = torch.Generator().manual_seed(20)
    N, H, S, C = 500, 64, 300, 101
    h = torch.randn(N, H, generator=gen)
    idx = torch.randint(0, N, (S,), generator=gen)
    h[idx[0]] = 0.0
    target = torch.randint(0, C, (S,), generator=gen)
    target[::9] = -100
    torch.manual_seed(21)
    gnn = StubGnn(H)
    m = Graph2ClassModule(gnn, C)
    with torch.no_grad():
        m._Graph2ClassModule__node_to_class.weight.mul_(0.1)     # uniform_ in [0, 1) saturates the softmax; scaled down
    hd = h.clone().requires_grad_(True)
    gnn.output = types.SimpleNamespace(output_node_representations=hd, reference_nodes_idx={"supernodes": idx},
                                       reference_nodes_graph_idx={"supernodes": torch.zeros_like(idx)})
    lin = m._Graph2ClassModule__node_to_class
    out = {"h": h.numpy(), "idx": idx.numpy(), "target": target.numpy(), "w": lin.weight.detach().numpy().copy(),
           "b": lin.bias.detach().numpy().copy()}
    if bf16:
        with torch.autocast("cpu", torch.bfloat16), torch.no_grad():
            loss = m({}, target, None)
            logits, _ = m._logits({})
        out["logits"] = logits.float().numpy()
    else:
        loss = m({}, target, None)
        loss.backward()
        out.update(grad_h=hd.grad.numpy(), grad_w=lin.weight.grad.numpy(), grad_b=lin.bias.grad.numpy())
    out.update(loss=np.float64(float(loss)), accuracy=np.float64(m.report_metrics()["Accuracy"]))
    return out


def ppi():
    N, H, C = 120, 256, 121
    for seed in range(30, 1000):       # the first draw whose logits all lie clear of the threshold by far more than the kernel's error
        gen = torch.Generator().manual_seed(seed)
        h = torch.randn(N, H, generator=gen)
        targets = torch.rand(N, C, generator=gen) < 0.3
        torch.manual_seed(seed + 1)
        gnn = StubGnn(H)
        m = PPIClassification(gnn, C)
        with torch.no_grad():
            if float(m._PPIClassification__output_representation_to_logits(h).abs().min()) > 2e-4:
                break
    hd = h.clone().requires_grad_(True)
    gnn.output = types.SimpleNamespace(output_node_representations=hd)
    loss = m({}, targets)
    loss.backward()
    lin = m._PPIClassification__output_representation_to_logits
    metrics = m.report_metrics()
    return {"h": h.numpy(), "targets": targets.numpy(), "w": lin.weight.detach().numpy().copy(), "b": lin.bias.detach().numpy().copy(),
            "loss": np.float64(float(loss)), "f1_score": np.float64(metrics["f1_score"]), "pr_score": np.float64(metrics["pr_score"]),
            "re_score": np.float64(metrics["re_score"]), "grad_h": hd.grad.numpy(), "grad_w": lin.weight.grad.numpy(),
            "grad_b": lin.bias.grad.numpy()}


if __name__ == "__main__":
    for name, data in (("heads_graph2class", graph2class(False)), ("heads_graph2class_bf16ac", graph2class(True)), ("heads_ppi", ppi())):
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **data)
        print(name, float(data["loss"]))
