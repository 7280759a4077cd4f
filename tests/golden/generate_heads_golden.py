"""Generates the task-head fixtures by running the UNMODIFIED reference in this container.

    python tests/golden/generate_heads_golden.py       # writes tests/golden/heads_*.npz

The reference's ``VarMisuseGraphModel`` (``implementations/varmisuse/varmisuse.py:41-91``) is imported read-only through
``oracle/refimport.py`` and run on the CPU in fp32, with the oracle's ``torch_scatter`` stub (whose ``scatter_log_softmax`` is
differentiable) and a stub GNN that returns a fixed ``GnnOutput``.

* ``heads_varmisuse``: N = 700 node states h [N, 64]; one batch of slots with 1, 2, 31, 32, 33 and 300 candidates (slot ids in a
  shuffled, unsorted order; candidate nodes drawn with repeats, so some candidates of a slot have tied scores); the score weight ``w``
  (``_VarMisuseGraphModel__candidate_scores.weight``, seeded) and, for the correct ids ``correct`` (one per slot), the loss, the accuracy
  and the autograd gradients ``grad_h`` and ``grad_w``.
* ``heads_varmisuse_crossed``: the same inputs with the correct ids permuted across slots, so that correct_s lies in another slot than
  s (the reference's formula is applied as written).
"""
import os
import sys

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

import_reference()
from ptgnn.neuralmodels.gnn import structs  # noqa: E402
from ptgnn.neuralmodels.gnn.structs import GnnOutput  # noqa: E402

# varmisuse.py annotates a helper with GraphData[Tuple[str, bool]], one parameter of the two-parameter Generic: this Python's typing
# rejects that when the module is imported.  The subscription is only an annotation, so it is let through for the import.
structs.GraphData.__class_getitem__ = classmethod(lambda cls, params: cls)
from ptgnn.implementations.varmisuse.varmisuse import VarMisuseGraphModel  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
H = 64
NUM_NODES = 700
SLOT_SIZES = (1, 2, 31, 32, 33, 300)
KEY = "_VarMisuseGraphModel__candidate_scores.weight"


class StubGnn(nn.Module):
    """Returns the GnnOutput it was given; h is the leaf whose gradient the fixture records."""

    def __init__(self, dim):
        super().__init__()
        self.output_node_state_dim = dim
        self.output = None

    def forward(self, **kwargs):
        return self.output


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrays.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def inputs():
    gen = torch.Generator().manual_seed(9100)
    h = torch.randn(NUM_NODES, H, generator=gen)
    J = len(SLOT_SIZES)
    slot_nodes = torch.randperm(NUM_NODES, generator=gen)[:J]
    order = torch.randperm(J, generator=gen)                      # slot j gets SLOT_SIZES[order[j]] candidates
    slot_of = torch.cat([torch.full((SLOT_SIZES[int(order[j])],), j, dtype=torch.int64) for j in range(J)])
    slot_of = slot_of[torch.randperm(slot_of.shape[0], generator=gen)]     # candidates of a slot interleaved with the others
    cand = torch.randint(0, NUM_NODES, (slot_of.shape[0],), generator=gen)
    # repeated candidate nodes inside a slot: equal scores, so the argmax must take the first of them
    for j in range(J):
        ks = (slot_of == j).nonzero().flatten()
        if ks.shape[0] >= 2:
            cand[ks[-1]] = cand[ks[0]]
    correct = torch.stack([(slot_of == j).nonzero().flatten()[int(torch.randint(0, int((slot_of == j).sum()), (1,), generator=gen))]
                           for j in range(J)])
    return h, cand, slot_of, slot_nodes, correct


def run(h, cand, slot_of, slot_nodes, correct):
    torch.manual_seed(9200)
    gnn = StubGnn(H)
    model = VarMisuseGraphModel(gnn)
    hl = h.clone().requires_grad_(True)
    gnn.output = GnnOutput(input_node_representations=hl, output_node_representations=hl, node_to_graph_idx=torch.zeros(NUM_NODES, dtype=torch.int64),
                           node_idx_references={"candidate_nodes": cand, "slot_node_idx": slot_nodes},
                           node_graph_idx_reference={"candidate_nodes": slot_of}, num_graphs=1)
    model.reset_metrics()
    loss = model(graph_data={}, correct_candidate_idxs=correct)
    loss.backward()
    return dict(h=h.numpy(), cand=cand.numpy(), slot_of=slot_of.numpy(), slot_nodes=slot_nodes.numpy(), correct=correct.numpy(),
                w=model.state_dict()[KEY].numpy(), loss=loss.detach().numpy(), accuracy=np.float64(model.report_metrics()["Accuracy"]),
                grad_h=hl.grad.numpy(), grad_w=dict(model.named_parameters())[KEY].grad.numpy())


def main():
    h, cand, slot_of, slot_nodes, correct = inputs()
    save("heads_varmisuse", **run(h, cand, slot_of, slot_nodes, correct))
    crossed = correct[torch.tensor([2, 0, 1, 5, 3, 4])]
    save("heads_varmisuse_crossed", **run(h, cand, slot_of, slot_nodes, crossed))


if __name__ == "__main__":
    main()
