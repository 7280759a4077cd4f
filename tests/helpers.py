"""Shared test helpers: golden-fixture loading and conversion between the reference ``state_dict`` layout, the
oracle's functional arguments and ptgnn_b200 modules."""
import contextlib
import os
from typing import Dict, List, Tuple

import numpy as np
import pytest
import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-5  # north_star: fp32 node representations within 1e-5 (scaled by max(1, |ref|))


def split_f16(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The kernels' 3xFP16 split of x rounded to fp32 (csrc/tc_common.cuh): (hi, lo') fp16 tensors on x's device, with
    hi = fl16(x) and lo' = fl16(2^11 (x - hi)), bit for bit what the kernels compute."""
    x = x.float()
    hi = x.half()
    return hi, ((x - hi.float()) * 2048.0).half()


def load_golden(name: str) -> Dict[str, np.ndarray]:
    with np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


def golden_adjacency(g: Dict[str, np.ndarray], prefix: str = "") -> List[Tuple[torch.Tensor, torch.Tensor]]:
    adj, t = [], 0
    while f"{prefix}src{t}" in g:
        adj.append((torch.from_numpy(g[f"{prefix}src{t}"]).long(), torch.from_numpy(g[f"{prefix}tgt{t}"]).long()))
        t += 1
    return adj


def golden_state_dict(g: Dict[str, np.ndarray], prefix: str = "sd::") -> Dict[str, torch.Tensor]:
    return {k[len(prefix):]: torch.from_numpy(v) for k, v in g.items() if k.startswith(prefix)}


def gated_oracle_args(sd: Dict[str, torch.Tensor]) -> dict:
    p = "_GatedMessagePassingLayer__"
    T = sum(1 for k in sd if k.startswith(p + "edge_message_transformation_layers."))
    return dict(
        edge_weights=[sd[f"{p}edge_message_transformation_layers.{t}.weight"] for t in range(T)],
        gru_w_ih=sd[p + "state_update.weight_ih"], gru_w_hh=sd[p + "state_update.weight_hh"],
        gru_b_ih=sd[p + "state_update.bias_ih"], gru_b_hh=sd[p + "state_update.bias_hh"],
    )


def mlp_oracle_args(sd: Dict[str, torch.Tensor], use_layer_norm=True, use_dense_layer=True) -> dict:
    p = "_MlpMessagePassingLayer__"
    T = sum(1 for k in sd if k.startswith(p + "edge_message_transformation_layers.") and k.endswith("_MLP__mlp_modules.1.weight"))
    out = dict(edge_mlp_weights=[[sd[f"{p}edge_message_transformation_layers.{t}._MLP__mlp_modules.1.weight"]] for t in range(T)])
    i = 0
    if use_layer_norm:
        out.update(ln_weight=sd[f"{p}state_update.{i}.weight"], ln_bias=sd[f"{p}state_update.{i}.bias"])
        i += 1
    if use_dense_layer:
        out.update(dense_weight=sd[f"{p}state_update.{i}.weight"], dense_bias=sd[f"{p}state_update.{i}.bias"])
    return out


def assert_close(actual: torch.Tensor, expected: torch.Tensor, tol: float = TOL, what: str = ""):
    actual, expected = actual.detach().cpu().double(), expected.detach().cpu().double()
    assert actual.shape == expected.shape, f"{what}: shape {tuple(actual.shape)} != {tuple(expected.shape)}"
    err = (actual - expected).abs() / expected.abs().clamp(min=1.0)
    worst = float(err.max()) if err.numel() else 0.0
    assert worst <= tol, f"{what}: max scaled error {worst:.3e} > {tol:.1e}"


@contextlib.contextmanager
def unchained():
    """Inside the block no layer sees a state chain (edgeplan.state_chain): every layer packs its own states.  The reference run
    for the packed-state hand-off between layers, which must be bit-identical to it."""
    from ptgnn_b200 import edgeplan, globalexchange, gnn, messagepassing

    with pytest.MonkeyPatch.context() as mp:
        for module in (edgeplan, messagepassing, globalexchange, gnn):   # embeddings looks it up in edgeplan at call time
            mp.setattr(module, "current_state_chain", lambda: None)
        yield


def random_adjacency(gen: torch.Generator, num_nodes: int, counts, low: int = 0):
    return [
        (torch.randint(low, num_nodes, (c,), generator=gen, dtype=torch.int64),
         torch.randint(low, num_nodes, (c,), generator=gen, dtype=torch.int64))
        for c in counts
    ]


# golden fixture name -> (layer kind, constructor kwargs for the ptgnn_b200 / reference class)
GOLDEN_MLP_KW = {
    "mlp_max": dict(input_state_dimension=32, output_state_dimension=32, message_dimension=32, message_aggregation_function="max"),
    "mlp_sum": dict(input_state_dimension=32, output_state_dimension=32, message_dimension=32, message_aggregation_function="sum"),
    "mlp_wide": dict(input_state_dimension=64, output_state_dimension=32, message_dimension=64, message_aggregation_function="max"),
    "mlp_notarget": dict(input_state_dimension=32, output_state_dimension=64, message_dimension=32, message_aggregation_function="mean",
                         use_target_state_as_message_input=False),
    "mlp_bare": dict(input_state_dimension=32, output_state_dimension=32, message_dimension=32, message_aggregation_function="min",
                     message_activation=None, use_layer_norm=False, use_dense_layer=False),
}
GOLDEN_GATED = ["gated_sum", "gated_max", "gated_mean", "gated_min"]


def mlp_oracle_call_kwargs(name: str, sd) -> dict:
    kw = GOLDEN_MLP_KW[name]
    args = mlp_oracle_args(sd, kw.get("use_layer_norm", True), kw.get("use_dense_layer", True))
    args.update(
        aggregation_fn=kw["message_aggregation_function"],
        use_target_state_as_message_input=kw.get("use_target_state_as_message_input", True),
        message_activation=None if ("message_activation" in kw and kw["message_activation"] is None) else "gelu",
        dense_activation="tanh",
    )
    return args


def minibatch_graphs(seed=21, num_graphs=9, num_types=4):
    """Per-graph LOCAL structure as GraphNeuralNetworkModel.tensorize produces it (graphneuralnetwork.py:313-322, :350-363): int32
    arrays, some edge types empty, reference nodes under two names (one of them absent from some graphs)."""
    rng = np.random.RandomState(seed)
    graphs = []
    for g in range(num_graphs):
        n = int(rng.randint(1, 60))
        adj = []
        for t in range(num_types):
            e = 0 if (t == 2 and g % 3 == 0) else int(rng.randint(0, 4 * n))
            adj.append((rng.randint(0, n, e).astype(np.int32), rng.randint(0, n, e).astype(np.int32)))
        refs = {"token-sequence": rng.randint(0, n, int(rng.randint(0, 7))).astype(np.int32)}
        if g % 2 == 0:
            refs["candidate_nodes"] = rng.randint(0, n, int(rng.randint(1, 4))).astype(np.int32)
        graphs.append((adj, refs, n))
    return graphs
