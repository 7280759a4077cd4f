"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol the header declares, the
module API mirrors the reference's, and the product refuses to run without CUDA (no CPU fallback)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

import ptgnn_b200 as P
from ptgnn_b200 import _native as N
from helpers import GOLDEN_MLP_KW, golden_state_dict, load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "ptgnn_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ptgnn_b200_\w+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    declared = _declared_symbols()
    assert len(declared) >= 12
    handle = N.lib()
    for name in declared:
        assert hasattr(handle, name), f"{name} declared in include/ptgnn_b200.h but not exported"
    assert sorted(N.SIGNATURES) == declared, "ctypes SIGNATURES must cover exactly the header's entry points"
    assert handle.ptgnn_b200_abi_version() == 4


def test_signatures_are_parsed_from_the_header():
    i32, i64, f32, size, P = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_size_t, ctypes.c_void_p
    sig = N.SIGNATURES
    assert sig["ptgnn_b200_last_error"] == (ctypes.c_char_p, [])
    assert sig["ptgnn_b200_plan_workspace_bytes"] == (size, [i64, i64])
    assert sig["ptgnn_b200_graph_norm_forward"] == (i32, [i32, P, i64, i32, P, P, P, i64, P, P, P, f32, P, P, P, P, size, P])
    assert sig["ptgnn_b200_gated_forward_fused"] == (i32, [i32, P, P, P, i64, i64, i32, i32, i32, P, P, P, P, P, P, P, i32, P, P, P, size, P,
                                                           size, i32, P])
    assert N.parse_signatures("/* ptgnn_b200_x(double); */\n#define A 1\nint32_t ptgnn_b200_x(const float *const *w, float eps, // e\n"
                              "  size_t n);\nint ptgnn_b200_y(void);") == {"ptgnn_b200_x": (i32, [P, f32, size]), "ptgnn_b200_y": (i32, [])}
    for proto in ("int ptgnn_b200_x(double eps);", "int ptgnn_b200_x(unsigned n);", "void ptgnn_b200_x(int32_t n);",
                  "float *ptgnn_b200_x(int32_t n);", "int ptgnn_b200_x();"):
        with pytest.raises(N.NativeLibraryError, match="ptgnn_b200_x"):
            N.parse_signatures(proto)


def test_call_checks_the_argument_count_before_touching_cuda(monkeypatch):
    def no_cuda(*args, **kwargs):
        raise AssertionError("reached CUDA")

    monkeypatch.setattr(torch.cuda, "device", no_cuda)
    monkeypatch.setattr(N, "current_stream", no_cuda)
    n = len(N.SIGNATURES["ptgnn_b200_segment_ids"][1]) - 1        # every parameter but the stream
    for count in (n - 1, n + 1):
        with pytest.raises(TypeError, match="ptgnn_b200_segment_ids"):
            N.call("ptgnn_b200_segment_ids", "cuda", *[0] * count)
    with pytest.raises(AssertionError, match="reached CUDA"):
        N.call("ptgnn_b200_segment_ids", "cuda", *[0] * n)


def test_fused_supported_shapes():
    """ptgnn_b200_fused_supported is 1 exactly on the shapes both fused layer kernels take (the fused aggregation and the
    weights-stationary GRU): D = 128 with H in {64, 128} (fp32 states) / {64, 128, 256} (bf16 states)."""
    handle = N.lib()
    dims = range(32, 513, 16)
    expected = {0: {(64, 128), (128, 128)}, 1: {(64, 128), (128, 128), (256, 128)}}
    for bf16, shapes in expected.items():
        got = {(H, D) for H in dims for D in dims if handle.ptgnn_b200_fused_supported(bf16, H, D) == 1}
        assert got == shapes, f"bf16_states={bf16}: {sorted(got)}"


def test_workspace_size_queries_run_without_a_gpu():
    handle = N.lib()
    assert handle.ptgnn_b200_plan_workspace_bytes(1000, 5000) > 4 * 5000 * 4
    assert handle.ptgnn_b200_gated_workspace_bytes(0, 1000, 5000, 17, 128, 128) >= 5000 * 128 * 4 + 1000 * 128 * 4
    assert handle.ptgnn_b200_mlp_workspace_bytes(0, 1000, 5000, 17, 128, 128, 128, 1) >= 5000 * 128 * 4
    assert handle.ptgnn_b200_scatter_workspace_bytes(1000, 5000) > handle.ptgnn_b200_plan_workspace_bytes(1000, 5000)


# (N, E, T, H, D) -> workspace bytes of the unfused gated layer, fp32 / bf16 states
_GATED_WS = {
    (1000, 5000, 17, 128, 128): (7269376, 2423808),
    (777, 4321, 3, 64, 64): (2044416, 777216),
    (500, 3001, 5, 256, 256): (12994560, 3632640),
    (1000, 5000, 4, 96, 36): (1851392, 597248),      # fp32 states: FFMA dims
    (123, 0, 2, 64, 128): (1105408, 213760),
}
# (T, H, D) -> weight-cache bytes of the unfused gated layer, fp32 / bf16 states (fp32: 0 unless every step runs on tensor cores)
_GATED_CACHE = {(17, 128, 128): (3278848, 887296), (3, 64, 64): (361472, 124416), (5, 256, 256): (6819840, 1839616),
                (4, 96, 36): (0, 164864), (2, 32, 16): (0, 27648), (2, 64, 128): (525312, 181760)}
# (N, E, T, H, D, out_dim, use_target_state) -> workspace bytes of the unfused Mlp layer, fp32 / bf16 states
_MLP_WS = {
    (1000, 5000, 17, 128, 128, 128, 0): (5431808, 2126848),
    (1000, 5000, 17, 128, 128, 192, 1): (7725568, 2700288),
    (777, 4321, 3, 64, 64, 64, 1): (1534976, 710656),
    (500, 3001, 5, 256, 256, 192, 0): (6600192, 2547200),
    (1000, 5000, 4, 96, 36, 36, 0): (985600, 463104),
    (1000, 5000, 4, 96, 36, 192, 1): (1140736, 502016),
    (1000, 5000, 4, 96, 36, 0, 1): (1096192, 0),     # out_dim <= 0: the message dim for fp32 states, no size for bf16
    (123, 0, 2, 64, 128, 128, 1): (456704, 130816),
}
# (N, N_src (0: N), T, H, D, out_dim (0: no dense layer), use_target_state) -> workspace bytes of the fused Mlp layer, fp32 / bf16
_MLP_FUSED_WS = {
    (1000, 0, 17, 128, 128, 128, 0): (2269952, 846592),
    (1000, 0, 17, 64, 128, 192, 1): (2335744, 862976),
    (777, 500, 3, 128, 128, 0, 1): (1576960, 429056),
    (500, 0, 5, 256, 128, 0, 0): (1555200, 489216),
    (123, 0, 2, 64, 128, 112, 0): (275456, 93696),
}
# (T, H, D, out_dim, use_target_state) -> weight-cache bytes of the fused Mlp layer, fp32 / bf16 (fp32: 0 off the fused dims)
_MLP_FUSED_CACHE = {(17, 128, 128, 128, 0): (1245440, 0), (17, 64, 128, 192, 1): (1310976, 0), (3, 128, 128, 0, 1): (524544, 0),
                    (5, 256, 128, 0, 0): (0, 0), (2, 64, 128, 112, 0): (180480, 0)}
# the stand-alone fp32 pieces: (in_dim, out_dim), (T, in_dim, message_dim, use_target_state), (state_dim, input_dim)
_LINEAR_WS = {(128, 128): 131328, (36, 200): 58112, (256, 64): 131328, (32, 16): 4352, (4, 4): 768}
_EDGE_MESSAGES_WS = {(17, 128, 128, 0): 2228480, (3, 64, 192, 1): 590080, (1, 36, 16, 0): 4864, (5, 256, 112, 1): 2294016}
_GRUCELL_WS = {(128, 128): 1968896, (64, 36): 522496, (256, 256): 6787840, (96, 32): 854272}

# every other size query of the header: name -> {arguments (bf16_states first where the query takes it): bytes}; 0 marks an
# unsupported shape
_OTHER_SIZES = {
    "plan_workspace_bytes": {(1000, 5000): 88576, (777, 4321): 76544, (0, 0): 2816, (5, 0): 2816, (100000, 1): 402688},
    "scatter_workspace_bytes": {(1000, 5000): 199168, (777, 4321): 171520, (0, 0): 4864, (5, 0): 4864, (100000, 1): 804608},
    "block_plan_workspace_bytes": {(1000, 5000, 17, 64): 129280, (777, 4321, 3, 64): 111616, (0, 0, 1, 64): 3584, (5, 0, 2, 64): 3584,
        (4096, 70000, 33, 64): 1733632},
    "gated_fused_workspace_bytes": {(0, 1000, 0, 17, 128, 128): 3046144, (0, 777, 500, 3, 64, 128): 972288,
        (0, 0, 0, 2, 128, 128): 527104, (0, 500, 0, 5, 256, 128): 3119872, (0, 1000, 0, 4, 96, 36): 1262848,
        (1, 1000, 0, 17, 128, 128): 1011968, (1, 777, 500, 3, 64, 128): 323072, (1, 0, 0, 2, 128, 128): 264448,
        (1, 500, 0, 5, 256, 128): 1049856, (1, 1000, 0, 4, 96, 36): 248064},
    "gated_fused_weight_cache_bytes": {(0, 17, 128, 128): 1509376, (0, 3, 64, 128): 246784, (0, 5, 256, 128): 1839104,
        (0, 1, 128, 128): 460800, (0, 4, 96, 36): 350208, (1, 17, 128, 128): 755712, (1, 3, 64, 128): 123904, (1, 5, 256, 128): 921600,
        (1, 1, 128, 128): 231424, (1, 4, 96, 36): 175872},
    "packed_state_bytes": {(1000, 128): 512256, (777, 64): 199168, (0, 128): 256, (1, 256): 1280, (5000, 96): 1920256},
    "egc_fused_workspace_bytes": {(0, 1000, 17, 128, 128, 8, 4): 5146368, (0, 777, 3, 64, 128, 4, 2): 427520,
        (0, 0, 2, 128, 128, 8, 4): 574208, (0, 500, 5, 256, 128, 8, 8): 0, (0, 1000, 4, 96, 36, 2, 2): 0,
        (1, 1000, 17, 128, 128, 8, 4): 2917888, (1, 777, 3, 64, 128, 4, 2): 328960, (1, 0, 2, 128, 128, 8, 4): 311808,
        (1, 500, 5, 256, 128, 8, 8): 3458560, (1, 1000, 4, 96, 36, 2, 2): 0},
    "egc_fused_weight_cache_bytes": {(0, 17, 128, 128, 8, 4): 4456448, (0, 3, 64, 128, 4, 2): 196608, (0, 5, 256, 128, 8, 8): 0,
        (0, 1, 128, 128, 1, 1): 65536, (0, 4, 96, 36, 2, 2): 0, (1, 17, 128, 128, 8, 4): 2228224, (1, 3, 64, 128, 4, 2): 98304,
        (1, 5, 256, 128, 8, 8): 2621440, (1, 1, 128, 128, 1, 1): 32768, (1, 4, 96, 36, 2, 2): 0},
    "global_gru_workspace_bytes": {(0, 1000, 10, 128, 128): 1119744, (0, 777, 3, 64, 36): 307200, (0, 0, 0, 128, 64): 395776,
        (0, 5, 1, 256, 256): 2372096, (0, 1000, 10, 96, 128): 0, (1, 1000, 10, 128, 128): 509184, (1, 777, 3, 64, 36): 83456,
        (1, 0, 0, 128, 64): 297216, (1, 5, 1, 256, 256): 1973504, (1, 1000, 10, 96, 128): 0},
    "global_gru_weight_cache_bytes": {(0, 64): 50176, (0, 128): 198656, (0, 192): 445440, (0, 256): 790528, (0, 96): 0, (1, 64): 25600,
        (1, 128): 100352, (1, 192): 224256, (1, 256): 397312, (1, 96): 0},
    "graph_readout_workspace_bytes": {(1000, 10, 128): 21760, (777, 3, 64): 7424, (0, 0, 32): 512, (0, 5, 256): 6400, (33, 1, 96): 1536,
        (10, 2, 36): 0},
    "attention_readout_workspace_bytes": {(1000, 10, 128, 8): 175360, (777, 3, 64, 1): 7936, (0, 0, 32, 4): 1280, (0, 5, 256, 2): 13056,
        (33, 1, 96, 3): 0},
    "selfatt_workspace_bytes": {(1000, 10, 8): 32256, (777, 3, 1): 3584, (0, 0, 4): 256, (0, 5, 2): 256, (4096, 1, 3): 49408},
    "graph_norm_workspace_bytes": {(1000, 10, 128): 73984, (777, 3, 64): 19200, (0, 0, 32): 512, (0, 5, 256): 43264, (33, 1, 96): 4864},
    "copy_attention_workspace_bytes": {(1000, 10, 128, 4): 86272, (777, 3, 64, 1): 7424, (0, 0, 32, 7): 1280, (0, 5, 256, 2): 12544,
        (33, 1, 96, 3): 0},
    "embedding_bag_backward_workspace_bytes": {(1000, 8, 5000, 128): 2708736, (777, 1, 100, 63): 32256, (0, 4, 10, 64): 3072,
        (5, 0, 10, 64): 0, (33, 3, 0, 32): 768},
    "char_cnn_workspace_bytes": {(0, 98, 64, 3, 128, 5, 128, 2): 372736, (0, 256, 256, 5, 64, 3, 64, 4): 1574912,
        (0, 0, 64, 3, 64, 3, 64, 2): 0, (0, 98, 128, 1, 256, 1, 200, 1): 445440, (0, 98, 64, 3, 64, 3, 300, 2): 0,
        (1, 98, 64, 3, 128, 5, 128, 2): 225280, (1, 256, 256, 5, 64, 3, 64, 4): 1443840, (1, 0, 64, 3, 64, 3, 64, 2): 0,
        (1, 98, 128, 1, 256, 1, 200, 1): 248832, (1, 98, 64, 3, 64, 3, 300, 2): 0},
}

def test_unfused_layer_buffer_sizes_are_pinned():
    """The layers' and stand-alone pieces' workspace and weight-cache layouts, per state dtype: exact byte counts (a layout
    change is an ABI change for callers that keep buffers across calls)."""
    handle = N.lib()
    for bf16 in (0, 1):
        for args, want in _GATED_WS.items():
            assert handle.ptgnn_b200_gated_workspace_bytes(bf16, *args) == want[bf16], (bf16, args)
        for args, want in _GATED_CACHE.items():
            assert handle.ptgnn_b200_gated_weight_cache_bytes(bf16, *args) == want[bf16], (bf16, args)
        for args, want in _MLP_WS.items():
            assert handle.ptgnn_b200_mlp_workspace_bytes(bf16, *args) == want[bf16], (bf16, args)
        for args, want in _MLP_FUSED_WS.items():
            assert handle.ptgnn_b200_mlp_fused_workspace_bytes(bf16, *args) == want[bf16], (bf16, args)
        for args, want in _MLP_FUSED_CACHE.items():
            assert handle.ptgnn_b200_mlp_fused_weight_cache_bytes(bf16, *args) == want[bf16], (bf16, args)
    for args, want in _LINEAR_WS.items():
        assert handle.ptgnn_b200_linear_workspace_bytes(*args) == want, args
    for args, want in _EDGE_MESSAGES_WS.items():
        assert handle.ptgnn_b200_edge_messages_workspace_bytes(*args) == want, args
    for args, want in _GRUCELL_WS.items():
        assert handle.ptgnn_b200_grucell_workspace_bytes(*args) == want, args
    # D = 20: fp32 states run the FFMA message and GRU kernels and cache nothing
    assert handle.ptgnn_b200_gated_weight_cache_bytes(0, 17, 128, 20) == 0


def test_every_other_buffer_size_is_pinned():
    """The plan, per-graph, fused-layer, embedding and char-CNN workspace and weight-cache layouts: exact byte counts, including
    zero nodes and zero graphs."""
    handle = N.lib()
    for name, cases in _OTHER_SIZES.items():
        query = getattr(handle, "ptgnn_b200_" + name)
        for args, want in cases.items():
            assert query(*args) == want, (name, args)


def test_no_cpu_fallback():
    layer = P.GatedMessagePassingLayer(32, 32, 1, "sum").eval()
    adj = [(torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.int64))]
    with torch.no_grad(), pytest.raises(N.NativeLibraryError):
        layer(node_states=torch.zeros(4, 32), adjacency_lists=adj, node_to_graph_idx=None, reference_node_ids={},
              reference_node_graph_idx={}, edge_features=[torch.empty(3, 0)])
    with pytest.raises(N.NativeLibraryError):
        P.scatter(torch.zeros(3, 4), torch.zeros(3, dtype=torch.int64), dim=0, dim_size=2, reduce="sum")


def test_constructor_signatures_match_reference_contract():
    gated = list(inspect.signature(P.GatedMessagePassingLayer.__init__).parameters)
    assert gated == ["self", "state_dimension", "message_dimension", "num_edge_types", "message_aggregation_function",
                     "dropout_rate", "edge_feature_dimension"]
    mlp = list(inspect.signature(P.MlpMessagePassingLayer.__init__).parameters)
    assert mlp == ["self", "input_state_dimension", "output_state_dimension", "message_dimension", "num_edge_types",
                   "message_aggregation_function", "message_activation", "use_target_state_as_message_input",
                   "mlp_hidden_layers", "use_layer_norm", "use_dense_layer", "dropout_rate", "dense_activation",
                   "features_dimension"]
    fwd = list(inspect.signature(P.AbstractMessagePassingLayer.forward).parameters)
    assert fwd == ["self", "node_states", "adjacency_lists", "node_to_graph_idx", "reference_node_ids",
                   "reference_node_graph_idx", "edge_features"]
    gnn = list(inspect.signature(P.GraphNeuralNetwork.__init__).parameters)
    assert gnn == ["self", "message_passing_layers", "node_embedder", "introduce_backwards_edges", "add_self_edges",
                   "edge_dropout_rate", "edge_feature_embedder"]


def test_reference_checkpoints_load():
    g = load_golden("gated_sum")
    layer = P.GatedMessagePassingLayer(32, 32, 4, "sum")
    layer.load_state_dict(golden_state_dict(g), strict=True)
    assert layer.input_state_dimension == 32 and layer.output_state_dimension == 32
    for name, kw in GOLDEN_MLP_KW.items():
        sd = golden_state_dict(load_golden(name))
        T = sum(1 for k in sd if k.endswith("_MLP__mlp_modules.1.weight"))
        P.MlpMessagePassingLayer(num_edge_types=T, **kw).load_state_dict(sd, strict=True)


def test_unsupported_configurations_fail_loudly():
    adj = [(torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.int64))]
    # training (SURVEY.md §8 f-1, tests/test_gpu_backward.py) exists for both layer classes -- on CUDA tensors only, fp32 only
    with pytest.raises(N.NativeLibraryError):
        P.MlpMessagePassingLayer(32, 32, 32, 1, "sum")(torch.zeros(4, 32), adj)
    with pytest.raises(N.NativeLibraryError):
        P.GatedMessagePassingLayer(32, 32, 1, "sum")(torch.zeros(4, 32), adj)
    with pytest.raises(NotImplementedError):  # ... not for bf16 states
        P.GatedMessagePassingLayer(32, 32, 1, "sum")(torch.zeros(4, 32, dtype=torch.bfloat16), adj)
    with pytest.raises(NotImplementedError):  # ... nor for message MLPs with hidden layers
        P.MlpMessagePassingLayer(32, 32, 32, 1, "sum", mlp_hidden_layers=1)(torch.zeros(4, 32), adj)
    with torch.no_grad():
        with pytest.raises(N.NativeLibraryError):  # training-mode dropout runs (per-edge mask on the gathered rows) -- on CUDA tensors
            P.GatedMessagePassingLayer(32, 32, 1, "sum", dropout_rate=0.5).train()(torch.zeros(4, 32), adj)
        with pytest.raises(N.NativeLibraryError):  # hidden MLP layers are supported (composed path) -- on CUDA tensors only
            P.MlpMessagePassingLayer(32, 32, 32, 1, "sum", mlp_hidden_layers=1).eval()(torch.zeros(4, 32), adj)
        with pytest.raises(NotImplementedError):  # unknown aggregation
            P.GatedMessagePassingLayer(32, 32, 1, "median").eval()(torch.zeros(4, 32), adj)
        with pytest.raises(ValueError):  # width mismatch is a shape error, not a read past the weight buffers (ADVICE r1)
            P.GatedMessagePassingLayer(32, 32, 1, "sum").eval()(torch.zeros(4, 64), adj)
        with pytest.raises(ValueError):
            P.MlpMessagePassingLayer(32, 32, 32, 1, "sum").eval()(torch.zeros(4, 32, 1), adj)


def test_per_graph_layers_refuse_before_building_the_plan():
    # On CPU tensors a call that gets as far as the graph plan raises NativeLibraryError; a refused call raises before it.
    n2g = torch.zeros(4, dtype=torch.int64)
    exchange = P.GruGlobalStateUpdate(P.SimpleVarSizedElementReduce("max"), 32, 32)      # GRUCell parameters: gradients are on
    for dtype in (torch.float16, torch.float64, torch.bfloat16):          # its readout and GRU kernels read fp32 states as they are
        with pytest.raises(NotImplementedError):
            exchange(torch.zeros(4, 32, dtype=dtype), [], n2g)
    with pytest.raises(N.NativeLibraryError):
        exchange(torch.zeros(4, 32), [], n2g)
    norm = P.GraphNorm(32)
    with pytest.raises(NotImplementedError):
        norm(torch.zeros(4, 32, dtype=torch.bfloat16), [], n2g)
    with pytest.raises(N.NativeLibraryError):                             # GraphNorm trains on an fp32 copy of fp64 states
        norm(torch.zeros(4, 32, dtype=torch.float64), [], n2g)
    with pytest.raises(NotImplementedError):                              # the layer's own checks come before the shape check
        P.MultiHeadSelfAttentionMessagePassing(32, 16, 16, 32, 64, 2, target_reference="tok")(torch.zeros(4, 48), [], n2g)


def test_container_metrics_protocol():
    layer = P.GatedMessagePassingLayer(32, 32, 3, "sum")
    gnn = P.GraphNeuralNetwork([layer, layer], torch.nn.Identity(), True, True)
    assert gnn.report_metrics() == {"num_graphs": 0, "num_nodes": 0, "num_edges": 0}
    assert gnn.input_node_state_dim == 32 and gnn.output_node_state_dim == 32
    assert len(gnn.message_passing_layers) == 2
    # weight sharing: the same module registered twice contributes its parameters once
    assert len(list(gnn.parameters())) == len(list(layer.parameters()))
    raw = [(torch.tensor([0, 1]), torch.tensor([1, 2]))]
    expanded = gnn.expand_adjacency(raw, 4, torch.device("cpu"))
    assert len(raw) == 1 and len(expanded) == 3  # caller's list is NOT mutated
    assert torch.equal(expanded[1][0], raw[0][1]) and torch.equal(expanded[2][0], torch.arange(4))


def test_weight_cache_bookkeeping_without_gpu(monkeypatch):
    """The derived-weight cache is keyed on (data_ptr, version) of every parameter: reuse only while nothing changed, never
    in training mode, never carried through deepcopy / pickling.  (The kernels behind it: tests/test_gpu_weight_cache.py.)"""
    import copy

    import ptgnn_b200 as P

    class _Stream:
        cuda_stream = 0

    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: _Stream())
    layer = P.GatedMessagePassingLayer(64, 64, 2, "sum").eval()
    params = list(layer.parameters())
    dev = torch.device("cpu")
    buf, valid = layer._weight_cache("f32", 1024, params, dev)
    assert buf is not None and not valid
    layer._weight_cache_filled("f32", dev)
    buf2, valid = layer._weight_cache("f32", 1024, params, dev)
    assert valid and buf2 is buf
    layer._weight_cache_filled("f32", dev)
    with torch.no_grad():
        params[0].mul_(2.0)                                   # what load_state_dict / an optimiser step does
    assert layer._weight_cache("f32", 1024, params, dev)[1] is False
    layer._weight_cache_filled("f32", dev)
    assert layer._weight_cache("f32", 1024, params, dev)[1] is True
    layer._weight_cache_filled("f32", dev)
    layer.train()
    assert layer._weight_cache("f32", 1024, params, dev)[1] is False       # never trusted in training mode
    layer.eval()
    assert layer._weight_cache("f32", 0, params, dev) == (None, False)     # nothing to cache for these dims
    assert copy.deepcopy(layer)._derived_weights == {}
    assert not any("derived" in k for k in layer.state_dict())
    layer.invalidate_weight_cache()
    assert layer._weight_cache("f32", 1024, params, dev)[1] is False


def test_bench_clock_summary_decodes_nvml_reason_bits():
    import importlib.util

    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    s = bench.ClockSampler(0)
    assert s.summary()["sm_mhz"] is None
    s.sm_max, s.source = 1965, "nvml"
    s.samples = [(1965, 300.0, 0x0), (1950, 320.0, 0x4), (1965, 310.0, 0x1), (1700, 330.0, 0x40)]
    out = s.summary()
    assert out["sm_mhz"] == 1965 and out["sm_max_mhz"] == 1965 and out["samples"] == 4
    assert out["reasons"] == ["hw_thermal_slowdown", "sw_power_cap"] and out["power_w_max"] == 330.0


def test_state_chain_bookkeeping_without_gpu():
    """edgeplan.state_chain: per-thread slot keyed on tensor identity + version; nests; other threads never see it.  (What the
    layers do with it: tests/test_gpu_round2.py::test_state_chain_*.)"""
    import threading

    from ptgnn_b200 import edgeplan as EP

    assert EP.current_state_chain() is None
    out, packed = torch.zeros(4, 8), torch.zeros(4, 32, dtype=torch.uint8)
    with EP.state_chain() as chain:
        assert EP.current_state_chain() is chain and chain.lookup(out) is None
        chain.store(out, packed)
        assert chain.lookup(out) is packed
        assert chain.lookup(out.clone()) is None                     # identity, not equality
        seen = []
        t = threading.Thread(target=lambda: seen.append(EP.current_state_chain()))
        t.start(); t.join()
        assert seen == [None]                                        # per thread
        with EP.state_chain() as inner:
            assert EP.current_state_chain() is inner and inner.lookup(out) is None
        assert EP.current_state_chain() is chain
        out.add_(1.0)                                                # in-place edit: the packed copy is stale
        assert chain.lookup(out) is None
        chain.store(out, None)                                       # a layer that produced no packed form clears the slot
        assert chain.lookup(out) is None
    assert EP.current_state_chain() is None


def test_minibatch_assembler_is_exported_and_egc_has_the_reference_signature():
    egc = list(inspect.signature(P.EGCMessagePassingLayer.__init__).parameters)
    assert egc == ["self", "input_state_dimension", "output_state_dimension", "num_edge_types", "message_aggregation_function",
                   "num_bases", "num_heads", "dropout_rate"]
    asm = P.MinibatchAssembler(3, stop_extending_minibatch_after_num_nodes=7)
    mb = asm.initialize_minibatch()
    assert sorted(mb) == ["adjacency_lists", "num_nodes_in_mb", "num_nodes_per_graph", "reference_node_ids"] and len(mb["adjacency_lists"]) == 3
