"""Makes the reference's own packages run on the ptgnn_b200 kernels WITHOUT editing them.

The reference constructs its GNN by class name (`/root/reference/ptgnn/neuralmodels/gnn/graphneuralnetwork.py:298-305`), its
factories import the layer classes by module path (`implementations/typilus/train.py:24-33`, `ppi/train.py:31-32`,
`varmisuse/train.py:17-25`) and its modules import ``torch_scatter`` by name (`abstractmessagepassing.py:4`).  ``install()``

1. registers ``ptgnn_b200.torch_scatter_shim`` as ``torch_scatter`` (if the real wheel is absent, or ``force_torch_scatter``),
2. pre-seeds ``sys.modules`` so that ``ptgnn.neuralmodels.gnn.messagepassing.{abstract,gated,mlp}messagepassing`` and
   ``...globalgraphexchange`` resolve to the ptgnn_b200 classes (everything else -- residual layers, PNA (unless step 8), GraphNorm (unless
   step 7), embedders, trainers, and the reducers of ``reduceops.varsizedsummary``, whose attention variants must keep working -- stays the
   reference's; the native ``GruGlobalStateUpdate`` reads the reference's WeightedSum and Simple reducers directly), and
   re-binds those names in reference modules that were imported earlier,
3. replaces ``GraphNeuralNetwork`` inside the reference's ``graphneuralnetwork`` module (``GraphNeuralNetworkModel`` stays),
4. registers the ptgnn_b200 container as a (virtual) ``ModuleWithMetrics`` so that a reference parent's ``report_metrics()`` /
   ``reset_metrics()`` see its ``num_graphs / num_nodes / num_edges`` (`baseneuralmodel/modulewithmetrics.py:44-57`),
5. with ``native_reducers=True`` only: re-binds ``SelfAttentionVarSizedElementReduce`` and
   ``MultiheadSelfAttentionVarSizedElementReduce`` in ``ptgnn.neuralmodels.reduceops.varsizedsummary``, in ``ptgnn.neuralmodels.reduceops``
   and in reference modules imported earlier, so that e.g. ``ptgnn.implementations.graph2seq`` builds its graph summary on the native
   attention readout.  The default leaves every reducer the reference's,
6. with ``native_selfattention=True`` only: pre-seeds / re-binds ``MultiHeadSelfAttentionMessagePassing`` at
   ``ptgnn.neuralmodels.gnn.messagepassing.selfattmessagepassing`` (the native chunked attention kernel, DESIGN.md §3.8) like the
   layers of step 2.  The default leaves the reference's class in place,
7. with ``native_graphnorm=True`` only: pre-seeds / re-binds ``GraphNorm`` at ``ptgnn.neuralmodels.gnn.messagepassing.graphnorm``
   (the native per-graph normalisation kernels, DESIGN.md §3.9) in the same way.  The default leaves the reference's class in place,
8. with ``native_pna=True`` only: pre-seeds / re-binds ``PnaMessageAggregation`` at
   ``ptgnn.neuralmodels.gnn.messagepassing.pna_aggregation`` (the native PNA kernel, DESIGN.md §3.10) in the same way, so that an
   ``MlpMessagePassingLayer`` built with it runs PNA on the kernel and trains.  The default leaves the reference's class in place,
9. with ``native_decoder=True`` only: re-binds ``GruCopyingDecoder`` inside ``ptgnn.neuralmodels.sequence.grucopydecoder`` and in
   reference modules imported earlier (the native copy and memory attention kernels, DESIGN.md §3.11), so that
   ``GruCopyingDecoderModel.build_neural_module`` builds the native class.  The module itself stays the reference's: it also holds
   ``DecoderData``, ``TokenizedOutput`` and ``GruCopyingDecoderModel``, which graph2seq imports.  The default leaves the reference's
   class in place,
10. with ``native_embedders=True`` only: re-binds ``TokenUnitEmbedder`` and ``SubtokenUnitEmbedder`` inside
   ``ptgnn.neuralmodels.embeddings.strelementrepresentationmodel`` and in reference modules imported earlier (the native
   embedding-bag kernels, DESIGN.md §3.12), so that ``StrElementRepresentationModel.build_neural_module`` builds the native classes for
   ``"token"``, ``"subtoken"`` and ``"bpe"``.  The module stays the reference's: it also holds ``StrElementRepresentationModel``,
   ``CnnConfig`` and ``CharUnitEmbedder``, which ``"char"`` still builds.  The default leaves the reference's classes in place,
11. with ``native_char_embedder=True`` only: re-binds ``CharUnitEmbedder`` inside the same module and in reference modules imported
   earlier (the native character-CNN kernel, DESIGN.md §3.13), so that ``"char"`` (VarMisuse's ``CandidateNodeAnnotationModel``) builds
   the native class.  ``native_embedders=True`` alone leaves the reference's ``CharUnitEmbedder`` in place,
12. with ``native_egc=True`` only: pre-seeds / re-binds ``EGCMessagePassingLayer`` at
   ``ptgnn.neuralmodels.gnn.messagepassing.egcmessagepassing`` (the fused aggregation kernel with the EGC write-out, DESIGN.md §3.14) in
   the same way as step 8, so that a GNN built with EGC layers runs them natively and trains.  The default leaves the reference's class
   in place,
13. with ``native_feature_embedder=True`` only: re-binds ``LinearFeatureEmbedder`` inside
   ``ptgnn.neuralmodels.embeddings.linearmapembedding`` and in reference modules imported earlier (the native feature-embedding kernel,
   DESIGN.md §3.15), so that ``FeatureRepresentationModel.build_neural_module`` (the PPI model's node embedder) builds the native class.
   The module stays the reference's: it also holds ``FeatureRepresentationModel``.  The default leaves the reference's class in place.

After ``install()``: ``import ptgnn.implementations.ppi.train`` etc. build ptgnn_b200 layers, unchanged.  ``uninstall()``
restores the reference's classes.  The reference must be importable as ``ptgnn`` for steps 2-4 (it is not on the GPU test box;
``install()`` then only does step 1 and says so in its report).
"""
import importlib
import sys
import types
from typing import Dict

from . import globalexchange as _gx
from . import gnn as _gnn
from . import messagepassing as _mp

_LAYER_MODULES = {
    "ptgnn.neuralmodels.gnn.messagepassing.abstractmessagepassing": ("AbstractMessagePassingLayer", "AbstractMessageAggregation"),
    "ptgnn.neuralmodels.gnn.messagepassing.gatedmessagepassing": ("GatedMessagePassingLayer",),
    "ptgnn.neuralmodels.gnn.messagepassing.mlpmessagepassing": ("MlpMessagePassingLayer",),
    "ptgnn.neuralmodels.gnn.messagepassing.globalgraphexchange": ("AbstractGlobalGraphExchange", "GruGlobalStateUpdate"),
}
_REDUCER_MODULES = ("ptgnn.neuralmodels.reduceops.varsizedsummary", "ptgnn.neuralmodels.reduceops")
_NATIVE_REDUCERS = ("SelfAttentionVarSizedElementReduce", "MultiheadSelfAttentionVarSizedElementReduce")
_SELFATT_MODULE = "ptgnn.neuralmodels.gnn.messagepassing.selfattmessagepassing"
_SELFATT_CLASS = "MultiHeadSelfAttentionMessagePassing"
_GRAPHNORM_MODULE = "ptgnn.neuralmodels.gnn.messagepassing.graphnorm"
_GRAPHNORM_CLASS = "GraphNorm"
_PNA_MODULE = "ptgnn.neuralmodels.gnn.messagepassing.pna_aggregation"
_PNA_CLASS = "PnaMessageAggregation"
_DECODER_MODULE = "ptgnn.neuralmodels.sequence.grucopydecoder"
_EMBEDDER_MODULE = "ptgnn.neuralmodels.embeddings.strelementrepresentationmodel"
_NATIVE_EMBEDDERS = ("TokenUnitEmbedder", "SubtokenUnitEmbedder")
_NATIVE_CHAR_EMBEDDER = "CharUnitEmbedder"
_EGC_MODULE = "ptgnn.neuralmodels.gnn.messagepassing.egcmessagepassing"
_EGC_CLASS = "EGCMessagePassingLayer"
_FEATURE_EMBEDDER_MODULE = "ptgnn.neuralmodels.embeddings.linearmapembedding"
_FEATURE_EMBEDDER_CLASS = "LinearFeatureEmbedder"
_saved: Dict[str, object] = {}


def _reference_importable() -> bool:
    try:
        return importlib.util.find_spec("ptgnn") is not None
    except (ImportError, ValueError):
        return False


def _native_class(name: str):
    return getattr(_mp, name) if hasattr(_mp, name) else getattr(_gx, name)


def _stub_module(name: str, names) -> types.ModuleType:
    m = types.ModuleType(name, f"ptgnn_b200 overlay of the reference module {name}")
    for n in names:
        setattr(m, n, _native_class(n))
    m.__ptgnn_b200_overlay__ = True
    return m


def _rebind_everywhere(replaced: Dict[object, object]) -> None:
    """Re-binds the values of ``replaced`` in every imported reference module (``from ... import X`` bindings made earlier)."""
    for mod_name, mod in list(sys.modules.items()):
        if mod is None or not mod_name.startswith("ptgnn.") or getattr(mod, "__ptgnn_b200_overlay__", False):
            continue
        for attr, val in list(vars(mod).items()):
            try:
                new = replaced.get(val)
            except TypeError:        # unhashable module attribute
                continue
            if new is not None:
                _saved.setdefault(f"{mod_name}:{attr}", val)
                setattr(mod, attr, new)


def _install_native_reducers() -> None:
    from . import reduceops as _ro

    importlib.import_module(_REDUCER_MODULES[0])
    replaced = {}
    for mod_name in _REDUCER_MODULES:
        mod = sys.modules[mod_name]
        for n in _NATIVE_REDUCERS:
            old = getattr(mod, n, None)
            if old is not None and old is not getattr(_ro, n):
                replaced[old] = getattr(_ro, n)
    _rebind_everywhere(replaced)       # the two reducer modules included


def _install_native_class(mod_name: str, class_name: str, native) -> None:
    """Pre-seeds ``mod_name`` with a module holding only ``native`` as ``class_name`` and re-binds the reference's class wherever an
    earlier import bound it; ``uninstall()`` restores the reference's module."""
    replaced = {}
    old = sys.modules.get(mod_name)
    if old is not None and not getattr(old, "__ptgnn_b200_overlay__", False):
        _saved[mod_name] = old
        if hasattr(old, class_name):
            replaced[getattr(old, class_name)] = native
    m = types.ModuleType(mod_name, f"ptgnn_b200 overlay of the reference module {mod_name}")
    setattr(m, class_name, native)
    m.__ptgnn_b200_overlay__ = True
    sys.modules[mod_name] = m
    _rebind_everywhere(replaced)


def _install_native_selfattention() -> None:
    from . import selfattention as _sa

    _install_native_class(_SELFATT_MODULE, _SELFATT_CLASS, getattr(_sa, _SELFATT_CLASS))


def _install_native_graphnorm() -> None:
    from . import graphnorm as _gn

    _install_native_class(_GRAPHNORM_MODULE, _GRAPHNORM_CLASS, getattr(_gn, _GRAPHNORM_CLASS))


def _install_native_pna() -> None:
    from . import aggregation as _agg

    _install_native_class(_PNA_MODULE, _PNA_CLASS, getattr(_agg, _PNA_CLASS))


def _install_native_egc() -> None:
    from . import egc as _egc

    _install_native_class(_EGC_MODULE, _EGC_CLASS, getattr(_egc, _EGC_CLASS))


def _install_native_decoder() -> None:
    from . import decoder as _dec

    old = importlib.import_module(_DECODER_MODULE).GruCopyingDecoder
    if old is not _dec.GruCopyingDecoder:
        _rebind_everywhere({old: _dec.GruCopyingDecoder})      # the decoder module included


def _install_native_embedders(names=_NATIVE_EMBEDDERS) -> None:
    from . import embeddings as _emb

    mod = importlib.import_module(_EMBEDDER_MODULE)
    replaced = {getattr(mod, n): getattr(_emb, n) for n in names if getattr(mod, n) is not getattr(_emb, n)}
    _rebind_everywhere(replaced)       # the embedder module included


def _install_native_feature_embedder() -> None:
    from . import embeddings as _emb

    old = getattr(importlib.import_module(_FEATURE_EMBEDDER_MODULE), _FEATURE_EMBEDDER_CLASS)
    if old is not _emb.LinearFeatureEmbedder:
        _rebind_everywhere({old: _emb.LinearFeatureEmbedder})      # the embedder module included


def install(force_torch_scatter: bool = False, native_reducers: bool = False, native_selfattention: bool = False,
            native_graphnorm: bool = False, native_pna: bool = False, native_decoder: bool = False,
            native_embedders: bool = False, native_char_embedder: bool = False, native_egc: bool = False,
            native_feature_embedder: bool = False) -> Dict[str, object]:
    report: Dict[str, object] = {"torch_scatter": "real", "layers": False, "container": False, "metrics": False, "reducers": False,
                                 "selfattention": False, "graphnorm": False, "pna": False, "decoder": False, "embedders": False,
                                 "char_embedder": False, "egc": False, "feature_embedder": False}
    # 1. torch_scatter
    have_real = False
    if not force_torch_scatter:
        try:
            have_real = importlib.util.find_spec("torch_scatter") is not None and not getattr(sys.modules.get("torch_scatter"), "__ptgnn_b200_overlay__", False)
        except (ImportError, ValueError):
            have_real = False
    if not have_real:
        from . import torch_scatter_shim as shim

        shim.__ptgnn_b200_overlay__ = True
        sys.modules["torch_scatter"] = shim
        sys.modules["torch_scatter.composite"] = shim.composite
        report["torch_scatter"] = "ptgnn_b200.torch_scatter_shim"
    if not _reference_importable():
        report["note"] = "reference package `ptgnn` not importable: only the torch_scatter shim was installed"
        return report
    # 2. layer modules: replace already-imported reference classes, pre-seed the ones not imported yet
    replaced = {}
    for mod_name, names in _LAYER_MODULES.items():
        old = sys.modules.get(mod_name)
        if old is not None and not getattr(old, "__ptgnn_b200_overlay__", False):
            _saved[mod_name] = old
            for n in names:
                if hasattr(old, n):
                    replaced[getattr(old, n)] = _native_class(n)
        sys.modules[mod_name] = _stub_module(mod_name, names)
    _rebind_everywhere(replaced)       # `from ... import GatedMessagePassingLayer` bindings made earlier
    report["layers"] = True
    # 3. the container class inside the reference's graphneuralnetwork module (GraphNeuralNetworkModel looks it up at call time)
    ref_gnn = importlib.import_module("ptgnn.neuralmodels.gnn.graphneuralnetwork")
    if ref_gnn.GraphNeuralNetwork is not _gnn.GraphNeuralNetwork:
        _saved["container"] = ref_gnn.GraphNeuralNetwork
        ref_gnn.GraphNeuralNetwork = _gnn.GraphNeuralNetwork
    pkg = sys.modules.get("ptgnn.neuralmodels.gnn")
    if pkg is not None and getattr(pkg, "GraphNeuralNetwork", None) is _saved.get("container"):
        pkg.GraphNeuralNetwork = _gnn.GraphNeuralNetwork
    report["container"] = True
    # 4. metrics protocol
    report["metrics"] = _gnn.register_with_reference_metrics()
    # 5. the attention reducers (opt-in)
    if native_reducers:
        _install_native_reducers()
        report["reducers"] = True
    # 6. the self-attention layer (opt-in)
    if native_selfattention:
        _install_native_selfattention()
        report["selfattention"] = True
    # 7. GraphNorm (opt-in)
    if native_graphnorm:
        _install_native_graphnorm()
        report["graphnorm"] = True
    # 8. PnaMessageAggregation (opt-in)
    if native_pna:
        _install_native_pna()
        report["pna"] = True
    # 9. GruCopyingDecoder (opt-in)
    if native_decoder:
        _install_native_decoder()
        report["decoder"] = True
    # 10. TokenUnitEmbedder / SubtokenUnitEmbedder (opt-in)
    if native_embedders:
        _install_native_embedders()
        report["embedders"] = True
    # 11. CharUnitEmbedder (opt-in)
    if native_char_embedder:
        _install_native_embedders((_NATIVE_CHAR_EMBEDDER,))
        report["char_embedder"] = True
    # 12. EGCMessagePassingLayer (opt-in)
    if native_egc:
        _install_native_egc()
        report["egc"] = True
    # 13. LinearFeatureEmbedder (opt-in)
    if native_feature_embedder:
        _install_native_feature_embedder()
        report["feature_embedder"] = True
    return report


def uninstall() -> None:
    for key, val in list(_saved.items()):
        if key == "container":
            ref_gnn = sys.modules.get("ptgnn.neuralmodels.gnn.graphneuralnetwork")
            if ref_gnn is not None:
                ref_gnn.GraphNeuralNetwork = val
            pkg = sys.modules.get("ptgnn.neuralmodels.gnn")
            if pkg is not None and getattr(pkg, "GraphNeuralNetwork", None) is _gnn.GraphNeuralNetwork:
                pkg.GraphNeuralNetwork = val
        elif ":" in key:
            mod_name, attr = key.split(":", 1)
            if mod_name in sys.modules:
                setattr(sys.modules[mod_name], attr, val)
        else:
            sys.modules[key] = val
    for mod_name in (*_LAYER_MODULES, _SELFATT_MODULE, _GRAPHNORM_MODULE, _PNA_MODULE, _EGC_MODULE):
        if getattr(sys.modules.get(mod_name), "__ptgnn_b200_overlay__", False):
            del sys.modules[mod_name]
    for name in ("torch_scatter", "torch_scatter.composite"):
        if getattr(sys.modules.get(name), "__ptgnn_b200_overlay__", False) or name.endswith("composite"):
            mod = sys.modules.get(name)
            if mod is not None and mod.__name__.startswith("ptgnn_b200."):
                del sys.modules[name]
    _saved.clear()
