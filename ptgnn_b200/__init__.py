"""ptgnn_b200 -- H100-native (sm_90a) implementation of microsoft/ptgnn's sparse message-passing hot path.

Scope (BASELINE.json ``north_star``, SURVEY.md §8): ``GatedMessagePassingLayer`` / ``MlpMessagePassingLayer``,
the ``GraphNeuralNetwork`` layer loop and the ``torch_scatter.scatter`` boundary below them, behind the reference's
own ``nn.Module`` API.  The arithmetic lives in ``libptgnn_b200.so`` (C ABI: ``include/ptgnn_b200.h``); this package
is the host-side mirror of the reference interface.  There is no CPU / PyTorch fallback.
"""
from .aggregation import PnaMessageAggregation
from .batching import MinibatchAssembler
from .decoder import GruCopyingDecoder
from .embeddings import CharUnitEmbedder, LinearFeatureEmbedder, SubtokenUnitEmbedder, TokenUnitEmbedder
from .edgeplan import EdgePlan, clear_plan_cache, plan_for
from .egc import EGCMessagePassingLayer
from .globalexchange import AbstractGlobalGraphExchange, GruGlobalStateUpdate
from .gnn import GnnOutput, GraphNeuralNetwork
from .messagepassing import (
    MLP,
    AbstractMessageAggregation,
    AbstractMessagePassingLayer,
    GatedMessagePassingLayer,
    MlpMessagePassingLayer,
)
from .reduceops import (
    AbstractVarSizedElementReduce,
    ElementsToSummaryRepresentationInput,
    MultiheadSelfAttentionVarSizedElementReduce,
    SelfAttentionVarSizedElementReduce,
    SimpleVarSizedElementReduce,
    WeightedSumVarSizedElementReduce,
)
from .selfattention import MultiHeadSelfAttentionMessagePassing
from .graphnorm import GraphNorm
from .residuallayers import ConcatResidualLayer, LinearResidualLayer, MeanResidualLayer
from .scatter import scatter, scatter_add, scatter_max, scatter_mean, scatter_min, scatter_sum

__all__ = [
    "EdgePlan", "plan_for", "clear_plan_cache", "GnnOutput", "GraphNeuralNetwork", "MLP", "AbstractMessageAggregation",
    "PnaMessageAggregation", "AbstractMessagePassingLayer", "GatedMessagePassingLayer", "MlpMessagePassingLayer", "EGCMessagePassingLayer", "MeanResidualLayer",
    "ConcatResidualLayer", "LinearResidualLayer", "MinibatchAssembler", "scatter", "scatter_add",
    "AbstractGlobalGraphExchange", "GruGlobalStateUpdate", "AbstractVarSizedElementReduce", "ElementsToSummaryRepresentationInput",
    "SimpleVarSizedElementReduce", "WeightedSumVarSizedElementReduce", "SelfAttentionVarSizedElementReduce",
    "MultiheadSelfAttentionVarSizedElementReduce", "MultiHeadSelfAttentionMessagePassing", "GraphNorm", "GruCopyingDecoder",
    "TokenUnitEmbedder", "SubtokenUnitEmbedder", "CharUnitEmbedder", "LinearFeatureEmbedder",
    "scatter_sum", "scatter_mean", "scatter_max", "scatter_min",
]
