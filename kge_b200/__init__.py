"""kge_b200 — H100-native scoring engine for knowledge-graph embeddings.

One hot path of uma-pi1/kge (LibKGE), rebuilt as hand-written sm_90a CUDA behind a C ABI
(include/b200kge.h): embedding gather + relational scorer forward for ComplEx / DistMult / SimplE /
CP / RESCAL (wgmma tensor-core kernels, fp32-equivalent via an operand split) and TransE / RotatE (CUDA-core distance kernels), fused with BCE/KL
loss, rank/tie counting and negative-sample gather+score.  No CPU fallback.
"""
from . import _lib, engine, indexing  # noqa: F401
from .model import (KgeModel, ReciprocalRelationsModel, LookupEmbedder, RelationalScorer, KgeLoss,  # noqa: F401
                    BatchNegativeSample)
from .evaluate import EntityRankingEvaluator  # noqa: F401
from .indexing import KvsAllIndex  # noqa: F401

__all__ = ["engine", "indexing", "KgeModel", "ReciprocalRelationsModel", "LookupEmbedder", "RelationalScorer", "KgeLoss", "BatchNegativeSample",
           "EntityRankingEvaluator", "KvsAllIndex"]
