"""Evaluation entry points (``tools/evaluate.py``): CMC / mAP on device, optionally after k-reciprocal re-ranking."""
from ..ops.rank import (evaluate, evaluate_sharded, rank_metrics, rank_metrics_reference,  # noqa: F401
                        re_ranking, re_ranking_reference, similarity)
from .sharded import ShardedRanker  # noqa: F401


def calculate_similarity_distance(query_feature, gallery_features):
    """``tools/evaluate.py:87-100`` (single query against the gallery)."""
    import numpy as np
    if isinstance(query_feature, np.ndarray):
        return np.dot(gallery_features, query_feature)
    return (gallery_features.float() @ query_feature.float().view(-1, 1)).squeeze(1).cpu().numpy()
