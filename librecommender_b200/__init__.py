"""librecommender_b200 — H100-native scoring / top-K engine behind LibRecommender's
``recommend_user`` hot path (see DESIGN.md).  Importing the package loads the
sm_90a shared library; it raises if the library is missing."""
from . import _lib  # noqa: F401  (fail loudly when the CUDA library is absent)
from .consumed import ConsumedCSR
from .recommendation import (
    construct_rec,
    rank_recommendations,
    recommend_from_embedding,
)

__all__ = [
    "ConsumedCSR",
    "construct_rec",
    "rank_recommendations",
    "recommend_from_embedding",
]
__version__ = "0.1.0"
