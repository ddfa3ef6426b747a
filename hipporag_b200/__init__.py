"""hipporag_b200 -- HippoRAG's online retrieval hot path (embedding similarity -> seeds ->
Personalized PageRank -> top-k passages) as hand-written CUDA for H100 (sm_90a), behind the
reference's own ``HippoRAG.retrieve()`` API.  See DESIGN.md / INTEGRATION.md."""
from ._lib import (HragError, PPR_CHEBYSHEV, PPR_FP32, PPR_MIXED, PPR_POWER, SIM_BF16, SIM_BF16X3,  # noqa: F401
                   SIM_FP32)
from .accelerate import accelerate, share  # noqa: F401
from .engine import B200Retriever, Engine, balanced_row_bounds, build_transition_csr, shard_rows  # noqa: F401

__all__ = ["accelerate", "share", "Engine", "B200Retriever", "HragError", "build_transition_csr", "shard_rows", "balanced_row_bounds",
           "PPR_POWER", "PPR_CHEBYSHEV", "PPR_FP32", "PPR_MIXED", "SIM_FP32", "SIM_BF16X3", "SIM_BF16"]
