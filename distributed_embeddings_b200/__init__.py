"""H100-native (sm_90a) distributed embeddings.

Public API (capability parity with ``distributed_embeddings/__init__.py:17-27`` of the reference):
``Embedding``, ``IntegerLookup``, ``ConcatOneHotEmbedding``, ``embedding_lookup``,
``DistributedEmbedding``, ``DistEmbeddingStrategy``, ``broadcast_variables``,
``DistributedGradientTape``, ``DistributedOptimizer``, ``BroadcastGlobalVariablesCallback``;
``dist_model_parallel`` is importable as a namespace (``from distributed_embeddings_b200 import
dist_model_parallel as dmp``).
"""
import os as _os

# The step overlaps kernels of several streams (embedding exchange, MLP GEMMs, streamed gradient
# push, all-reduce); with the default of 8 hardware queues distinct streams alias onto one queue
# and serialise.  Only effective when set before the CUDA context is created.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

from .version import __version__
from .layers.embedding import ConcatOneHotEmbedding, Embedding, IntegerLookup
from .ops.embedding_lookup_ops import (embedding_lookup, integer_lookup, read_var_no_copy,
                                       row_to_split)
from .ops.ragged import RaggedIds, SparseIds
from .parallel import dist_model_parallel
from .parallel.comm import CommContext
from .parallel.dist_model_parallel import DistributedEmbedding, broadcast_variables
from .parallel.hybrid import (BroadcastGlobalVariablesCallback, DistributedGradientTape,
                              DistributedOptimizer, GradBucket, allreduce_gradients,
                              exclude_model_parallel_from_ddp)
from .parallel.strategy import DistEmbeddingStrategy

# the reference exposes the hybrid helpers through the dist_model_parallel module
dist_model_parallel.DistributedGradientTape = DistributedGradientTape
dist_model_parallel.DistributedOptimizer = DistributedOptimizer
dist_model_parallel.BroadcastGlobalVariablesCallback = BroadcastGlobalVariablesCallback
dist_model_parallel.allreduce_gradients = allreduce_gradients
dist_model_parallel.exclude_model_parallel_from_ddp = exclude_model_parallel_from_ddp

__all__ = [
    "Embedding", "IntegerLookup", "ConcatOneHotEmbedding", "embedding_lookup", "integer_lookup",
    "read_var_no_copy", "row_to_split", "RaggedIds", "SparseIds", "DistributedEmbedding",
    "DistEmbeddingStrategy", "broadcast_variables", "DistributedGradientTape",
    "DistributedOptimizer", "BroadcastGlobalVariablesCallback", "GradBucket",
    "allreduce_gradients", "exclude_model_parallel_from_ddp", "CommContext", "dist_model_parallel", "__version__"
]
