"""Distributed runtime: model parallelism for embedding tables on H100 (one process per GPU, NCCL + NVLink peer memory).

Mirrors the top-level surface of ``torchrec/distributed/__init__.py``; also importable as ``torchrec_b200.distributed``.

* ``DistributedModelParallel`` / ``DMPCollection`` - shard a model's embedding modules by a ``ShardingPlan``, data-parallel the rest.
* sharded modules (``embeddingbag.py``, ``embedding.py``, ...) on ONE lookup engine (``engine.py``) whose lookup + output dist are fused CUDA kernels
  over NVLink peer memory; the decomposed per-type form lives in ``sharding/`` + ``embedding_sharding.py`` + ``embedding_lookup.py``.
* collectives (``comm_ops.py``, ``dist_data.py``), planner (``planner/``), train pipelines (``train_pipeline/``).
"""
from .comm import get_local_rank, get_local_size  # noqa: F401
from .model_parallel import DistributedModelParallel, DMPCollection  # noqa: F401
from .train_pipeline import (  # noqa: F401
    DataLoadingThread,
    EvalPipelineSparseDist,
    PrefetchTrainPipelineSparseDist,
    TrainPipeline,
    TrainPipelineBase,
    TrainPipelineSparseDist,
)
from .types import (  # noqa: F401
    Awaitable,
    ModuleSharder,
    NoWait,
    ParameterSharding,
    ShardedModule,
    ShardedTensor,
    ShardingEnv,
    ShardingPlan,
    ShardingPlanner,
    ShardingType,
)
from .utils import get_unsharded_module_names, sharded_model_copy  # noqa: F401
