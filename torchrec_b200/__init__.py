"""torchrec_b200 - an H100-native (sm_90a) recommender-systems framework with the capabilities of TorchRec.

Top-level surface mirrors ``torchrec/__init__.py``: sparse types, embedding configs / modules, the distributed runtime (``torchrec_b200.distributed`` ==
``torchrec_b200.parallel``), quantization and the FX tracer. The CUDA extensions under ``ops/`` are built in-tree by ``__graft_entry__.build()`` and are
loaded on first use, not at import.
"""
from . import distributed  # noqa: F401  (alias of .parallel, installs the import hook)
from . import parallel  # noqa: F401
from . import quant  # noqa: F401
from .fx import tracer  # noqa: F401
from .modules.embedding_configs import DataType, EmbeddingBagConfig, EmbeddingConfig, PoolingType  # noqa: F401
from .modules.embedding_modules import EmbeddingBagCollection, EmbeddingBagCollectionInterface, EmbeddingCollection  # noqa: F401
from .sparse.jagged_tensor import JaggedTensor, KeyedJaggedTensor, KeyedTensor  # noqa: F401
from .streamable import Multistreamable, Pipelineable  # noqa: F401
from .version import __version__, github_version  # noqa: F401
