"""Inference preparation: quantize + shard a trained model, predict module / factory contracts
(reference torchrec/inference/modules.py:121-659)."""
from __future__ import annotations

import abc
import copy
import itertools
import logging
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple, Type, Union

import torch
import torch.nn as nn

from ..modules.embedding_configs import DataType, QuantConfig, data_type_to_dtype, dtype_to_data_type
from ..modules.embedding_modules import EmbeddingBagCollection, EmbeddingBagCollectionInterface, EmbeddingCollection, EmbeddingCollectionInterface
from ..quant.embedding_modules import EmbeddingBagCollection as QuantEmbeddingBagCollection
from ..quant.embedding_modules import EmbeddingCollection as QuantEmbeddingCollection
from ..quant.embedding_modules import MODULE_ATTR_EMB_CONFIG_NAME_TO_NUM_ROWS_POST_PRUNING_DICT, quant_prep_enable_register_tbes

logger = logging.getLogger(__name__)

DEFAULT_FUSED_PARAMS: Dict[str, Any] = {"register_tbes": True, "quant_state_dict_split_scale_bias": True}
DEFAULT_SHARDERS_NAMES = ("QuantEmbeddingBagCollectionSharder", "QuantEmbeddingCollectionSharder")
DEFAULT_QUANT_MAPPING: Dict[str, Type[torch.nn.Module]] = {}


def trim_torch_package_prefix_from_typename(typename: str) -> str:
    if typename.startswith("<torch_package_"):
        typename = ".".join(typename.split(".")[1:])
    return typename


@dataclass
class BatchingMetadata:
    """How the serving runtime batches one input of the model: ``type`` in {dense, sparse, embedding}."""

    type: str
    device: str
    pinned: List[str]


@dataclass
class QualNameMetadata:
    """Per-submodule serving metadata keyed by qualified name: does the runtime have to run a pre-processing module in front of it?"""

    need_preproc: bool


class PredictFactory(abc.ABC):
    """Creates the (already quantized / sharded) predict module inside the serving process."""

    @abc.abstractmethod
    def create_predict_module(self) -> nn.Module:
        ...

    @abc.abstractmethod
    def batching_metadata(self) -> Dict[str, BatchingMetadata]:
        ...

    def batching_metadata_json(self) -> str:
        import json

        return json.dumps({k: {"type": v.type, "device": v.device, "pinned": v.pinned} for k, v in self.batching_metadata().items()})

    @abc.abstractmethod
    def result_metadata(self) -> str:
        ...

    @abc.abstractmethod
    def run_weights_independent_tranformations(self, predict_module: torch.nn.Module) -> torch.nn.Module:
        ...

    @abc.abstractmethod
    def run_weights_dependent_transformations(self, predict_module: torch.nn.Module) -> torch.nn.Module:
        ...

    def qualname_metadata(self) -> Dict[str, QualNameMetadata]:
        return {}

    def qualname_metadata_json(self) -> str:
        import json

        return json.dumps({k: {"need_preproc": bool(v.need_preproc)} for k, v in self.qualname_metadata().items()})

    def model_inputs_data(self) -> Dict[str, Any]:
        return {}


class PredictModule(nn.Module):
    """Wraps a model for serving: ``forward(batch: Dict[str, Tensor]) -> Any`` runs ``predict_forward`` under
    ``inference_mode`` on the module's device."""

    def __init__(self, module: nn.Module, device: Optional[str] = None) -> None:
        super().__init__()
        self._module: nn.Module = module
        self._device: Optional[torch.device] = torch.device(device) if device is not None else None
        self._module.eval()

    @property
    def predict_module(self) -> nn.Module:
        return self._module

    @abc.abstractmethod
    def predict_forward(self, batch: Dict[str, torch.Tensor]) -> Any:
        ...

    def forward(self, batch: Dict[str, torch.Tensor]) -> Any:
        if self._device is None:
            self._device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        with torch.inference_mode():
            return self.predict_forward(batch)

    def state_dict(self, destination=None, prefix: str = "", keep_vars: bool = False) -> Dict[str, Any]:
        return self._module.state_dict(destination=destination, prefix=prefix, keep_vars=keep_vars)


def quantize_feature(module: torch.nn.Module, inputs: Tuple[torch.Tensor, ...]) -> Tuple[torch.Tensor, ...]:
    return tuple(inp.half() if isinstance(inp, torch.Tensor) and inp.dtype in (torch.float32, torch.float64) else inp for inp in inputs)


def quantize_embeddings(module: nn.Module, dtype: Union[torch.dtype, DataType], inplace: bool, additional_qconfig_spec_keys: Optional[List[Type[nn.Module]]] = None,
                        additional_mapping: Optional[Dict[Type[nn.Module], Type[nn.Module]]] = None, output_dtype: torch.dtype = torch.float,
                        per_table_weight_dtype: Optional[Dict[str, Union[torch.dtype, DataType]]] = None) -> nn.Module:
    """Swap float EmbeddingBagCollection / EmbeddingCollection modules for their quantized versions."""
    qconfig = QuantConfig(activation=output_dtype, weight=dtype, per_table_weight_dtype=per_table_weight_dtype)
    from ..modules.fp_embedding_modules import FeatureProcessedEmbeddingBagCollection
    from ..modules.mc_embedding_modules import ManagedCollisionEmbeddingBagCollection, ManagedCollisionEmbeddingCollection
    from ..quant.embedding_modules import FeatureProcessedEmbeddingBagCollection as QuantFeatureProcessedEmbeddingBagCollection
    from ..quant.embedding_modules import QuantManagedCollisionEmbeddingBagCollection, QuantManagedCollisionEmbeddingCollection

    mapping: Dict[Type[nn.Module], Type[nn.Module]] = {EmbeddingBagCollection: QuantEmbeddingBagCollection, EmbeddingCollection: QuantEmbeddingCollection,
                                                       FeatureProcessedEmbeddingBagCollection: QuantFeatureProcessedEmbeddingBagCollection,
                                                       ManagedCollisionEmbeddingCollection: QuantManagedCollisionEmbeddingCollection,
                                                       ManagedCollisionEmbeddingBagCollection: QuantManagedCollisionEmbeddingBagCollection}
    if additional_mapping is not None:
        mapping.update(additional_mapping)
    if not inplace:
        module = copy.deepcopy(module)

    def swap(m: nn.Module) -> nn.Module:
        if type(m) in mapping:
            m.qconfig = qconfig  # type: ignore[assignment]
            return mapping[type(m)].from_float(m)  # type: ignore[attr-defined]
        for name, child in list(m.named_children()):
            setattr(m, name, swap(child))
        return m

    return swap(module)


def quantize_dense(predict_module: nn.Module, dtype: torch.dtype, additional_embedding_module_type: Optional[List[Type[nn.Module]]] = None) -> nn.Module:
    """Cast the dense (non-embedding) parameters to ``dtype`` (fp16 / bf16 serving).

    ``dtype=torch.float8_e4m3fn`` instead swaps every ``MLP`` and ``LowRankCrossNet`` outside the embedding collections for its FP8
    inference form (``quant.dense_modules``: ``Fp8MLP``, ``Fp8LowRankCrossNet``) and leaves every other parameter as it is. An MLP
    without an FP8-eligible layer and a cross net whose width or rank is not a multiple of 16 stay unchanged."""
    skip = (EmbeddingBagCollectionInterface, EmbeddingCollectionInterface) + tuple(additional_embedding_module_type or [])
    if dtype == torch.float8_e4m3fn:
        from ..quant.dense_modules import Fp8LowRankCrossNet, Fp8MLP

        def swap(m: nn.Module) -> nn.Module:
            if isinstance(m, skip):
                return m
            if Fp8MLP.eligible(m):
                return Fp8MLP.from_float(m)
            if Fp8LowRankCrossNet.eligible(m):
                return Fp8LowRankCrossNet.from_float(m)
            for name, child in list(m.named_children()):
                setattr(m, name, swap(child))
            return m

        return swap(predict_module)

    def cast(m: nn.Module) -> None:
        if isinstance(m, skip):
            return
        for n, p in list(m._parameters.items()):
            if p is not None and p.is_floating_point():
                m._parameters[n] = nn.Parameter(p.detach().to(dtype), requires_grad=False)
        for n, b in list(m._buffers.items()):
            if b is not None and b.is_floating_point():
                m._buffers[n] = b.to(dtype)
        for c in m.children():
            cast(c)

    cast(predict_module)
    return predict_module


def quantize_inference_model(model: torch.nn.Module, quantization_mapping: Optional[Dict[str, Type[torch.nn.Module]]] = None,
                             per_table_weight_dtype: Optional[Dict[str, Union[torch.dtype, DataType]]] = None, fp_weight_dtype: Union[torch.dtype, DataType] = DataType.INT8,
                             quantization_dtype: Union[torch.dtype, DataType] = DataType.INT8, output_dtype: torch.dtype = torch.float) -> torch.nn.Module:
    """Quantize every embedding collection of a trained model for serving (module swap, per-table dtypes).

    Example::

        quant_model = quantize_inference_model(dlrm, per_table_weight_dtype={"t_big": DataType.INT4})
        sharded_model, plan = shard_quant_model(quant_model, world_size=torch.cuda.device_count())
    """
    additional = None
    if quantization_mapping:
        additional = {}
        for m in model.modules():
            nm = trim_torch_package_prefix_from_typename(torch.typename(m))
            if nm in quantization_mapping:
                additional[type(m)] = quantization_mapping[nm]
    return quantize_embeddings(model, dtype=quantization_dtype, inplace=True, additional_mapping=additional, output_dtype=output_dtype,
                               per_table_weight_dtype=per_table_weight_dtype)


def shard_quant_model(model: torch.nn.Module, world_size: int = 1, compute_device: str = "cuda", sharding_device: str = "meta",
                      sharders: Optional[List[Any]] = None, device_memory_size: Optional[int] = None, constraints: Optional[Dict[str, Any]] = None,
                      ddr_cap: Optional[int] = None, sharding_plan: Optional[Any] = None) -> Tuple[torch.nn.Module, Any]:
    """Plan (inference cost model, no reservation; or take ``sharding_plan``) and shard a quantized model over ``world_size`` local devices."""
    from ..parallel.planner import EmbeddingShardingPlanner, Topology
    from ..parallel.planner.enumerators import EmbeddingEnumerator, EmbeddingPerfEstimator, EmbeddingStorageEstimator
    from ..parallel.planner.storage_reservations import FixedPercentageStorageReservation
    from ..parallel.quant_embedding import QuantEmbeddingCollectionSharder
    from ..parallel.quant_embeddingbag import QuantEmbeddingBagCollectionSharder
    from ..parallel.shard import _shard_modules
    from ..parallel.types import ShardingEnv

    if constraints is None:
        constraints = {}
    if sharders is None:
        from ..parallel.quant_embedding import QuantManagedCollisionEmbeddingCollectionSharder
        from ..parallel.quant_embeddingbag import QuantFeatureProcessedEmbeddingBagCollectionSharder, QuantManagedCollisionEmbeddingBagCollectionSharder

        sharders = [QuantEmbeddingBagCollectionSharder(), QuantEmbeddingCollectionSharder(), QuantFeatureProcessedEmbeddingBagCollectionSharder(),
                    QuantManagedCollisionEmbeddingCollectionSharder(), QuantManagedCollisionEmbeddingBagCollectionSharder()]
    if compute_device == "cuda" and not torch.cuda.is_available():
        compute_device = "cpu"
    topology = Topology(world_size=world_size, compute_device=compute_device, local_world_size=world_size, hbm_cap=device_memory_size, ddr_cap=ddr_cap)
    enumerator = EmbeddingEnumerator(topology=topology, batch_size=1, constraints=constraints,
                                     estimator=[EmbeddingPerfEstimator(topology=topology, constraints=constraints, is_inference=True),
                                                EmbeddingStorageEstimator(topology=topology, constraints=constraints, is_inference=True)])
    planner = EmbeddingShardingPlanner(topology=topology, batch_size=1, enumerator=enumerator, storage_reservation=FixedPercentageStorageReservation(percentage=0.0),
                                       constraints=constraints)
    plan = sharding_plan if sharding_plan is not None else planner.plan(model, sharders)
    sharded = _shard_modules(module=model, device=torch.device(compute_device), sharders=sharders, env=ShardingEnv.from_local(world_size=world_size, rank=0), plan=plan)
    return sharded, plan


MODULE_ATTR_EMB_CONFIG_NAME_TO_NUM_ROWS_POST_PRUNING_DICT = "__emb_name_to_num_rows_post_pruning"


def set_pruning_data(model: torch.nn.Module, tables_to_rows_post_pruning: Dict[str, int], module_types: Optional[List[Type[nn.Module]]] = None) -> torch.nn.Module:
    """Record the post-pruning row counts of embedding tables (produced by ITEP / offline pruning) on the collections of ``model``: the
    quantized modules built from them allocate ``num_embeddings_post_pruning`` rows instead of ``num_embeddings`` and remap ids through the
    pruning index at lookup time. Both the module attribute of the reference and the per-table config field are set."""
    from ..modules.embedding_modules import EmbeddingBagCollection, EmbeddingCollection

    types = tuple(module_types) if module_types is not None else (EmbeddingBagCollection, EmbeddingCollection)
    for m in model.modules():
        if isinstance(m, types) or type(m).__name__ == "FeatureProcessedEmbeddingBagCollection":
            setattr(m, MODULE_ATTR_EMB_CONFIG_NAME_TO_NUM_ROWS_POST_PRUNING_DICT, dict(tables_to_rows_post_pruning))
            cfgs = m.embedding_bag_configs() if hasattr(m, "embedding_bag_configs") else (m.embedding_configs() if hasattr(m, "embedding_configs") else [])
            for c in cfgs:
                if c.name in tables_to_rows_post_pruning:
                    c.num_embeddings_post_pruning = int(tables_to_rows_post_pruning[c.name])
    return model


def _quant_tbes(model: torch.nn.Module):
    from ..ops.quant_tbe import QuantTableBatchedEmbeddingBags

    return [m for m in model.modules() if isinstance(m, QuantTableBatchedEmbeddingBags)]


def get_table_to_weights_from_tbe(model: torch.nn.Module) -> Dict[str, torch.Tensor]:
    """``{table (shard) name: uint8 [rows, row_bytes]}`` views of every quantized table of ``model`` - sharded modules expose one entry
    per local shard (``<table>_<row_off>_<col_off>``). The views alias the kernels' storage (weight publishing writes through them)."""
    out: Dict[str, torch.Tensor] = {}
    for tbe in _quant_tbes(model):
        for (name, _, _, _), w in zip(tbe.embedding_specs, tbe.split_embedding_weights()):
            out[name] = w
    return out


@torch.no_grad()
def assign_weights_to_tbe(model: torch.nn.Module, table_to_weight: Dict[str, torch.Tensor]) -> None:
    """Copy quantized rows into the model's tables (e.g. a fresher snapshot published by training): every table of every quantized TBE
    must be present with its exact ``[rows, row_bytes]`` shape."""
    for tbe in _quant_tbes(model):
        for (name, rows, _, _), w in zip(tbe.embedding_specs, tbe.split_embedding_weights()):
            assert name in table_to_weight, f"{name} not in table_to_weight"
            src = table_to_weight[name]
            assert tuple(src.shape) == tuple(w.shape), f"{name}: got {tuple(src.shape)}, table is {tuple(w.shape)}"
            w.copy_(src.to(w.device))
        tbe.invalidate_cache()  # host-resident tables behind an HBM row cache: the cached copies are stale now
