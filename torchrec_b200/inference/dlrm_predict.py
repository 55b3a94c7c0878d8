"""DLRM serving recipe: model config -> quantized, sharded ``PredictModule`` + the metadata the batching server needs.

Parity: reference ``inference/dlrm_predict.py`` (``DLRMModelConfig`` :52, ``DLRMPredictModule`` :67, ``DLRMPredictFactory`` :145). The
request layout is the same ("float_features", "id_list_features.lengths", "id_list_features.values"), so a client written against
the reference's ``predictor.proto`` works unchanged; quantization + sharding go through this package's own
``quantize_inference_model`` / ``shard_quant_model`` (inference planner, NVLink gathers)."""
from __future__ import annotations

import logging
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from ..datasets.utils import Batch
from ..models.dlrm import DLRM
from ..modules.embedding_configs import DataType, EmbeddingBagConfig
from ..modules.embedding_modules import EmbeddingBagCollection
from ..sparse import KeyedJaggedTensor
from .modules import BatchingMetadata, PredictFactory, PredictModule, quantize_dense, quantize_inference_model, shard_quant_model

logger: logging.Logger = logging.getLogger(__name__)


@dataclass
class DLRMModelConfig:
    dense_arch_layer_sizes: List[int]
    dense_in_features: int
    embedding_dim: int
    id_list_features_keys: List[str]
    num_embeddings_per_feature: List[int]
    num_embeddings: int
    over_arch_layer_sizes: List[int]
    sample_input: Optional[Batch] = None
    weight_dtype: DataType = DataType.INT8
    per_table_weight_dtype: Dict[str, DataType] = field(default_factory=dict)
    # dtype of the dense arch (bottom / top MLP, cross net) in the served module: None keeps it as trained; torch.float8_e4m3fn runs it
    # on the FP8 GEMM (quantize_dense)
    dense_dtype: Optional[torch.dtype] = None


def create_training_batch(num_dense: int, keys: List[str], num_embeddings: int, batch_size: int, ids_per_feature: int = 1, seed: int = 0) -> Batch:
    """A random ``Batch`` of the served shape (sample input for packaging / smoke requests)."""
    g = torch.Generator().manual_seed(seed)
    F = len(keys)
    lengths = torch.full((F * batch_size,), ids_per_feature, dtype=torch.int32)
    values = torch.randint(0, num_embeddings, (F * batch_size * ids_per_feature,), generator=g)
    return Batch(dense_features=torch.rand(batch_size, num_dense, generator=g), sparse_features=KeyedJaggedTensor(keys=keys, values=values, lengths=lengths),
                 labels=torch.randint(0, 2, (batch_size,), generator=g).float())


class DLRMPredictModule(PredictModule):
    """``predict_forward({"float_features", "id_list_features.lengths", "id_list_features.values"}) -> {"default": probabilities}``."""

    def __init__(self, module: Optional[torch.nn.Module] = None, id_list_features_keys: Optional[List[str]] = None, device: Optional[str] = None,
                 embedding_bag_collection: Optional[torch.nn.Module] = None, dense_in_features: Optional[int] = None, dense_arch_layer_sizes: Optional[List[int]] = None,
                 over_arch_layer_sizes: Optional[List[int]] = None, dense_device: Optional[torch.device] = None) -> None:
        """Either wrap a ready model (``module`` - a sharded / quantized DLRM), or give the pieces and a float DLRM is built from them
        (the reference's constructor: ``embedding_bag_collection, dense_in_features, dense_arch_layer_sizes, over_arch_layer_sizes,
        id_list_features_keys, dense_device``)."""
        if module is None or isinstance(module, torch.nn.Module) and embedding_bag_collection is None and dense_in_features is not None:
            embedding_bag_collection = embedding_bag_collection if embedding_bag_collection is not None else module
            module = None
        if module is None:
            from ..models.dlrm import DLRM

            assert embedding_bag_collection is not None and dense_in_features is not None and dense_arch_layer_sizes is not None and over_arch_layer_sizes is not None, \
                "DLRMPredictModule needs a module, or the embedding bags and the dense / over arch sizes to build a DLRM"
            module = DLRM(embedding_bag_collection=embedding_bag_collection, dense_in_features=dense_in_features, dense_arch_layer_sizes=dense_arch_layer_sizes,
                          over_arch_layer_sizes=over_arch_layer_sizes, dense_device=dense_device)
            device = device if device is not None else (str(dense_device) if dense_device is not None else None)
        assert id_list_features_keys is not None, "id_list_features_keys is required"
        super().__init__(module, device)
        self.id_list_features_keys: List[str] = list(id_list_features_keys)

    def predict_forward(self, batch: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        kjt = KeyedJaggedTensor(keys=self.id_list_features_keys, lengths=batch["id_list_features.lengths"], values=batch["id_list_features.values"])
        logits = self.predict_module(batch["float_features"], kjt)
        predictions = logits.sigmoid().reshape(logits.shape[0])
        return {"default": predictions.to(torch.device("cpu"), non_blocking=True).float()}


class DLRMPredictFactory(PredictFactory):
    def __init__(self, model_config: DLRMModelConfig) -> None:
        self.model_config = model_config

    def create_predict_module(self, world_size: int = 1, device: str = "cuda") -> torch.nn.Module:
        cfg = self.model_config
        if device == "cuda" and not torch.cuda.is_available():
            device = "cpu"
        per_feature = cfg.num_embeddings_per_feature or [cfg.num_embeddings] * len(cfg.id_list_features_keys)
        tables = [EmbeddingBagConfig(name=f"t_{k}", embedding_dim=cfg.embedding_dim, num_embeddings=n, feature_names=[k]) for k, n in zip(cfg.id_list_features_keys, per_feature)]
        model = DLRM(EmbeddingBagCollection(tables, device=torch.device("cpu")), dense_in_features=cfg.dense_in_features, dense_arch_layer_sizes=cfg.dense_arch_layer_sizes,
                     over_arch_layer_sizes=cfg.over_arch_layer_sizes, dense_device=torch.device("cpu"))
        model.eval()
        model = self.run_weights_independent_tranformations(model)
        sharded, _plan = shard_quant_model(model, world_size=world_size, compute_device=device, sharding_device="cpu")
        if device == "cuda":
            sharded = sharded.to(torch.device("cuda", 0))
        return DLRMPredictModule(self.run_weights_dependent_transformations(sharded), cfg.id_list_features_keys, device=device if device != "cuda" else "cuda:0")

    def batching_metadata(self) -> Dict[str, BatchingMetadata]:
        return {"float_features": BatchingMetadata(type="dense", device="cuda", pinned=[]),
                "id_list_features": BatchingMetadata(type="sparse", device="cuda", pinned=["lengths", "values"])}

    def result_metadata(self) -> str:
        return "dict_of_tensor"

    def run_weights_independent_tranformations(self, predict_module: torch.nn.Module) -> torch.nn.Module:
        cfg = self.model_config
        per_table = {f"t_{k}": v for k, v in cfg.per_table_weight_dtype.items()} if cfg.per_table_weight_dtype else None
        return quantize_inference_model(predict_module, quantization_dtype=cfg.weight_dtype, per_table_weight_dtype=per_table)

    def run_weights_dependent_transformations(self, predict_module: torch.nn.Module) -> torch.nn.Module:
        if self.model_config.dense_dtype is not None:
            predict_module = quantize_dense(predict_module, self.model_config.dense_dtype)
        return predict_module

    def model_inputs_data(self) -> Dict[str, object]:
        cfg = self.model_config
        return {"float_features": {"shape": [-1, cfg.dense_in_features], "dtype": "float32"}, "id_list_features": {"keys": list(cfg.id_list_features_keys)}}
