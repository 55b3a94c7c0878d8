"""Command-line packager of the DLRM predict factory: writes the archive the inference server loads
(``python -m torchrec_b200.inference.dlrm_packager --output_path /tmp/model_package.zip``).

Parity: reference ``torchrec/inference/dlrm_packager.py`` (same flags; ``torch.package`` there, a zip of pickled configs + optional
state dict here: ``model_packager.PredictFactoryPackager``)."""
from __future__ import annotations

import argparse
import sys
from typing import List, Optional

from ..datasets.criteo import DEFAULT_CAT_NAMES, DEFAULT_INT_NAMES
from ..types import DataType
from .dlrm_predict import DLRMModelConfig, DLRMPredictFactory, create_training_batch
from .model_packager import PredictFactoryPackager

CRITEO_KAGGLE_ROWS = "45833188,36746,17245,7413,20243,3,7114,1441,62,29275261,1572176,345138,10,2209,11267,128,4,974,14,48937457,11316796,40094537,452104,12606,104,35"


def parse_args(argv: List[str]) -> argparse.Namespace:
    p = argparse.ArgumentParser(description="torchrec_b200 DLRM model packager")
    p.add_argument("--num_embeddings", type=int, default=100_000, help="rows of every table when --num_embeddings_per_feature is empty")
    p.add_argument("--num_embeddings_per_feature", type=str, default=CRITEO_KAGGLE_ROWS, help="comma separated rows per sparse feature (26 values for Criteo)")
    p.add_argument("--sparse_feature_names", type=str, default=",".join(DEFAULT_CAT_NAMES), help="comma separated sparse feature names")
    p.add_argument("--dense_arch_layer_sizes", type=str, default="512,256,64")
    p.add_argument("--over_arch_layer_sizes", type=str, default="512,512,256,1")
    p.add_argument("--embedding_dim", type=int, default=64)
    p.add_argument("--num_dense_features", type=int, default=len(DEFAULT_INT_NAMES))
    p.add_argument("--weight_dtype", type=str, default="INT8", choices=[d.value for d in (DataType.FP32, DataType.FP16, DataType.BF16, DataType.INT8, DataType.INT4, DataType.FP8)],
                   help="row format of the quantized tables (FP8 = block-scaled e4m3)")
    p.add_argument("--sample_batch_size", type=int, default=2, help="rows of the sample input stored with the package")
    p.add_argument("--output_path", type=str, required=True)
    return p.parse_args(argv)


def build_config(args: argparse.Namespace) -> DLRMModelConfig:
    keys = [k for k in args.sparse_feature_names.split(",") if k]
    per_feature = [int(x) for x in args.num_embeddings_per_feature.split(",") if x] if args.num_embeddings_per_feature else []
    if per_feature and len(per_feature) != len(keys):
        raise ValueError(f"{len(per_feature)} table sizes for {len(keys)} sparse features")
    rows_for_sample = min(per_feature) if per_feature else args.num_embeddings
    return DLRMModelConfig(
        dense_arch_layer_sizes=[int(x) for x in args.dense_arch_layer_sizes.split(",")] + ([] if args.dense_arch_layer_sizes.split(",")[-1] == str(args.embedding_dim) else [args.embedding_dim]),
        dense_in_features=args.num_dense_features, embedding_dim=args.embedding_dim, id_list_features_keys=keys, num_embeddings_per_feature=per_feature,
        num_embeddings=args.num_embeddings, over_arch_layer_sizes=[int(x) for x in args.over_arch_layer_sizes.split(",")],
        sample_input=create_training_batch(args.num_dense_features, keys, rows_for_sample, args.sample_batch_size), weight_dtype=DataType(args.weight_dtype))


def main(argv: Optional[List[str]] = None) -> str:
    args = parse_args(sys.argv[1:] if argv is None else argv)
    PredictFactoryPackager.save_predict_factory(DLRMPredictFactory, {"model_config": build_config(args)}, args.output_path)
    print(f"packaged DLRM predict factory -> {args.output_path}")
    return args.output_path


if __name__ == "__main__":
    main()
