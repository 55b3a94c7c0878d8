"""Quantize -> serve (reference examples/inference_legacy, torchrec/inference): build a DLRM, quantize its tables to INT8,
start the native batching server with a gRPC front end, send requests.

    python examples/inference_server.py            # CPU works too; on a GPU box the executor runs on cuda:0
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchrec_b200.inference.modules import quantize_inference_model  # noqa: E402
from torchrec_b200.inference.server import InferenceServer, PredictorClient, ServerConfig, serve_grpc  # noqa: E402
from torchrec_b200.models.dlrm import DLRM  # noqa: E402
from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig  # noqa: E402
from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection  # noqa: E402


def main() -> None:
    dev = torch.device("cuda:0" if torch.cuda.is_available() else "cpu")
    keys = [f"cat_{i}" for i in range(8)]
    ebc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"t_{k}", embedding_dim=32, num_embeddings=10_000, feature_names=[k]) for k in keys], device=dev)
    model = DLRM(ebc, 13, [64, 32], [64, 1], dense_device=dev).eval()
    qmodel = quantize_inference_model(model)

    def predict(dense, kjt, _wkjt):
        return torch.sigmoid(qmodel(dense, kjt)).squeeze(-1)

    server = InferenceServer([predict], [dev], id_list_keys=keys, config=ServerConfig(max_batch_size=512, batching_interval_ms=2.0))
    grpc_server = serve_grpc(server, port=0)
    client = PredictorClient(f"127.0.0.1:{grpc_server.bound_port}")
    rng = np.random.default_rng(0)
    for B in (1, 4, 16):
        lengths = rng.integers(1, 4, size=len(keys) * B).astype(np.int32)
        out = client.predict(B, rng.standard_normal((B, 13)).astype(np.float32), (lengths, rng.integers(0, 10_000, size=int(lengths.sum()))), num_id_list_features=len(keys))
        print(B, out["default"][:4])
    print(server.stats())
    client.close()
    grpc_server.stop(0)
    server.shutdown()


if __name__ == "__main__":
    main()
