"""DLRM model family: DLRM, DLRM_Projection, DLRM_DCN, DLRMTrain.

Architecture parity with the reference (torchrec/models/dlrm.py:38-960): SparseArch (EBC ->
[B, F, D]), DenseArch (bottom MLP), InteractionArch (pairwise dots) / InteractionDCNArch
(low-rank cross net) / InteractionProjectionArch, OverArch (top MLP, last layer linear).
Dense compute is routed through ``torchrec_b200.ops.dense`` so that on an H100 the MLP layers and
the dot interaction run as hand-written wgmma kernels.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import os

import torch
from torch import nn

from ..datasets.utils import Batch
from ..modules.crossnet import LowRankCrossNet
from ..modules.embedding_modules import EmbeddingBagCollection
from ..modules.mlp import MLP
from ..ops import dense as _dense
from ..sparse.jagged_tensor import KeyedJaggedTensor, KeyedTensor


def choose(n: int, k: int) -> int:
    """n choose k (0 when k > n)."""
    if 0 <= k <= n:
        ntok = ktok = 1
        for t in range(1, min(k, n - k) + 1):
            ntok *= n
            ktok *= t
            n -= 1
        return ntok // ktok
    return 0


class SparseArch(nn.Module):
    """EBC lookup reshaped to ``[B, F, D]`` (all tables share D)."""

    def __init__(self, embedding_bag_collection: EmbeddingBagCollection) -> None:
        super().__init__()
        self.embedding_bag_collection = embedding_bag_collection
        cfgs = self.embedding_bag_collection.embedding_bag_configs()
        assert cfgs, "Embedding bag collection cannot be empty!"
        self.D: int = cfgs[0].embedding_dim
        self._sparse_feature_names: List[str] = [name for c in cfgs for name in c.feature_names]
        self.F: int = len(self._sparse_feature_names)

    def forward(self, features: KeyedJaggedTensor) -> torch.Tensor:
        sparse_features: KeyedTensor = self.embedding_bag_collection(features)
        sparse_values = sparse_features.values()
        return sparse_values.reshape(-1, self.F, self.D)

    @property
    def sparse_feature_names(self) -> List[str]:
        return self._sparse_feature_names


class DenseArch(nn.Module):
    """Bottom MLP over the dense features."""

    def __init__(self, in_features: int, layer_sizes: List[int], device: Optional[torch.device] = None) -> None:
        super().__init__()
        self.model: nn.Module = MLP(in_features, layer_sizes, bias=True, activation="relu", device=device)

    def forward(self, features: torch.Tensor) -> torch.Tensor:
        return self.model(features)


class InteractionArch(nn.Module):
    """cat(dense, pairwise dot products among [dense; sparse features])."""

    def __init__(self, num_sparse_features: int) -> None:
        super().__init__()
        self.F: int = num_sparse_features

    def forward(self, dense_features: torch.Tensor, sparse_features: torch.Tensor) -> torch.Tensor:
        if self.F <= 0:
            return dense_features
        return _dense.dot_interaction(dense_features, sparse_features)


class InteractionDCNArch(nn.Module):
    """Cross-net (DCN-v2) interaction over cat(dense, flattened sparse)."""

    def __init__(self, num_sparse_features: int, crossnet: nn.Module) -> None:
        super().__init__()
        self.F: int = num_sparse_features
        self.crossnet = crossnet

    def forward(self, dense_features: torch.Tensor, sparse_features: torch.Tensor) -> torch.Tensor:
        if self.F <= 0:
            return dense_features
        B = dense_features.shape[0]
        combined = torch.cat((dense_features.unsqueeze(1), sparse_features.to(dense_features.dtype)), dim=1)
        return self.crossnet(combined.reshape(B, -1))


class InteractionProjectionArch(nn.Module):
    """Project the F+1 feature vectors with two MLPs and take dots between the projections."""

    def __init__(self, num_sparse_features: int, interaction_branch1: nn.Module, interaction_branch2: nn.Module) -> None:
        super().__init__()
        self.F: int = num_sparse_features
        self.interaction_branch1 = interaction_branch1
        self.interaction_branch2 = interaction_branch2

    def forward(self, dense_features: torch.Tensor, sparse_features: torch.Tensor) -> torch.Tensor:
        if self.F <= 0:
            return dense_features
        B, D = dense_features.shape
        combined = torch.cat((dense_features.unsqueeze(1), sparse_features.to(dense_features.dtype)), dim=1)
        flat = torch.reshape(combined, (B, -1))
        b1 = torch.reshape(self.interaction_branch1(flat), (B, -1, D))
        b2 = torch.reshape(self.interaction_branch2(flat), (B, D, -1))
        interactions = torch.bmm(b1, b2)
        return torch.cat((dense_features, torch.reshape(interactions, (B, -1))), dim=1)


class OverArch(nn.Module):
    """Top MLP; the final layer has no activation."""

    def __init__(self, in_features: int, layer_sizes: List[int], device: Optional[torch.device] = None) -> None:
        super().__init__()
        if len(layer_sizes) <= 1:
            raise ValueError("OverArch must have multiple layers.")
        self.model: nn.Module = nn.Sequential(
            MLP(in_features, layer_sizes[:-1], bias=True, activation="relu", device=device),
            nn.Linear(layer_sizes[-2], layer_sizes[-1], bias=True, device=device),
        )

    def forward(self, features: torch.Tensor) -> torch.Tensor:
        hidden = self.model[0](features)
        last = self.model[1]
        if hidden.dtype == torch.bfloat16 and last.out_features == 1:
            from ..ops import dense as _dense
            from ..ops import head as _head

            if _dense.get_dense_backend() == "wgmma" and _head.rowdot_supported(hidden, last.weight):
                return _head.RowDotFn.apply(hidden, last.weight, last.bias)  # fused logit layer (+ ReLU mask of `hidden` in its dgrad)
        if hidden.dtype != last.weight.dtype:  # bf16 activations from the fused kernels -> fp32 logits
            hidden = hidden.to(last.weight.dtype)
        return last(hidden)


class DLRM(nn.Module):
    """Deep Learning Recommendation Model (https://arxiv.org/abs/1906.00091)."""

    def __init__(
        self,
        embedding_bag_collection: EmbeddingBagCollection,
        dense_in_features: int,
        dense_arch_layer_sizes: List[int],
        over_arch_layer_sizes: List[int],
        dense_device: Optional[torch.device] = None,
    ) -> None:
        super().__init__()
        cfgs = embedding_bag_collection.embedding_bag_configs()
        assert len(cfgs) > 0, "At least one embedding bag is required"
        for i in range(len(cfgs)):
            assert cfgs[i].embedding_dim == cfgs[0].embedding_dim, "Embedding dimensions of all embedding bags must be the same"
        embedding_dim = cfgs[0].embedding_dim
        if dense_arch_layer_sizes[-1] != embedding_dim:
            raise ValueError(f"embedding_bag_collection dimension ({embedding_dim}) and final dense arch layer size ({dense_arch_layer_sizes[-1]}) must match.")
        self.sparse_arch: SparseArch = SparseArch(embedding_bag_collection)
        num_sparse_features = len(self.sparse_arch.sparse_feature_names)
        self.dense_arch = DenseArch(in_features=dense_in_features, layer_sizes=dense_arch_layer_sizes, device=dense_device)
        self.inter_arch = InteractionArch(num_sparse_features=num_sparse_features)
        over_in_features = embedding_dim + choose(num_sparse_features, 2) + num_sparse_features
        self.over_arch = OverArch(in_features=over_in_features, layer_sizes=over_arch_layer_sizes, device=dense_device)

    # Run the (memory / latency-bound) embedding arch on a side CUDA stream concurrently with the (tensor-core bound) bottom
    # MLP: their kernels co-reside on the SMs, in the forward AND in the backward (autograd replays every op on the stream of
    # its forward). Opt in with ``model.overlap_sparse_dense = True`` or TRB_OVERLAP_SPARSE=1.
    overlap_sparse_dense: bool = False

    def _sparse_stream(self, device: torch.device):
        st = self.__dict__.get("_trb_sparse_stream")
        if st is None or st.device != device:
            st = torch.cuda.Stream(device=device)
            self.__dict__["_trb_sparse_stream"] = st
        return st

    # ---- CUDA graphs for the dense sub-modules -------------------------------------------------------------------------------
    def capture_dense_graphs(self, sample_dense_features: torch.Tensor, sample_embedded_sparse: torch.Tensor, num_warmup_iters: int = 3) -> None:
        """Capture forward AND backward of the bottom MLP and of interaction + top MLP into CUDA graphs
        (``torch.cuda.make_graphed_callables``). The dense part of a DLRM step is ~50 small launches + ~100 ATen calls whose
        *enqueue* time can match the GPU time of the whole step: with more ranks (DDP, NVLink dists) the step becomes launch-bound. Replaying two graphs removes that host time; the sparse part stays eager, so jagged
        inputs keep their dynamic shapes. Batches whose shapes differ from the samples fall back to the eager modules.

        Call it BEFORE the dense part is wrapped in DDP (``DistributedModelParallel(..., init_data_parallel=False)``, capture, then
        ``dmp.init_data_parallel()``): DDP keeps the parameters' AccumulateGrad nodes alive on the default stream and a capture that
        has to synchronise with the legacy stream is rejected by CUDA (cudaErrorStreamCaptureImplicit)."""
        assert sample_dense_features.is_cuda, "CUDA graphs need CUDA tensors"
        plane = self._sparse_plane()

        from ..ops import gemm as _gemm

        ext_push = plane is not None and plane.W > 1 and os.environ.get("TRB_PUSH_IN_DENSE_GRAPH", "1") != "0"

        def push_embedding_grads(grads) -> None:
            # backward of the module INPUTS = last node of the captured backward: the NVLink gradient dist of the embedding gradients
            # becomes part of the dense backward graph, right behind the interaction backward and beside the deferred weight gradients
            if ext_push:
                g = grads[1].reshape(grads[1].shape[0], -1)
                plane._push_kernels(g if g.stride(1) == 1 else g.contiguous())

        class _InterOver(nn.Module):
            def __init__(self, inter: nn.Module, over: nn.Module) -> None:
                super().__init__()
                self.inter, self.over = inter, over

            def forward(self, embedded_dense: torch.Tensor, embedded_sparse: torch.Tensor) -> torch.Tensor:
                if embedded_dense.is_cuda and torch.is_grad_enabled():
                    embedded_dense, embedded_sparse = _gemm.DeferredGradJoin.apply(push_embedding_grads, embedded_dense, embedded_sparse)
                return self.over(self.inter(dense_features=embedded_dense, sparse_features=embedded_sparse))

        from ..ops import _lib

        class _Dense(nn.Module):  # thin wrappers: make_graphed_callables patches THEIR forward, the real modules stay eager
            def __init__(self, m: nn.Module) -> None:
                super().__init__()
                self.m = m

            def forward(self, x: torch.Tensor) -> torch.Tensor:
                return self.m(x)

        with torch.no_grad():
            emb_dense = self.dense_arch(sample_dense_features)
        n0 = _lib.launch_count() if _lib.available() else 0
        s_dense = sample_dense_features.detach().clone()
        s_ed = emb_dense.detach().clone().requires_grad_()
        s_es = sample_embedded_sparse.detach().clone().requires_grad_()
        if plane is not None and sample_embedded_sparse.numel() == plane.B_local * plane.total_cols and sample_embedded_sparse.dtype == plane.wire_dtype:
            # the embedding arch's TRAINING output always lands in slot 0 of the plane's symmetric buffer: make that memory the graph's
            # static input, so that the per-step copy of the [B, F * D] embeddings into the graph disappears
            s_es = plane.out_local(0).view(sample_embedded_sparse.shape).requires_grad_()
        inter_over = _InterOver(self.inter_arch, self.over_arch)
        # capture on a HIGH-priority stream: the captured nodes inherit it, the deferred weight-gradient kernels (side stream, default
        # priority) then yield to the dgrad chain / gradient push whenever both have work
        prev_cap = torch.cuda.graph.default_capture_stream
        torch.cuda.graph.default_capture_stream = torch.cuda.Stream(device=sample_dense_features.device, priority=-1)
        try:
            with _gemm.defer_wgrad_scope():
                g_dense, g_top = torch.cuda.make_graphed_callables((_Dense(self.dense_arch), inter_over), ((s_dense,), (s_ed, s_es)), num_warmup_iters=num_warmup_iters)
        finally:
            torch.cuda.graph.default_capture_stream = prev_cap
        # native launches replayed per training step by the two graphs (the host counter only sees the capture): forward + backward
        # were each recorded once after `num_warmup_iters` eager warm-up rounds
        per_step = ((_lib.launch_count() - n0) // (num_warmup_iters + 1)) if _lib.available() else 0
        self.__dict__["_trb_graphs"] = {"dense": g_dense, "top": g_top, "dense_sig": (tuple(s_dense.shape), s_dense.dtype),
                                        "sparse_sig": (tuple(s_es.shape), s_es.dtype), "launches_per_step": int(per_step),
                                        "ext_push_plane": plane if ext_push else None}

    def _sparse_plane(self):
        """The NVLink sparse plane behind the embedding arch (None before its first batch / for unsharded collections)."""
        eng = getattr(self.sparse_arch.embedding_bag_collection, "_engine", None)
        if eng is None:
            return None
        planes = [p for p in eng.__dict__.get("_planes", {}).values() if p.capacity > 0]
        return planes[0] if len(planes) == 1 else None

    def _graphed(self, dense_features: torch.Tensor):
        g = self.__dict__.get("_trb_graphs")
        if g is None or not self.training or not torch.is_grad_enabled() or (tuple(dense_features.shape), dense_features.dtype) != g["dense_sig"]:
            return None
        return g

    def forward(self, dense_features: torch.Tensor, sparse_features: KeyedJaggedTensor) -> torch.Tensor:
        import os

        g = self._graphed(dense_features)
        if g is not None:
            overlap = self.overlap_sparse_dense or os.environ.get("TRB_OVERLAP_SPARSE") == "1"
            if overlap:
                # embedding arch on a side stream: its forward (lookup + NVLink output dist) runs beside the bottom MLP, and - autograd
                # replays every op on the stream of its forward - its backward (gradient push over NVLink, fused optimizer) runs beside
                # the bottom MLP's backward and the dense gradient all-reduce instead of after them
                main = torch.cuda.current_stream(dense_features.device)
                side = self._sparse_stream(dense_features.device)
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    embedded_sparse = self.sparse_arch(sparse_features)
                    if isinstance(embedded_sparse, torch.Tensor):
                        embedded_sparse.record_stream(main)
                embedded_dense = g["dense"](dense_features)
                main.wait_stream(side)
            else:
                embedded_sparse = self.sparse_arch(sparse_features)
                embedded_dense = None
            if (tuple(embedded_sparse.shape), embedded_sparse.dtype) == g["sparse_sig"]:
                from ..ops import _lib

                if embedded_dense is None:
                    embedded_dense = g["dense"](dense_features)
                if g.get("ext_push_plane") is not None:
                    g["ext_push_plane"].external_push = True  # this step's gradient push is replayed by the top graph's backward
                out = g["top"](embedded_dense, embedded_sparse)
                _lib.add_launches(g["launches_per_step"])
                return out
            if embedded_dense is None:
                embedded_dense = self.dense_arch(dense_features)
            return self.over_arch(self.inter_arch(dense_features=embedded_dense, sparse_features=embedded_sparse))
        if dense_features.is_cuda and (self.overlap_sparse_dense or os.environ.get("TRB_OVERLAP_SPARSE") == "1"):
            main = torch.cuda.current_stream(dense_features.device)
            side = self._sparse_stream(dense_features.device)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                embedded_sparse = self.sparse_arch(sparse_features)
                if isinstance(embedded_sparse, torch.Tensor):
                    embedded_sparse.record_stream(main)  # allocated on the side stream's pool, consumed on the main stream
            embedded_dense = self.dense_arch(dense_features)
            main.wait_stream(side)
        else:
            embedded_dense = self.dense_arch(dense_features)
            embedded_sparse = self.sparse_arch(sparse_features)
        concatenated_dense = self.inter_arch(dense_features=embedded_dense, sparse_features=embedded_sparse)
        return self.over_arch(concatenated_dense)


class DLRM_Projection(DLRM):
    """DLRM with projected interactions (DLRM_Projection in the reference)."""

    def __init__(
        self,
        embedding_bag_collection: EmbeddingBagCollection,
        dense_in_features: int,
        dense_arch_layer_sizes: List[int],
        over_arch_layer_sizes: List[int],
        interaction_branch1_layer_sizes: List[int],
        interaction_branch2_layer_sizes: List[int],
        dense_device: Optional[torch.device] = None,
    ) -> None:
        super().__init__(embedding_bag_collection, dense_in_features, dense_arch_layer_sizes, over_arch_layer_sizes, dense_device)
        embedding_dim = embedding_bag_collection.embedding_bag_configs()[0].embedding_dim
        num_sparse_features = len(self.sparse_arch.sparse_feature_names)
        if interaction_branch1_layer_sizes[-1] % embedding_dim != 0:
            raise ValueError(f"Final interaction branch1 layer size ({interaction_branch1_layer_sizes[-1]}) is not a multiple of embedding size ({embedding_dim})")
        projected_dim_1 = interaction_branch1_layer_sizes[-1] // embedding_dim
        if interaction_branch2_layer_sizes[-1] % embedding_dim != 0:
            raise ValueError(f"Final interaction branch2 layer size ({interaction_branch2_layer_sizes[-1]}) is not a multiple of embedding size ({embedding_dim})")
        projected_dim_2 = interaction_branch2_layer_sizes[-1] // embedding_dim
        self.inter_arch = InteractionProjectionArch(
            num_sparse_features=num_sparse_features,
            interaction_branch1=MLP(in_size=(num_sparse_features + 1) * embedding_dim, layer_sizes=interaction_branch1_layer_sizes, bias=True, device=dense_device),
            interaction_branch2=MLP(in_size=(num_sparse_features + 1) * embedding_dim, layer_sizes=interaction_branch2_layer_sizes, bias=True, device=dense_device),
        )
        over_in_features = embedding_dim + projected_dim_1 * projected_dim_2
        self.over_arch = OverArch(in_features=over_in_features, layer_sizes=over_arch_layer_sizes, device=dense_device)


class DLRM_DCN(DLRM):
    """DLRM with a DCN-v2 low-rank cross network interaction (MLPerf DLRM-DCNv2)."""

    def __init__(
        self,
        embedding_bag_collection: EmbeddingBagCollection,
        dense_in_features: int,
        dense_arch_layer_sizes: List[int],
        over_arch_layer_sizes: List[int],
        dcn_num_layers: int,
        dcn_low_rank_dim: int,
        dense_device: Optional[torch.device] = None,
    ) -> None:
        super().__init__(embedding_bag_collection, dense_in_features, dense_arch_layer_sizes, over_arch_layer_sizes, dense_device)
        embedding_dim = embedding_bag_collection.embedding_bag_configs()[0].embedding_dim
        num_sparse_features = len(self.sparse_arch.sparse_feature_names)
        over_in_features = embedding_dim * (num_sparse_features + 1)
        crossnet = LowRankCrossNet(in_features=over_in_features, num_layers=dcn_num_layers, low_rank=dcn_low_rank_dim)
        if dense_device is not None:
            crossnet = crossnet.to(dense_device)
        self.inter_arch = InteractionDCNArch(num_sparse_features=num_sparse_features, crossnet=crossnet)
        self.over_arch = OverArch(in_features=over_in_features, layer_sizes=over_arch_layer_sizes, device=dense_device)


class DLRMTrain(nn.Module):
    """Training wrapper: BCE-with-logits loss; returns ``(loss, (loss.detach(), logits.detach(), labels.detach()))``."""

    def __init__(self, dlrm_module: DLRM) -> None:
        super().__init__()
        self.model = dlrm_module
        self.loss_fn: nn.Module = nn.BCEWithLogitsLoss()

    def forward(self, batch: Batch) -> Tuple[torch.Tensor, Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
        logits = self.model(batch.dense_features, batch.sparse_features)
        logits = logits.squeeze(-1)
        if type(self.loss_fn) is nn.BCEWithLogitsLoss and logits.is_cuda and logits.dtype == torch.float32:
            from ..ops.head import bce_with_logits_mean

            loss = bce_with_logits_mean(logits, batch.labels)  # loss + d(loss)/d(logits) in one kernel
        else:
            loss = self.loss_fn(logits.float(), batch.labels.float())
        return loss, (loss.detach(), logits.detach(), batch.labels.detach())


class DLRMWrapper(DLRM):
    """DLRM taking a ``Batch``-like object as the single input (used by inference packaging)."""

    def forward(self, model_input) -> torch.Tensor:  # type: ignore[override]
        return super().forward(model_input.float_features, model_input.idlist_features)
