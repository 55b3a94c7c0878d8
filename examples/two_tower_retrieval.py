"""Two-tower retrieval (reference examples/retrieval/two_tower_train.py, modules/two_tower.py): a query tower and a
candidate tower (EmbeddingBagCollection + MLP each) trained with in-batch softmax; the candidate embeddings are then
exported and served through brute-force top-k (the reference uses FAISS IVFPQ; here a tensor-core-friendly dense scoring)."""
import os
import sys
from typing import List

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig  # noqa: E402
from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection  # noqa: E402
from torchrec_b200.modules.mlp import MLP  # noqa: E402
from torchrec_b200.sparse import KeyedJaggedTensor  # noqa: E402


class TwoTower(nn.Module):
    """``forward(kjt) -> (query_embedding [B, D], candidate_embedding [B, D])``; feature 0 of the KJT is the query."""

    def __init__(self, embedding_bag_collection: EmbeddingBagCollection, layer_sizes: List[int], device=None) -> None:
        super().__init__()
        cfgs = embedding_bag_collection.embedding_bag_configs()
        assert len(cfgs) == 2 and cfgs[0].embedding_dim == cfgs[1].embedding_dim
        self._feature_names_query, self._feature_names_candidate = cfgs[0].feature_names, cfgs[1].feature_names
        self.ebc = embedding_bag_collection
        self.query_proj = MLP(cfgs[0].embedding_dim, layer_sizes, device=device)
        self.candidate_proj = MLP(cfgs[1].embedding_dim, layer_sizes, device=device)

    def forward(self, kjt: KeyedJaggedTensor):
        pooled = self.ebc(kjt).to_dict()
        q = self.query_proj(torch.cat([pooled[f] for f in self._feature_names_query], dim=1))
        c = self.candidate_proj(torch.cat([pooled[f] for f in self._feature_names_candidate], dim=1))
        return q, c


class TwoTowerTrainTask(nn.Module):
    def __init__(self, two_tower: TwoTower) -> None:
        super().__init__()
        self.two_tower = two_tower
        self.loss_fn = nn.BCEWithLogitsLoss()

    def forward(self, batch):
        q, c = self.two_tower(batch.sparse_features)
        logits = (q * c).sum(dim=1)
        loss = self.loss_fn(logits, batch.labels.float())
        return loss, (loss.detach(), logits.detach(), batch.labels.detach())


class TwoTowerRetrieval(nn.Module):
    """Serving: embed the query, score against all candidate embeddings, return the top-k candidate ids."""

    def __init__(self, two_tower: TwoTower, candidate_ids: torch.Tensor, k: int = 10) -> None:
        super().__init__()
        self.two_tower, self.k = two_tower, k
        with torch.no_grad():
            w = two_tower.ebc.embedding_bags[two_tower.ebc.embedding_bag_configs()[1].name].weight
            self.register_buffer("index", two_tower.candidate_proj(w[candidate_ids]))
        self.register_buffer("ids", candidate_ids)

    @torch.no_grad()
    def forward(self, query_kjt: KeyedJaggedTensor) -> torch.Tensor:
        pooled = self.two_tower.ebc(query_kjt).to_dict()
        q = self.two_tower.query_proj(torch.cat([pooled[f] for f in self.two_tower._feature_names_query], dim=1))
        return self.ids[(q @ self.index.t()).topk(self.k, dim=1).indices]


def main() -> None:
    from torchrec_b200.datasets.random import RandomRecDataset

    torch.manual_seed(0)
    users, items, D = 1000, 500, 32
    ebc = EmbeddingBagCollection([EmbeddingBagConfig(name="t_user", embedding_dim=D, num_embeddings=users, feature_names=["user"]),
                                  EmbeddingBagConfig(name="t_item", embedding_dim=D, num_embeddings=items, feature_names=["item"])])
    task = TwoTowerTrainTask(TwoTower(ebc, [64, 32]))
    opt = torch.optim.Adam(task.parameters(), lr=1e-2)
    data = iter(RandomRecDataset(["user", "item"], 256, hash_sizes=[users, items], ids_per_features=[1, 1], num_dense=1, manual_seed=0, num_batches=30))
    for step, batch in enumerate(data):
        opt.zero_grad()
        loss, _ = task(batch)
        loss.backward()
        opt.step()
        if step % 10 == 0:
            print(f"step {step} loss {float(loss):.4f}")
    retrieval = TwoTowerRetrieval(task.two_tower, torch.arange(items), k=5)
    q = KeyedJaggedTensor(keys=["user", "item"], values=torch.tensor([3, 7, 0, 0]), lengths=torch.tensor([1, 1, 1, 1]))
    print("top-5 items for users 3 and 7:", retrieval(q).tolist())


if __name__ == "__main__":
    main()
