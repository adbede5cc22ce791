"""Fused kNN kernel (stego_knn_topk, SURVEY.md §8(f) rank 1) against the oracle restatement of
src/precompute_knns.py:83-92.  Similarities are fp32 sums of 384 products: the bf16 hi/lo tensor-core path differs from
the fp32 einsum by ~1e-6, so rankings are compared exactly where the oracle's neighbouring similarities are separated by
more than that, and through the similarity values everywhere."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,E,k", [(1000, 384, 30), (257, 768, 30), (40, 64, 5), (3000, 384, 30), (31, 64, 30)])
def test_knn_topk_matches_oracle(cuda_dev, n, E, k):
    import stego_oracle as O
    from stego_b200.knn import knn_topk
    g = torch.Generator().manual_seed(n + E)
    base = torch.randn(max(8, n // 20), E, generator=g)                       # clustered descriptors: realistic ties
    feats = base[torch.randint(0, base.shape[0], (n,), generator=g)] + 0.35 * torch.randn(n, E, generator=g)
    feats = feats * (0.5 + torch.rand(n, 1, generator=g))                    # un-normalised input
    normed = torch.nn.functional.normalize(feats, dim=1)
    want_idx, want_val = O.knn_indices(normed.double(), k + 1)               # fp64 reference similarities (+ the runner-up)
    next_gap = (want_val[:, k - 1] - want_val[:, k]).abs()                   # separation of the k-th from the (k+1)-th
    want_idx, want_val = want_idx[:, :k], want_val[:, :k]
    idx, val = knn_topk(feats.to(cuda_dev), k, return_values=True)
    idx, val = idx.cpu(), val.cpu().double()
    assert idx.shape == (n, k) and idx.dtype == torch.long
    assert (idx[:, 0] == torch.arange(n)).all()                              # column 0 is the row itself, by contract
    assert (val[:, :-1] >= val[:, 1:]).all()                                 # sorted by descending similarity
    assert (val - want_val).abs().max().item() < 2e-5                        # the k best similarities, in order
    true_sims = (normed.double() @ normed.double().t()).gather(1, idx)       # returned indices really have those sims
    assert (true_sims - val).abs().max().item() < 2e-5
    gap = (want_val[:, :-1] - want_val[:, 1:]).abs()
    clear = torch.cat([gap > 1e-4, (next_gap > 1e-4).unsqueeze(1)], 1) & \
        torch.cat([torch.ones(n, 1, dtype=torch.bool), gap > 1e-4], 1)       # positions separated from both neighbours
    assert (idx[clear] == want_idx[clear]).all()


def test_knn_rejects_bad_shapes(cuda_dev):
    from stego_b200.knn import knn_topk
    with pytest.raises(RuntimeError, match="multiple of 64"):
        knn_topk(torch.zeros(100, 100, device=cuda_dev), 5)
    with pytest.raises(RuntimeError, match="k="):
        knn_topk(torch.zeros(100, 64, device=cuda_dev), 40)


def test_knn_descriptors_fused_layernorm_gap(cuda_dev):
    """precompute_knns.py:19 `model(img).mean([2, 3])`: the fused final-LayerNorm + pooling kernel against pooling the
    feature map DinoFeaturizer returns, eval and train mode (the reference never calls .eval(): Dropout2d is live)."""
    import torch
    from stego_b200.config import make_cfg
    from stego_b200.knn import knn_descriptors, nns_file_name, precompute_knns, save_nns
    from stego_b200.modules import DinoFeaturizer
    cfg = make_cfg(random_backbone_init=True)
    torch.manual_seed(0)
    net = DinoFeaturizer(70, cfg).to(cuda_dev)
    img = torch.randn(5, 3, 64, 96, device=cuda_dev)
    net.eval()
    with torch.no_grad():
        want = net(img)[0].mean([2, 3])
        got = knn_descriptors(net, img)
    assert got.shape == (5, 384)
    assert ((got - want).norm() / want.norm()).item() < 2e-3  # the feature map path rounds tokens to bf16 first
    net.train()
    torch.manual_seed(11)
    with torch.no_grad():
        want_t = net(img)[0].mean([2, 3])
    st = torch.cuda.get_rng_state(cuda_dev)
    torch.manual_seed(11)
    with torch.no_grad():
        got_t = knn_descriptors(net, img)
    assert ((got_t - want_t).norm() / want_t.norm()).item() < 2e-3
    assert (got_t == 0).float().mean().item() > 0.05  # ~10 % of the channels dropped
    # end to end: descriptors of a small image set -> top-k -> the .npz ContrastiveSegDataset loads
    net.eval()
    batches = [dict(img=torch.randn(4, 3, 64, 64)) for _ in range(3)]
    idx = precompute_knns(net, batches, k=5)
    assert idx.shape == (12, 5) and torch.equal(idx[:, 0].cpu(), torch.arange(12))
    import numpy as np
    import tempfile, os
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, nns_file_name("vit_small", "cocostuff27", "train", None, 224))
        save_nns(path, idx)
        loaded = np.load(path)["nns"]
        assert loaded.dtype == np.int64 and loaded.shape == (12, 5) and (loaded == idx.cpu().numpy()).all()
