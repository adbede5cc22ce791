"""Fused kNN over image descriptors (SURVEY.md §8(f) rank 1): the device-side replacement of the similarity + top-k
loop of the reference's `src/precompute_knns.py:83-96`, which produces the `nns_*.npz` files `img_pos` is drawn from."""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _lib


def knn_topk(feats: torch.Tensor, k: int = 30, return_values: bool = False
             ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """feats: [n, E] fp32 CUDA (un-normalised descriptors, e.g. `model(img).mean([2, 3])`, precompute_knns.py:19).
    Returns int64 [n, k] neighbour indices of the reference's `torch.topk(einsum("nf,mf->nm", ...), 30)[1]` with the
    order pinned: column 0 is the row's own index, always (also next to exact or near duplicates and for an all-zero
    row — src/data.py:524 reads columns 1..k as "not the image itself"), columns 1..k-1 the other rows by (cosine
    similarity descending, index ascending); and the fp32 similarities of those indices if requested."""
    _lib.require_cuda(feats)
    if feats.dim() != 2 or feats.dtype != torch.float32:
        raise RuntimeError("stego_b200.knn_topk: feats must be a 2-D fp32 tensor")
    feats = feats.contiguous()
    n, E = feats.shape
    planes = torch.empty(2, n, E, dtype=torch.bfloat16, device=feats.device)
    idx = torch.empty(n, k, dtype=torch.long, device=feats.device)
    vals = torch.empty(n, k, dtype=torch.float32, device=feats.device) if return_values else None
    rc = _lib.load().stego_knn_topk(_lib.ptr(feats), n, E, k, _lib.ptr(planes), _lib.ptr(idx), _lib.ptr(vals), _lib.stream())
    _lib.check(rc, "stego_knn_topk")
    return idx, vals


def knn_descriptors(net, img: torch.Tensor) -> torch.Tensor:
    """`model.forward(img).mean([2, 3])` of precompute_knns.py:19 for a `DinoFeaturizer`, un-normalised fp32 [B, E]:
    frozen ViT -> global average pool of the teacher features the config selects, without writing the feature map —
    "feat": final LayerNorm + pooling in one kernel; "KK": the last block's LN1 + pooling, then the key projection of the
    pooled row (the mean of the keys, the projection being linear).  In training mode with cfg.dropout the
    reference's returned features carry the third Dropout2d mask (src/modules.py:115-116 — precompute_knns.py never calls
    .eval()); a per-(image, channel) scale commutes with the spatial mean, so the same noise tensors are drawn (all three,
    to keep the RNG stream of `net(img)`) and the last one is applied to the pooled vector."""
    if net.feat_type == "feat":
        pool = net.model.pooled_patch_features
    elif net.feat_type == "KK":
        pool = net.model.pooled_key_features
    else:
        raise ValueError("Unknown feat type:{}".format(net.feat_type))
    net.model.eval()
    pooled = pool(img)
    _, _, m3 = net.draw_masks(img.shape[0], img.device)
    if net.cfg.dropout and m3 is not None:
        pooled = pooled * m3
    return pooled


def precompute_knns(net, batches, k: int = 30) -> torch.Tensor:
    """The device-side body of precompute_knns.py:83-96: descriptors of every image (`batches` yields image tensors or
    dicts with an "img" entry, like the reference's loader), cosine-similarity top-k over the whole set."""
    feats = []
    for pack in batches:
        img = pack["img"] if isinstance(pack, dict) else pack
        feats.append(knn_descriptors(net, img.to(next(net.parameters()).device)))
    idx, _ = knn_topk(torch.cat(feats, 0), k)
    return idx


def nns_file_name(model_type: str, dataset_name: str, image_set: str, crop_type, res: int) -> str:
    """File name `ContrastiveSegDataset` looks for (src/data.py:503-504, src/precompute_knns.py:66-67)."""
    return "nns_{}_{}_{}_{}_{}.npz".format(model_type, dataset_name, image_set, crop_type, res)


def save_nns(path: str, nearest_neighbors: torch.Tensor) -> None:
    """precompute_knns.py:94: `np.savez_compressed(file, nns=int64 [n, k])` — what src/data.py:509-510 loads."""
    import numpy as np
    np.savez_compressed(path, nns=nearest_neighbors.detach().cpu().numpy().astype("int64"))
