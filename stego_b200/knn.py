"""Fused kNN over image descriptors (SURVEY.md §8(f) rank 1): the device-side replacement of the similarity + top-k
loop of the reference's `src/precompute_knns.py:83-96`, which produces the `nns_*.npz` files `img_pos` is drawn from."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from .devices import DeviceLike, check_devices, split

KNN_ROW_BLOCK = 128  # knn.cu KNN_BM: a row range of stego_knn_topk_rows starts on a multiple of it


def knn_topk(feats: torch.Tensor, k: int = 30, return_values: bool = False,
             devices: Optional[Sequence[DeviceLike]] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """feats: [n, E] fp32 CUDA (un-normalised descriptors, e.g. `model(img).mean([2, 3])`, precompute_knns.py:19).
    Returns int64 [n, k] neighbour indices of the reference's `torch.topk(einsum("nf,mf->nm", ...), 30)[1]` with the
    order pinned: column 0 is the row's own index, always (also next to exact or near duplicates and for an all-zero
    row — src/data.py:524 reads columns 1..k as "not the image itself"), columns 1..k-1 the other rows by (cosine
    similarity descending, index ascending); and the fp32 similarities of those indices if requested.

    devices: several GPUs of the node, the first being feats' device (see stego_b200.devices.check_devices).  The
    normalised descriptors are prepared once on it and copied to the others; each device searches a contiguous range of
    128-row blocks against all n rows and the results are gathered on the first device.  A row's result depends only on
    the row and the fixed key-tile order, so the output is bit-identical to the single-device call."""
    devs = check_devices(devices, feats.device, "knn_topk")
    _lib.require_cuda(feats)
    if feats.dim() != 2 or feats.dtype != torch.float32:
        raise RuntimeError("stego_b200.knn_topk: feats must be a 2-D fp32 tensor")
    feats = feats.contiguous()
    n, E = feats.shape
    # several devices are refused here, before any launch; on one device the C entries refuse bad sizes themselves
    if devs is not None and (n < 1 or E < 1 or E % 64 or not 1 <= k <= min(32, n)):
        raise ValueError(f"knn_topk: n={n}, E={E}, k={k} unsupported (E a positive multiple of 64, 1 <= k <= "
                         f"min(32, n))")
    devs = devs or [feats.device]
    ranges = split(n, len(devs), KNN_ROW_BLOCK)
    return _knn_topk_sharded(feats, k, return_values, [(d, r0, r1) for d, (r0, r1) in zip(devs, ranges)])


def _knn_topk_sharded(feats: torch.Tensor, k: int, return_values: bool, shards: List[Tuple[torch.device, int, int]]
                      ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """knn_topk over query-row ranges [r0, r1) (r0 a multiple of 128), one per (device, r0, r1) entry, launched from the
    calling thread one device after another.  The first entry runs on feats' device and writes into the outputs in
    place; every other entry gets its own copy of the planes and its own outputs, copied back into the first device's
    (the copies are ordered on the devices' current streams; no host synchronisation)."""
    lib = _lib.load()
    n, E = feats.shape
    primary = feats.device
    planes = torch.empty(2, n, E, dtype=torch.bfloat16, device=primary)
    _lib.check(lib.stego_knn_prep(_lib.ptr(feats), n, E, _lib.ptr(planes), _lib.stream()), "stego_knn_prep")
    idx = torch.empty(n, k, dtype=torch.long, device=primary)
    vals = torch.empty(n, k, dtype=torch.float32, device=primary) if return_values else None
    for i, (dev, r0, r1) in enumerate(shards):
        if r1 <= r0:
            continue
        with torch.cuda.device(dev):
            if i == 0:
                pl, out_i, out_v = planes, idx[r0:r1], vals[r0:r1] if return_values else None
            else:
                pl = planes.to(dev)
                out_i = torch.empty(r1 - r0, k, dtype=torch.long, device=dev)
                out_v = torch.empty(r1 - r0, k, dtype=torch.float32, device=dev) if return_values else None
            _lib.check(lib.stego_knn_topk_rows(_lib.ptr(pl), n, E, k, r0, r1 - r0, _lib.ptr(out_i), _lib.ptr(out_v),
                                               _lib.stream()), "stego_knn_topk_rows")
            if i > 0:
                idx[r0:r1].copy_(out_i)
                if return_values:
                    vals[r0:r1].copy_(out_v)
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


def precompute_knns(net, batches, k: int = 30, devices: Optional[Sequence[DeviceLike]] = None) -> torch.Tensor:
    """The device-side body of precompute_knns.py:83-96: descriptors of every image (`batches` yields image tensors or
    dicts with an "img" entry, like the reference's loader), cosine-similarity top-k over the whole set.

    devices: several GPUs of the node, the first being the net's device.  Batch i's descriptors are computed on
    devices[i % len(devices)] (the frozen ViT's prepared weights are cached per device), gathered in loader order on
    the first device, and the search runs as knn_topk(..., devices=devices).  The result equals the single-device one;
    the exception is a net in training mode with cfg.dropout, whose Dropout2d noise each device draws from its own
    generator (as nn.DataParallel does)."""
    primary = next(net.parameters()).device
    devs = check_devices(devices, primary, "precompute_knns") or [primary]
    feats = []
    for i, pack in enumerate(batches):
        img = pack["img"] if isinstance(pack, dict) else pack
        img = img.to(devs[i % len(devs)])
        with torch.cuda.device_of(img):
            feats.append(knn_descriptors(net, img).to(primary))
    idx, _ = knn_topk(torch.cat(feats, 0), k, devices=devs)
    return idx


def nns_file_name(model_type: str, dataset_name: str, image_set: str, crop_type, res: int) -> str:
    """File name `ContrastiveSegDataset` looks for (src/data.py:503-504, src/precompute_knns.py:66-67)."""
    return "nns_{}_{}_{}_{}_{}.npz".format(model_type, dataset_name, image_set, crop_type, res)


def save_nns(path: str, nearest_neighbors: torch.Tensor) -> None:
    """precompute_knns.py:94: `np.savez_compressed(file, nns=int64 [n, k])` — what src/data.py:509-510 loads."""
    import numpy as np
    np.savez_compressed(path, nns=nearest_neighbors.detach().cpu().numpy().astype("int64"))
