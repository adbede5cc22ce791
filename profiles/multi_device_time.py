"""Time of the multi-device inference paths at 1, 2 and 8 GPUs (as many of those counts as the node has):

  * eval_step, ViT-B/8, 64 frames of 320², without and with the CRF (`devices=`);
  * eval_scene, a 15 x 15 scene of 320² tiles (4800²), ViT-B/8, without the CRF and with the cluster-only CRF;
  * knn_topk, n = 118 287 descriptors (COCO-Stuff train), E = 384, k = 30;
  * nn.DataParallel(model.net) forward, ViT-B/8, 64 frames of 320².

    python profiles/multi_device_time.py [--out profiles/multi_device_time_h100.json]

At one device the calls are the single-device ones (devices=None, the plain module).  Every call ends on the host
(the CRF paths synchronise per frame), so each figure is the host clock from an idle device to the synchronise after
the call, per call over REPS calls after one warm-up call of the same shape.  The CRF scene's calls each start by
emptying torch's allocator cache (its 31 GiB value buffer does not fit in the fragments other calls leave cached).  The card's name, power limit and
maximum SM clock are read in the same run, for every device used.  Prints one JSON object.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
from _measure import card, emit, host_ms  # noqa: E402

COUNTS = (1, 2, 8)
REPS = 3


def _model(dev):
    import stego_oracle as O
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(27, make_cfg(random_backbone_init=True, model_type="vit_base")).to(dev)
    model.net.model.load_state_dict(O.perturb_vit_state(O.vit_random_state("vit_base", 8, seed=3)))
    model.eval()
    return model


def _time(fn):
    torch.cuda.empty_cache()
    fn()
    return round(host_ms(fn, REPS), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from stego_b200.knn import knn_topk
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n_visible = torch.cuda.device_count()
    counts = [c for c in COUNTS if c <= n_visible]
    model = _model(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    img = torch.randn(64, 3, 320, 320, device=dev, generator=g)
    label = torch.randint(0, 27, (64, 320, 320), device=dev, generator=g)
    tiles = torch.randn(225, 3, 320, 320, device=dev, generator=g)
    tile_label = torch.randint(0, 27, (225, 320, 320), device=dev, generator=g)
    feats = torch.randn(118287, 384, device=dev, generator=g)
    rows = []
    for c in counts:
        devices = list(range(c)) if c > 1 else None
        par = torch.nn.DataParallel(model.net, device_ids=list(range(c))) if c > 1 else model.net
        row = dict(devices=c)
        with torch.no_grad():
            # first, and with the cache emptied before every call: the 4800² mean field's value buffers take one
            # 31 GiB block, which the blocks other calls leave cached would fragment
            row["eval_scene_15x15_cluster_crf_ms"] = _time(lambda: (torch.cuda.empty_cache(), model.eval_scene(
                tiles, (15, 15), tile_label, run_crf=True, probes=("cluster",), devices=devices)))
            row["eval_step_b64_ms"] = _time(lambda: model.eval_step(dict(img=img, label=label), devices=devices))
            row["eval_step_b64_crf_ms"] = _time(lambda: model.eval_step(dict(img=img, label=label), run_crf=True,
                                                                         devices=devices))
            row["eval_scene_15x15_ms"] = _time(lambda: model.eval_scene(tiles, (15, 15), tile_label,
                                                                        devices=devices))
            row["knn_118287x384_ms"] = _time(lambda: knn_topk(feats, 30, devices=devices))
            row["data_parallel_forward_b64_ms"] = _time(lambda: par(img))
        rows.append(row)
        torch.cuda.empty_cache()
    cards = []
    for i in range(max(counts)):
        with torch.cuda.device(i):
            cards.append(card())
    emit(dict(what="multi-device inference, ViT-B/8 320² (kNN: 118 287 x 384, k 30)", visible_gpus=n_visible,
              cards=cards, reps=REPS, rows=rows), args.out)


if __name__ == "__main__":
    main()
