"""Cost of LitUnsupervisedSegmenter.eval_scene on plot_potsdam.py's scene (15 x 15 tiles of 320², ViT-B/8, 3 classes,
loader batches of 64), against what a caller does without it:

  * stitched: eval_step per chunk of 64 tiles, the outputs stitched with torch (cat + the reference's permutes), and
    with the CRF crf.dense_crf on the stitched image and stitched cluster log-probabilities (one 4800² frame) plus
    UnsupervisedMetrics.update of its predictions against the stitched label;
  * eval_scene: one call, the probe kernels writing into the mosaic, with the CRF the cluster-only unary rows and one
    mean field over the mosaic.

With the CRF, every path is timed in the lattice-cache state a user's call meets.  eval_scene builds the mosaic's
position lattice on every call (it never caches it), so no cached copy is left for it to reuse: the 4800² entry of
crf's cache is removed before each of its calls.  dense_crf caches that lattice per frame size, so the stitched path
is timed twice: stitched_cold removes the entry first (a process's first scene) and stitched_warm reuses it (every
later scene of that size, with the lattice kept for the life of the process).

Without the CRF both probes are evaluated (eval_segmentation's loop body); with it only the cluster probe
(plot_potsdam's case).

    python profiles/eval_scene_time.py [--out profiles/eval_scene_time_h100.json]

Per case and path: ms per scene (host clock from an idle device to the synchronise after the call: the lattice build
syncs the host; one warm-up call, then the paths alternate for three rounds, the median kept) and the peak of
torch.cuda.max_memory_allocated over the call.  Prints one JSON object with the card.
"""
from __future__ import annotations

import argparse
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from _measure import card, emit, host_ms  # noqa: E402

ARCH, R, C, T, CHUNK, N_CLASSES, ROUNDS = "vit_base", 15, 15, 320, 64, 3, 3


def paths(run_crf, dev):
    import scene_oracle as SO
    import stego_oracle as O
    from stego_b200 import crf
    from stego_b200.config import make_cfg
    from stego_b200.segmenter import LitUnsupervisedSegmenter
    torch.manual_seed(0)
    model = LitUnsupervisedSegmenter(N_CLASSES, make_cfg(model_type=ARCH, random_backbone_init=True)).to(dev)
    model.net.model.load_state_dict(O.perturb_vit_state(O.vit_random_state(ARCH, 8, seed=3)))
    g = torch.Generator(device=dev).manual_seed(0)
    m = torch.linspace(-1.5, 1.5, C * T, device=dev).view(1, 1, -1).expand(3, R * T, C * T).clone()
    m[1] = torch.linspace(-1.5, 1.5, R * T, device=dev).view(-1, 1)
    tiles = m.view(3, R, T, C, T).permute(1, 3, 0, 2, 4).reshape(R * C, 3, T, T) + \
        0.3 * torch.randn(R * C, 3, T, T, device=dev, generator=g)
    label = torch.randint(0, N_CLASSES, (R * C, T, T), device=dev, generator=g).to(torch.uint8)
    probes = ("cluster",) if run_crf else ("linear", "cluster")

    def drop_lattice():
        crf._POSITION_LATTICES.pop((R * T, C * T, dev.index), None)

    def ours():
        drop_lattice()
        return model.eval_scene(tiles, (R, C), label=label, run_crf=run_crf, probes=probes, chunk=CHUNK)

    def stitched():
        outs = [model.eval_step(dict(img=tiles[t0:t0 + CHUNK], label=None if run_crf else label[t0:t0 + CHUNK]),
                                want_probs=run_crf) for t0 in range(0, R * C, CHUNK)]
        if not run_crf:
            return {k: SO.stitch(torch.cat([o[k] for o in outs], 0), R, C) for k in ("linear_preds", "cluster_preds")}
        logp = SO.stitch(torch.cat([o["cluster_probs"] for o in outs], 0), R, C)
        _, pred = crf.dense_crf(SO.stitch(tiles, R, C), logp, want_argmax=True)
        model.test_cluster_metrics.update(pred, SO.stitch(label, R, C))
        return pred

    if not run_crf:
        return dict(eval_scene=ours, stitched=stitched)

    def stitched_cold():
        drop_lattice()
        return stitched()

    return dict(eval_scene=ours, stitched_cold=stitched_cold, stitched_warm=stitched)


def case(run_crf, dev):
    fns = paths(run_crf, dev)
    times = {k: [] for k in fns}
    peaks = {}
    for k, fn in fns.items():  # warm-up (graphs; stitched_warm runs after stitched_cold's cached lattice) and the peak
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        fn()
        torch.cuda.synchronize()
        peaks[k] = (torch.cuda.max_memory_allocated(dev), base)
    for _ in range(ROUNDS):
        for k, fn in fns.items():
            times[k].append(host_ms(fn, 1))
    ms = {k: statistics.median(v) for k, v in times.items()}
    out = dict(arch=ARCH, grid=[R, C], tile=T, chunk=CHUNK, n_classes=N_CLASSES, run_crf=run_crf,
               probes=["cluster"] if run_crf else ["linear", "cluster"])
    for k, t in ms.items():
        out[f"{k}_ms"] = round(t, 1)
        out[f"{k}_rounds_ms"] = [round(x, 1) for x in times[k]]
        out[f"{k}_peak_gib"] = round(peaks[k][0] / 2**30, 2)
        out[f"{k}_peak_above_inputs_gib"] = round((peaks[k][0] - peaks[k][1]) / 2**30, 2)
    for k in ms:
        if k != "eval_scene":
            out[f"speedup_vs_{k}"] = round(ms[k] / ms["eval_scene"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    result = dict(card=card(), cases=[])
    for run_crf in (False, True):
        result["cases"].append(case(run_crf, dev))
        torch.cuda.empty_cache()
    from stego_b200 import crf
    result["position_lattices_cached"] = [list(k[:2]) for k in crf._POSITION_LATTICES]
    result["card_after"] = card()
    emit(result, a.out)


if __name__ == "__main__":
    main()
