"""TensorBoard histograms binned on the GPU: what `SummaryWriter.add_histogram(tag, values)` writes with its default
bins="tensorflow", as the fields of `SummaryWriter.add_histogram_raw`.

The reference's training step logs the code correlations of its three loss groups every `hist_freq` steps
(train_segmentation.py:144-146, 165-168: tags intra_cd, inter_cd, neg_cd).  Here those cd tensors are never
materialised: the forward correlation kernels bin them in their epilogue (corr.LossSpec.forward with a CdHistogram), and
only 3 x 1548 counts and 3 x 4 statistics leave the device.  `tb_histogram` bins any fp32 CUDA tensor with the same
bucket rule (csrc/tb_hist.cuh).
"""
from __future__ import annotations

import ctypes
import functools
from typing import Dict, Tuple

import numpy as np
import torch

from . import _lib

TAGS = ("intra_cd", "inter_cd", "neg_cd")  # groups 0 (call 0), 1 (call 1), 2 (calls 2.., concatenated)
N_EDGES = 1549
N_BINS = N_EDGES - 1
GENERIC_CTAS = 264  # per-CTA partials of stego_tb_histogram


@functools.lru_cache(maxsize=None)
def _tables() -> Tuple[np.ndarray, np.ndarray]:
    edges = np.empty(N_EDGES, dtype=np.float64)
    thr = np.empty(N_EDGES + 1, dtype=np.float32)
    _lib.check(_lib.load().stego_tb_tables(edges.ctypes.data, thr.ctypes.data), "stego_tb_tables")
    edges.flags.writeable = False
    thr.flags.writeable = False
    return edges, thr


def default_bins() -> np.ndarray:
    """torch's SummaryWriter.default_bins as float64 (the library's copy, which the kernels' thresholds are made from)."""
    return _tables()[0]


def thresholds() -> np.ndarray:
    """The fp32 table the kernels compare against: RU(e) for every edge e, then RD(last edge)."""
    return _tables()[1]


_device_thresholds: Dict[torch.device, torch.Tensor] = {}


def device_thresholds(device) -> torch.Tensor:
    device = torch.device(device)
    t = _device_thresholds.get(device)
    if t is None:
        t = torch.from_numpy(thresholds().copy()).to(device)
        _device_thresholds[device] = t
    return t


def trim(counts: np.ndarray, edges: np.ndarray = None):
    """(bucket_limit, bucket) as summary.make_histogram keeps them: the buckets from the first to the last non-empty one,
    with the bucket left of the first one (an empty one at index 0 when the support starts there); the limits are the
    right edges."""
    if edges is None:
        edges = default_bins()
    counts = np.asarray(counts, dtype=np.int64)
    cum = np.cumsum(counts > 0)
    start, end = np.searchsorted(cum, [0, cum[-1] - 1], side="right")
    start, end = int(start), int(end) + 1
    kept = counts[start - 1:end] if start > 0 else np.concatenate([[0], counts[:end]])
    limits = edges[start:end + 1]
    if kept.size == 0 or limits.size == 0:
        raise ValueError("histogram: no value falls inside the TensorBoard buckets")
    return limits, kept


def fields(counts: np.ndarray, stats: np.ndarray, num: int) -> dict:
    """add_histogram_raw's keyword arguments from the counts [1548] and stats (min, max, sum, sum of squares)."""
    limits, kept = trim(counts)
    return dict(min=float(stats[0]), max=float(stats[1]), num=int(num), sum=float(stats[2]),
                sum_squares=float(stats[3]), bucket_limits=limits.tolist(), bucket_counts=kept.tolist())


def tb_histogram(values: torch.Tensor) -> dict:
    """The add_histogram_raw fields of `values` (an fp32 CUDA tensor) for the default TensorBoard buckets, equal to
    what SummaryWriter.add_histogram(tag, values) writes.  Synchronises (the result is on the host)."""
    _lib.require_cuda(values)
    if values.dtype != torch.float32:
        raise RuntimeError(f"stego_b200: tb_histogram takes fp32 values, got {values.dtype}")
    if values.numel() == 0:
        raise ValueError("The input has no element.")
    x = values.contiguous().view(-1)
    dev = x.device
    counts = torch.empty(N_BINS, dtype=torch.int64, device=dev)
    part = torch.empty(GENERIC_CTAS, 4, dtype=torch.float64, device=dev)
    stats = torch.empty(4, dtype=torch.float64, device=dev)
    _lib.check(_lib.load().stego_tb_histogram(_lib.ptr(x), x.numel(), _lib.ptr(device_thresholds(dev)),
                                              _lib.ptr(counts), _lib.ptr(part), _lib.ptr(stats), _lib.stream()),
               "stego_tb_histogram")
    return fields(counts.cpu().numpy(), stats.cpu().numpy(), x.numel())


class CdHistogram:
    """Device buffers for the histogram variant of one correlation-loss forward (spec.forward(..., hist=self)), and
    their pinned host copies.  `stage` copies the results behind an event without waiting; `results` waits for that
    event and returns {tag: add_histogram_raw fields}."""

    def __init__(self, spec, B: int, device):
        S = spec.fs * spec.fs
        self.ngroups = min(spec.ncalls, 3)
        calls = [1, 1, spec.ncalls - 2][:self.ngroups]
        self.num = [c * B * S * S for c in calls]
        self.thresholds = device_thresholds(device)
        self.counts = torch.empty(3, N_BINS, dtype=torch.int64, device=device)
        self.stats = torch.empty(3, 4, dtype=torch.float64, device=device)
        self.cta_partials = torch.empty(spec.ncalls * B * spec.hist_ctas * 4, dtype=torch.float64, device=device)
        self.counts_host = torch.empty(3, N_BINS, dtype=torch.int64, pin_memory=True)
        self.stats_host = torch.empty(3, 4, dtype=torch.float64, pin_memory=True)
        self.ready = None

    def args(self):
        """the trailing pointer arguments of the *_fwd_hist entry points"""
        return (_lib.ptr(self.thresholds), _lib.ptr(self.counts), _lib.ptr(self.cta_partials), _lib.ptr(self.stats))

    def stage(self) -> None:
        """Queue the device -> pinned host copies on the current stream (no host synchronisation)."""
        self.counts_host.copy_(self.counts, non_blocking=True)
        self.stats_host.copy_(self.stats, non_blocking=True)
        self.ready = torch.cuda.Event()
        self.ready.record()

    def results(self) -> Dict[str, dict]:
        self.ready.synchronize()
        counts, stats = self.counts_host.numpy(), self.stats_host.numpy()
        return {TAGS[g]: fields(counts[g], stats[g], self.num[g]) for g in range(self.ngroups)}
