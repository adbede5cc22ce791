"""The `devices=` argument of the multi-device inference paths (eval_step, eval_scene, knn_topk, precompute_knns): one
process spreads independent frames / rows over several GPUs of a node, launching from the calling thread, device after
device (every launch is asynchronous), and gathers the results on the first device, the primary."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple, Union

import torch

DeviceLike = Union[int, torch.device]


def check_devices(devices: Optional[Sequence[DeviceLike]], primary: torch.device, who: str
                  ) -> Optional[List[torch.device]]:
    """The validated devices, or None for the single-device path (devices None or a list of one device: the primary,
    which must be the inputs' device).  Refused with a ValueError, before anything is enqueued: an empty list, a
    non-CUDA device, an ordinal out of range, a duplicate, a primary other than `primary` (the inputs' and the model's
    device), and a device without peer access to and from the primary."""
    if devices is None:
        return None
    if isinstance(devices, (int, torch.device, str)):
        raise ValueError(f"{who}: devices must be a sequence of CUDA ordinals or devices, got {devices!r}")
    devices = list(devices)
    if not devices:
        raise ValueError(f"{who}: devices must name at least one CUDA device")
    n_visible = torch.cuda.device_count()
    out: List[torch.device] = []
    for d in devices:
        if isinstance(d, bool) or not isinstance(d, (int, torch.device)):
            raise ValueError(f"{who}: devices entries must be CUDA ordinals or torch.device, got {d!r}")
        if isinstance(d, int) and not 0 <= d < n_visible:
            raise ValueError(f"{who}: device ordinal {d} out of range ({n_visible} CUDA devices visible)")
        dev = torch.device("cuda", d) if isinstance(d, int) else d
        if dev.type != "cuda":
            raise ValueError(f"{who}: devices must be CUDA devices, got {dev}")
        if dev.index is None:
            raise ValueError(f"{who}: device {dev} has no ordinal; name it as cuda:<i>")
        if not 0 <= dev.index < n_visible:
            raise ValueError(f"{who}: device {dev} out of range ({n_visible} CUDA devices visible)")
        if dev in out:
            raise ValueError(f"{who}: device {dev} listed twice")
        out.append(dev)
    for dev in out[1:]:
        if not (torch.cuda.can_device_access_peer(out[0].index, dev.index)
                and torch.cuda.can_device_access_peer(dev.index, out[0].index)):
            raise ValueError(f"{who}: {out[0]} and {dev} have no peer access to each other")
    if out[0] != primary:
        raise ValueError(f"{who}: the first device ({out[0]}) must be the device of the inputs and the model "
                         f"({primary})")
    return out if len(out) > 1 else None


def split(n: int, parts: int, align: int = 1) -> List[Tuple[int, int]]:
    """[start, end) ranges of `parts` contiguous, nearly equal slices of n items; with align > 1 every start is a
    multiple of `align` (slices of whole align-blocks, the last one ragged).  With more parts than blocks some slices
    are empty (start == end): their devices stay idle."""
    blocks = (n + align - 1) // align
    return [(min(blocks * i // parts * align, n), min(blocks * (i + 1) // parts * align, n)) for i in range(parts)]
