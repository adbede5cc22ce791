"""Oracle of the use_salience coordinate draws.  TEST INFRASTRUCTURE ONLY.

src/modules.py:298-311 (sample_nonzero_locations) and :357-364 (ContrastiveCorrelationLoss.forward with
cfg.use_salience), restated line for line as plain torch on CPU or CUDA tensors; the masks arrive as the training step
passes them (train_segmentation.py:147-152: batch["mask"].to(torch.float32).squeeze(1)).  The `*_from_draws` variants
apply the same expressions to given values instead of the generator's, so a kernel fed those values can be checked
against them.
"""
from __future__ import annotations

import torch

Tensor = torch.Tensor


def sample_nonzero_locations(t: Tensor, target_size) -> Tensor:
    """modules.py:298-311."""
    nonzeros = torch.nonzero(t)
    coords = torch.zeros(target_size, dtype=nonzeros.dtype, device=nonzeros.device)
    n = target_size[1] * target_size[2]
    for i in range(t.shape[0]):
        selected = nonzeros[nonzeros[:, 0] == i]
        if selected.shape[0] == 0:
            picked = torch.randint(t.shape[1], size=(n, 2), device=nonzeros.device)
        else:
            picked = selected[torch.randint(len(selected), size=(n,)), 1:]
        coords[i, :, :, :] = picked.reshape(target_size[1], target_size[2], 2)
    coords = coords.to(torch.float32) / t.shape[1]
    coords = coords * 2 - 1
    return torch.flip(coords, dims=[-1])


def mix(nz1: Tensor, nz2: Tensor, reg1: Tensor, reg2: Tensor, keep_u: Tensor):
    """modules.py:360-364 after the draws: reg = u * 2 - 1 (reg1 / reg2 are the uniforms), keep = u > .1."""
    reg1 = reg1 * 2 - 1
    reg2 = reg2 * 2 - 1
    mask = (keep_u > .1).unsqueeze(-1).to(torch.float32)
    return nz1 * mask + reg1 * (1 - mask), nz2 * mask + reg2 * (1 - mask)


def draw_coords(salience: Tensor, salience_pos: Tensor, feature_samples: int):
    """modules.py:355-364 with use_salience: (coords1, coords2), drawing from the device's default generator."""
    shape = [salience.shape[0], feature_samples, feature_samples, 2]
    dev = salience.device
    nz1 = sample_nonzero_locations(salience, shape)
    nz2 = sample_nonzero_locations(salience_pos, shape)
    reg1 = torch.rand(shape, device=dev)
    reg2 = torch.rand(shape, device=dev)
    keep = torch.rand(shape[:-1], device=dev)
    return mix(nz1, nz2, reg1, reg2, keep)


def nonzero_locations_from_draws(t: Tensor, feature_samples: int, draws: Tensor) -> Tensor:
    """sample_nonzero_locations with image i's randint replaced by draws[i] (raw uint32 values held in int64, at least
    2 fs^2 of them): `draw % count` picks the nonzero, or, without nonzeros, y, x = draws[2 s], draws[2 s + 1] % H."""
    fs = feature_samples
    n = fs * fs
    nonzeros = torch.nonzero(t)
    coords = torch.zeros([t.shape[0], fs, fs, 2], dtype=nonzeros.dtype, device=nonzeros.device)
    for i in range(t.shape[0]):
        selected = nonzeros[nonzeros[:, 0] == i]
        d = draws[i].to(torch.int64)
        if selected.shape[0] == 0:
            picked = (d[:2 * n] % t.shape[1]).reshape(n, 2)
        else:
            picked = selected[d[:n] % len(selected), 1:]
        coords[i] = picked.reshape(fs, fs, 2)
    coords = coords.to(torch.float32) / t.shape[1]
    coords = coords * 2 - 1
    return torch.flip(coords, dims=[-1])
