"""Generate tests/golden/salience.pt from the REAL reference: sample_nonzero_locations and the use_salience lines of
ContrastiveCorrelationLoss.forward (src/modules.py:298-311, 357-364) on the CPU.

    STEGO_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_salience.py

The masks are rebuilt by the tests from `cases()` (seeded); each case stores the coordinates the reference's function
returned for both maps, the mixed coords1 / coords2 of the loss's lines, the CPU generator seed they were drawn from
and the generator's next four draws (the state it was left in).
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import reference_shim  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "salience.pt")


def cases():
    """name -> (salience, salience_pos, feature_samples): fp32 [B, H, W] masks as the training step passes them.
    Empty images, one-pixel masks, full masks, non-square maps, NaN / -0 entries and fs 1 / 11 / 16."""
    g = torch.Generator().manual_seed(31)

    def sparse(B, H, W, p):
        return (torch.rand(B, H, W, generator=g) < p).to(torch.float32) * torch.rand(B, H, W, generator=g).add(0.5)

    out = {}
    m = sparse(4, 12, 12, 0.2)
    m[1] = 0                      # an empty image
    m[2] = 0
    m[2, 7, 3] = 1.0              # one pixel
    m[3] = 1.0                    # full
    out["square_mixed_fs11"] = (m, sparse(4, 12, 12, 0.05), 11)
    m = sparse(3, 9, 17, 0.3)     # W > H: coordinates still divide by H
    m[0] = 0
    out["wide_fs16"] = (m, sparse(3, 9, 17, 0.01), 16)
    m = sparse(2, 19, 7, 0.3)     # H > W
    m[1] = 0
    m[1, 18, 6] = float("nan")    # NaN is nonzero
    m[1, 0, 0] = -0.0             # -0 is not
    out["tall_nan_fs1"] = (m, torch.zeros(2, 19, 7), 1)
    out["one_by_one_fs11"] = (torch.tensor([[[1.0]], [[0.0]]]), torch.tensor([[[0.0]], [[2.0]]]), 11)
    return out


def main():
    modules, _ = reference_shim.import_reference()
    golden = {}
    for i, (name, (sal, sal_pos, fs)) in enumerate(sorted(cases().items())):
        seed = 1000 + i
        torch.manual_seed(seed)
        coord_shape = [sal.shape[0], fs, fs, 2]
        # modules.py:358-364 (forward computes the coordinates inside; these are its lines, in its order)
        coords1_nonzero = modules.sample_nonzero_locations(sal, coord_shape)
        coords2_nonzero = modules.sample_nonzero_locations(sal_pos, coord_shape)
        coords1_reg = torch.rand(coord_shape) * 2 - 1
        coords2_reg = torch.rand(coord_shape) * 2 - 1
        mask = (torch.rand(coord_shape[:-1]) > .1).unsqueeze(-1).to(torch.float32)
        golden[name] = dict(seed=seed, fs=fs, nz1=coords1_nonzero, nz2=coords2_nonzero,
                            coords1=coords1_nonzero * mask + coords1_reg * (1 - mask),
                            coords2=coords2_nonzero * mask + coords2_reg * (1 - mask),
                            next=torch.randint(1 << 30, (4,)))
    torch.save(golden, OUT)
    print(f"wrote {OUT}: {len(golden)} cases")


if __name__ == "__main__":
    main()
