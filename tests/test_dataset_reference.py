"""CPU: the resident training set's host draws (stego_b200.dataset.Sampler) against the live reference training loader
(ContrastiveSegDataset under DataLoader(shuffle=True, num_workers=W), run by oracle/make_golden_dataset.py's harness),
for W = 0, 1 and 3 across the epoch boundaries.  Skipped unless STEGO_REFERENCE_SRC names the reference's src
directory."""
import os
import sys
import tempfile
from types import SimpleNamespace

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import reference_shim  # noqa: E402

pytestmark = pytest.mark.skipif(not reference_shim.available(), reason="STEGO_REFERENCE_SRC not set")


@pytest.mark.parametrize("layout", ["cropped", "directory"])
def test_sampler_matches_live_reference_loader(layout):
    import make_golden_dataset as G
    from make_golden_frames import _import_reference_loaders
    from stego_b200.dataset import Sampler
    utils, data = _import_reference_loaders()
    images, labels, nns = G.inputs()
    res = 30
    cfg = SimpleNamespace(dir_dataset_n_classes=27, dir_dataset_name="myset", crop_ratio=0.5, crop_type="five",
                          model_type="vit_small", res=res)
    with tempfile.TemporaryDirectory() as root:
        name, crop = G.write_layout(root, layout, images, labels, nns, res, cfg)
        for workers in G.WORKERS:
            batches = G.run(data, utils, root, name, crop, res, cfg, workers)
            got = []
            for epoch in Sampler(nns, G.BATCH, G.NUM_NEIGHBORS, G.SEED, workers, res=res):
                for b in epoch:
                    got.append(b)
                    if len(got) == len(batches):
                        break
                if len(got) == len(batches):
                    break
            for want, (ind, pos, seeds) in zip(batches, got):
                assert ind.tolist() == want["ind"].tolist()
                assert pos.tolist() == want["ind_pos"].tolist()
                assert seeds.tolist() == want["seed"].tolist()
