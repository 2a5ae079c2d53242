import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")
# offline test boxes: random-init encoders without the download attempt + warning (the product default follows the
# reference: ImageNet V1 weights, see bts_b200.model._load_backbone)
os.environ.setdefault("BTS_B200_PRETRAINED", "0")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    def load(name):          # NAME.npz plus its NAME.partK.npz spill files (oracle/make_golden.py keeps each below 1 MB)
        d = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
        k = 1
        while os.path.isfile(os.path.join(GOLDEN, "%s.part%d.npz" % (name, k))):
            d.update(np.load(os.path.join(GOLDEN, "%s.part%d.npz" % (name, k))))
            k += 1
        return d
    return load


def head_planes(B, h, w, max_depth, seed, device="cpu"):
    """Plane coefficients through the real head parametrisation (BASELINE.md, LPG-u inputs)."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 3, h, w, generator=g)
    th = torch.sigmoid(z[:, 0]) * np.pi / 3
    ph = torch.sigmoid(z[:, 1]) * np.pi * 2
    d = torch.sigmoid(z[:, 2]) * max_depth
    p = torch.stack([torch.sin(th) * torch.cos(ph), torch.sin(th) * torch.sin(ph), torch.cos(th), d], 1)
    return p.contiguous().to(device)
