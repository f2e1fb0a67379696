"""Generate tests/golden/preprocess_small.npz by running the UNMODIFIED reference image preparation in the build container:
ResizeLongestSide.apply_image_torch (stage1/data/transforms.py:48-54) and SA1BDataset.norm / pad (stage1/data/sa1b_dataset.py:216-227),
in the order SA1BDataset.__getitem__ applies them (:163-170).

    python tests/golden/gen_golden_preprocess.py

Needs /root/reference (absent on the GPU box -- the fixture is committed).  The uint8 inputs are not stored: `case_image` regenerates
them from their seeds, and the fixture holds the prepared [3,S,S] outputs and the sizes before padding.
"""
from __future__ import annotations

import collections.abc
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

# (tag, h, w, S, seed): landscape / portrait downscale, upscale, identity, a 1-pixel-high strip, odd prime sizes
CASES = [
    ("landscape_down", 150, 225, 96, 1),
    ("portrait_down", 225, 150, 96, 2),
    ("upscale", 37, 23, 96, 3),
    ("identity", 96, 64, 96, 4),
    ("strip", 1, 200, 128, 5),
    ("primes_down", 131, 101, 128, 6),
    ("primes_up", 53, 97, 128, 7),
]


def case_image(h, w, seed):
    """The seeded HWC uint8 RGB input of a case."""
    return torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))


def pseudo_collate(data_batch):
    """mmengine.dataset.pseudo_collate, which sa1b_dataset.py:14 imports (not installed here): the batch keeps one item's
    structure, nothing is stacked -- sequences are transposed, mappings collated key by key, anything else stays the list."""
    elem = data_batch[0]
    if isinstance(elem, str) or not isinstance(elem, (collections.abc.Sequence, collections.abc.Mapping)):
        return data_batch
    if isinstance(elem, collections.abc.Mapping):
        return type(elem)({k: pseudo_collate([d[k] for d in data_batch]) for k in elem})
    return [pseudo_collate(list(s)) for s in zip(*data_batch)]


def _import_sa1b():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    import install  # oracle/ref_shim/install.py
    install.install()
    if "mmengine" not in sys.modules:
        mm = types.ModuleType("mmengine")
        mm.__path__ = []
        mm.dataset = types.ModuleType("mmengine.dataset")
        mm.dataset.pseudo_collate = pseudo_collate
        sys.modules["mmengine"], sys.modules["mmengine.dataset"] = mm, mm.dataset
    # the stage1/data package __init__ pulls in every dataset; register the package without running it
    pkg = types.ModuleType("data")
    pkg.__path__ = [os.path.join(install.REFERENCE_ROOT, "stage1", "data")]
    sys.modules["data"] = pkg
    from data.sa1b_dataset import SA1BDataset
    return SA1BDataset


def main():
    SA1BDataset = _import_sa1b()
    torch.set_grad_enabled(False)
    outs, sizes = [], []
    for tag, h, w, S, seed in CASES:
        ds = SA1BDataset(os.path.join(HERE, "no-such-dataset"), img_size=S)     # default pixel_mean / pixel_std = DATA.MEAN / STD
        img = case_image(h, w, seed).permute(2, 0, 1)                            # pil_to_tensor layout, :68-69
        x = ds.transform.apply_image_torch(img[None].float()).squeeze(0)         # :163
        sizes.append(tuple(x.shape))                                             # img_size_before_pad, :167
        outs.append(ds.pad(ds.norm(x)).numpy().astype(np.float32))               # :168
        print(tag, (h, w), "->", tuple(x.shape), "S", S)
    path = os.path.join(HERE, "preprocess_small.npz")
    kw = {f"out_{t}": o for (t, *_), o in zip(CASES, outs)}
    np.savez_compressed(path, sizes=np.array(sizes, dtype=np.int64), **kw)
    print(path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
