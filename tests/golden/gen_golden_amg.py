"""Generate tests/golden/amg_small.json by running the UNMODIFIED reference SamAutomaticMaskGenerator
(sam3/sam3/model/student_sam/automatic_mask_generator.py) on the seeded synthetic decoder of oracle/amg.py.

    python tests/golden/gen_golden_amg.py

Needs the reference checkout (absent on the GPU box -- the fixture is committed).  The reference module's missing imports are
registered in sys.modules first: `.utils.amg` (never vendored) is oracle/amg.py; `.modeling` is a stub; `.predictor` (EdgeSAM's
SamPredictor, which needs the external edge_sam package) is a stub serving the synthetic decoder's logits upsampled by
F.interpolate(bilinear, align_corners=False), with the decoder's IoU as the prediction.  Every torchvision batched_nms call of
the reference is checked against the stable-tie rule (oracle.amg.nms_stable): if they differed, the fixture would depend on
torch.sort's order of equal scores and is not written.  Records are stored as record_row()s: each RLE as its length and digest.
"""
from __future__ import annotations

import hashlib
import importlib.util
import json
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import amg as OA  # noqa: E402

SEED = 7
KEYS = ["segmentation", "area", "bbox", "predicted_iou", "point_coords", "stability_score", "crop_box"]
_F = dict(pred_iou_thresh=0.88, stability_score_thresh=0.95)      # the reference defaults
# (tag, image (h, w), generator kwargs): one full batch, a partial last batch, one and two crop layers, explicit point grids,
# both filters off (empty masks, NaN stability); both output modes
CASES = [
    ("one_batch", (150, 200), dict(points_per_side=8, points_per_batch=64, output_mode="uncompressed_rle", **_F)),
    ("partial_batch", (150, 200), dict(points_per_side=7, points_per_batch=16, box_nms_thresh=0.5, output_mode="binary_mask", **_F)),
    ("crops_1", (150, 200), dict(points_per_side=6, points_per_batch=20, crop_n_layers=1, output_mode="uncompressed_rle", **_F)),
    ("crops_2", (151, 203), dict(points_per_side=8, crop_n_layers=2, crop_n_points_downscale_factor=2, crop_nms_thresh=0.5,
                                 output_mode="binary_mask", **_F)),
    ("point_grids", (150, 200), dict(points_per_side=None, point_grids="seeded", points_per_batch=16, crop_n_layers=1,
                                     output_mode="uncompressed_rle", **_F)),
    ("no_filters", (97, 131), dict(points_per_side=6, pred_iou_thresh=0.0, stability_score_thresh=0.0, stability_score_offset=2.0,
                                   box_nms_thresh=0.1, output_mode="uncompressed_rle")),
]


def case_kwargs(kw):
    """A case's generator arguments, its explicit point grids (layer 0 and 1) regenerated from their seed."""
    kw = dict(kw)
    if kw.get("point_grids") == "seeded":
        rng = np.random.default_rng(11)
        kw["point_grids"] = [rng.uniform(0.02, 0.98, size=(30, 2)), rng.uniform(0.02, 0.98, size=(12, 2))]
    return kw


def record_row(r, digest=True):
    """One record as a list in KEYS order; a binary mask as its uncompressed RLE; an RLE as [h, w, runs, digest] (or as itself);
    NaN as "nan"."""
    assert list(r) == KEYS, list(r)
    seg = r["segmentation"]
    if isinstance(seg, np.ndarray):
        assert seg.dtype == bool
        seg = OA.mask_to_rle_pytorch(torch.from_numpy(seg)[None])[0]
    if digest:
        seg = [*seg["size"], len(seg["counts"]), hashlib.sha256(json.dumps(seg["counts"]).encode()).hexdigest()[:16]]
    f = lambda v: "nan" if math.isnan(v) else v
    assert float(r["area"]).is_integer() and all(float(v).is_integer() for v in r["bbox"] + r["crop_box"])
    return [seg, int(r["area"]), [int(v) for v in r["bbox"]], f(r["predicted_iou"]), r["point_coords"], f(r["stability_score"]),
            [int(v) for v in r["crop_box"]]]


class _StubPredictor:
    """student_sam/predictor.py's SamPredictor as _process_crop / _process_batch use it (AMG:236-285)."""

    def __init__(self, model):
        self.model, self._hw = model, None
        self.transform = types.SimpleNamespace(apply_coords=lambda coords, size: coords)   # the decoder takes crop pixels
        self.device = torch.device("cpu")

    def set_image(self, image):
        self._hw = tuple(image.shape[:2])

    def reset_image(self):
        self._hw = None

    def predict_torch(self, features, point_coords, point_labels, num_multimask_outputs=3, return_logits=False):
        assert num_multimask_outputs == 3 and return_logits and bool((point_labels == 1).all())
        low, iou = OA.synthetic_decoder(point_coords[:, 0, :].numpy(), self._hw, SEED)
        return OA.bilinear_upsample(low, *self._hw), iou, low


def load_reference_generator():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
    import install  # oracle/ref_shim/install.py
    install.install()
    pkg_dir = os.path.join(install.REFERENCE_ROOT, "sam3", "sam3", "model", "student_sam")
    name = "student_sam_ref"
    mods = {n: types.ModuleType(n) for n in (name, name + ".utils", name + ".modeling", name + ".predictor")}
    mods[name].__path__, mods[name + ".utils"].__path__ = [pkg_dir], []
    mods[name + ".modeling"].Sam = object
    mods[name + ".predictor"].SamPredictor = _StubPredictor
    sys.modules.update(mods, **{name + ".utils.amg": OA})
    spec = importlib.util.spec_from_file_location(name + ".automatic_mask_generator", os.path.join(pkg_dir, "automatic_mask_generator.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    real = mod.batched_nms

    def checked_nms(boxes, scores, idxs, iou_threshold):
        assert bool((idxs == 0).all())
        ref = real(boxes, scores, idxs, iou_threshold)
        assert ref.tolist() == OA.nms_stable(boxes, scores, iou_threshold).tolist(), "tie order differs: ambiguous fixture"
        return ref

    mod.batched_nms = checked_nms
    return mod.SamAutomaticMaskGenerator


def main():
    Gen = load_reference_generator()
    cases = []
    for tag, hw, kw in CASES:
        recs = Gen(types.SimpleNamespace(mask_threshold=0.0), **case_kwargs(kw)).generate(np.zeros((*hw, 3), dtype=np.uint8))
        print(f"{tag}: image {hw}, {len(recs)} records")
        cases.append({"tag": tag, "image_hw": list(hw), "kwargs": kw, "records": [record_row(r) for r in recs]})
    path = os.path.join(HERE, "amg_small.json")
    with open(path, "w") as f:    # one record per line
        f.write('{"seed": %d, "keys": %s, "cases": [\n' % (SEED, json.dumps(KEYS)))
        f.write(",\n".join('{"tag": %s, "image_hw": %s, "kwargs": %s, "records": [\n%s]}' % (
            json.dumps(c["tag"]), json.dumps(c["image_hw"]), json.dumps(c["kwargs"]),
            ",\n".join(json.dumps(r) for r in c["records"])) for c in cases))
        f.write("]}\n")
    json.load(open(path))
    print(path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
