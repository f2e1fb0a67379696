"""Time of SamAutomaticMaskGenerator.generate per image: native post-processing against the oracle's eager torch one
(oracle.amg.generate, the reference's post-processing with the logits upsampled by ops.bilinear_nchw and torchvision's CUDA NMS
on tie-free scores in the stable-tie order), fed the same decoder outputs on the same GPU.  Prints one JSON line.

    python scripts/bench_amg.py [--rounds 1] [--points-per-side 32] [--models "EV-M,SAM3 ViT"] [--out results.json]

Seeded 1500 x 2250 uint8 image; the EV-M and SAM3 ViT point segmenters at 1008^2 with default initialisation; crop_n_layers 0
and 1; both filters off, so every mask reaches NMS (default weights would otherwise drop every mask).  Each call is split by
CUDA events into encode (set_image_batch), decode (decode_prompts) and post-processing (the rest of the wall time).  The arms
alternate over --rounds after one warm-up round; native and eager records must be equal before any time is reported.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_text import gpu_info  # noqa: E402


class Timer:
    """CUDA events around the segmenter's set_image_batch and decode_prompts; summed when read."""

    def __init__(self, seg):
        self.ev = {"encode": [], "decode": []}
        for name, kind in (("set_image_batch", "encode"), ("decode_prompts", "decode")):
            fn = getattr(seg, name)

            def wrapped(*a, _fn=fn, _kind=kind, **k):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = _fn(*a, **k)
                e1.record()
                self.ev[_kind].append((e0, e1))
                return out
            setattr(seg, name, wrapped)

    def reset(self):
        for v in self.ev.values():
            v.clear()

    def read(self):
        torch.cuda.synchronize()
        return {k: sum(a.elapsed_time(b) for a, b in v) for k, v in self.ev.items()}


def tie_free_nms(boxes, scores, thr):
    """torchvision's CUDA batched_nms with scores replaced by their rank in a stable descending sort (distinct, same order)."""
    from torchvision.ops import batched_nms
    order = torch.sort(scores, descending=True, stable=True).indices
    rank = torch.empty_like(order)
    rank[order] = torch.arange(len(order), device=order.device)
    return batched_nms(boxes.float(), (len(order) - rank).float(), torch.zeros_like(rank), thr)


def eager_generate(gen, image):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model.sam1_task import host_transform_coords
    from oracle import amg as OA
    pred, seg = gen.predictor, gen.predictor.model
    cur = {}

    def decode(crop_box, points, hw):
        if cur.get("box") != crop_box:
            x0, y0, x1, y1 = crop_box
            pred.set_image(image[y0:y1, x0:x1, :])
            cur["box"] = crop_box
        c = host_transform_coords(torch.as_tensor(points, dtype=torch.float), True, hw, seg.image_size).to(pred.device)
        lab = torch.ones((len(points), 1), dtype=torch.int32, device=pred.device)
        low, iou, _ = seg.decode_prompts(0, (c[:, None, :], lab), multimask_output=True, obj_gate=False)
        return low, iou

    return OA.generate(image.shape[:2], decode, gen.point_grids, points_per_batch=gen.points_per_batch,
                       pred_iou_thresh=gen.pred_iou_thresh, stability_score_thresh=gen.stability_score_thresh,
                       stability_score_offset=gen.stability_score_offset, box_nms_thresh=gen.box_nms_thresh,
                       crop_n_layers=gen.crop_n_layers, crop_nms_thresh=gen.crop_nms_thresh,
                       crop_overlap_ratio=gen.crop_overlap_ratio, output_mode=gen.output_mode,
                       upsample=lambda low, h, w: ops.bilinear_nchw(low, h, w)[0], nms=tie_free_nms)


def as_ints(recs):
    """The records with integer bbox / crop_box: the reference's are floats when a crop or batch kept no mask."""
    return [dict(r, bbox=[int(v) for v in r["bbox"]], crop_box=[int(v) for v in r["crop_box"]]) for r in recs]


def first_difference(a, b):
    """The first pair of records that differ, each field but the segmentation's runs (their count instead)."""
    brief = lambda r: dict(r, segmentation=dict(size=r["segmentation"]["size"], runs=len(r["segmentation"]["counts"])))
    for i, (x, y) in enumerate(zip(a, b)):
        if json.dumps(x) != json.dumps(y):
            return dict(index=i, native=brief(x), eager=brief(y))
    return dict(n_native=len(a), n_eager=len(b))


def run(arm, gen, timer, image):
    timer.reset()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    recs = gen.generate(image) if arm == "native" else eager_generate(gen, image)
    torch.cuda.synchronize()
    total = (time.perf_counter() - t0) * 1e3
    t = timer.read()
    return recs, dict(total_ms=total, encode_ms=t["encode"], decode_ms=t["decode"], post_ms=total - t["encode"] - t["decode"],
                      peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--points-per-side", type=int, default=32)
    ap.add_argument("--models", default="EV-M,SAM3 ViT", help="comma-separated subset of: EV-M, SAM3 ViT")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from efficientsam3_b200.model.automatic_mask_generator import SamAutomaticMaskGenerator
    from efficientsam3_b200.model.sam1_task import Sam3PointPromptSegmenter
    from efficientsam3_b200.model_builder import build_efficientsam3_point_segmenter
    assert torch.cuda.is_available(), "bench_amg.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    res = dict(**gpu_info(dev), image=[1500, 2250], points_per_side=args.points_per_side, rounds=args.rounds,
               pred_iou_thresh=0.0, stability_score_thresh=0.0, arms={}, records_equal=True)
    image = np.random.default_rng(0).integers(0, 256, size=(1500, 2250, 3), dtype=np.uint8)
    models = [("EV-M", lambda: build_efficientsam3_point_segmenter("efficientvit", "b1")), ("SAM3 ViT", Sam3PointPromptSegmenter)]
    for mname, make in models:
        if mname not in args.models.split(","):
            continue
        seg = make().to(dev).eval()
        timer = Timer(seg)
        gens = {L: SamAutomaticMaskGenerator(seg, points_per_side=args.points_per_side, pred_iou_thresh=0.0,
                                             stability_score_thresh=0.0, crop_n_layers=L, output_mode="uncompressed_rle")
                for L in (0, 1)}
        samples = {}
        for r in range(args.rounds + 1):            # round 0 warms up every arm
            for L in (0, 1):
                recs = {}
                for arm in ("native", "eager"):
                    recs[arm], t = run(arm, gens[L], timer, image)
                    print(f"{mname} crops{L} {arm} round {r}: {len(recs[arm])} records, " +
                          ", ".join(f"{k} {v:.1f}" for k, v in t.items()), file=sys.stderr, flush=True)
                    if r:
                        samples.setdefault((L, arm), []).append(t)
                recs = {k: as_ints(v) for k, v in recs.items()}
                if json.dumps(recs["native"]) != json.dumps(recs["eager"]):
                    res["records_equal"] = False
                    print(json.dumps(dict(res, error=f"{mname} crop_n_layers={L}: native and eager records differ",
                                          first_difference=first_difference(recs["native"], recs["eager"]))))
                    sys.exit(1)
                res.setdefault("records", {})[f"{mname} crops{L}"] = len(recs["native"])
        for (L, arm), ts in samples.items():
            res["arms"][f"{mname} crops{L} {arm}"] = {k: round(float(np.median([t[k] for t in ts])), 2) for k in ts[0]}
        del seg, gens, timer
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
