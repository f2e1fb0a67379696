"""Automatic mask generation ("segment everything") on the point segmenter, with native post-processing.

Native counterpart of SamAutomaticMaskGenerator (sam3/sam3/model/student_sam/automatic_mask_generator.py:35-373), whose
utilities are those of SAM1's segment_anything/utils/amg.py.  A grid of single-point prompts is laid over the image and,
with crop_n_layers > 0, over overlapping crops of it.  Each crop is encoded once (SAM3InteractiveImagePredictor.set_image)
and its points are decoded in batches of points_per_batch (decode_prompts, three masks per point, no object gating).

The masks are never upsampled to the crop's size in memory.  For each decoded batch es3_amg_mask_stats evaluates every pixel
of every mask as the bilinear sample of its low-res logits (the value ops.bilinear_nchw would write), applies the
predicted-IoU filter, the stability-score filter and the crop-edge test, and appends the survivors (low-res logits, box,
scores, point) to a per-crop arena on the device.  es3_box_nms then removes duplicates within the crop, and across crops
(scored by 1 / crop area) when there are several.  es3_amg_rle encodes only the masks that remain.

Behaviour that differs from the reference, on purpose:
- predicted_iou is the SAM heads' IoU prediction, as SAM3InteractiveImagePredictor.predict returns it.  EdgeSAM's predictor
  replaces it by a low-res stability score by default (use_stability_score=True, student_sam/predictor.py:187, 249-252),
  a workaround for its distilled decoder; the SAM3 heads carry a trained sigmoid IoU head.
- Equal NMS scores are ordered by index (a stable descending sort).  The reference leaves that order to torch.sort; it
  matters in the cross-crop NMS, where every mask of a crop has the same score.
- min_mask_region_area > 0 is not supported (the reference runs OpenCV on the host for it).
- bbox and crop_box are always ints (the reference's become floats when a batch or crop kept no mask).

With the segmenter's CUDA graphs enabled, each batch's decode replays from its graph; the batch's outputs are consumed on
the device (copied into the arena) before the next decode overwrites them.
"""
from __future__ import annotations

import math
from itertools import product
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch

from .. import ops
from .sam1_task import SAM3InteractiveImagePredictor, host_transform_coords


# ------------------------------------------------------------------------------------------------------ host geometry (amg.py)
def build_point_grid(n_per_side: int) -> np.ndarray:
    """n_per_side^2 points evenly spaced in [0,1]^2, x fastest."""
    offset = 1 / (2 * n_per_side)
    points_one_side = np.linspace(offset, 1 - offset, n_per_side)
    points_x = np.tile(points_one_side[None, :], (n_per_side, 1))
    points_y = np.tile(points_one_side[:, None], (1, n_per_side))
    return np.stack([points_x, points_y], axis=-1).reshape(-1, 2)


def build_all_layer_point_grids(n_per_side: int, n_layers: int, scale_per_layer: int) -> List[np.ndarray]:
    """One point grid per crop layer; layer i has int(n_per_side / scale_per_layer**i) points per side."""
    return [build_point_grid(int(n_per_side / (scale_per_layer ** i))) for i in range(n_layers + 1)]


def generate_crop_boxes(im_size: Tuple[int, ...], n_layers: int, overlap_ratio: float) -> Tuple[List[List[int]], List[int]]:
    """The whole image, then 2^(i+1) x 2^(i+1) overlapping crops per layer i, as XYXY boxes, with their layer indices."""
    crop_boxes, layer_idxs = [], []
    im_h, im_w = im_size
    short_side = min(im_h, im_w)
    crop_boxes.append([0, 0, im_w, im_h])
    layer_idxs.append(0)

    def crop_len(orig_len, n_crops, overlap):
        return int(math.ceil((overlap * (n_crops - 1) + orig_len) / n_crops))

    for i_layer in range(n_layers):
        n_crops_per_side = 2 ** (i_layer + 1)
        overlap = int(overlap_ratio * short_side * (2 / n_crops_per_side))
        crop_w = crop_len(im_w, n_crops_per_side, overlap)
        crop_h = crop_len(im_h, n_crops_per_side, overlap)
        crop_box_x0 = [int((crop_w - overlap) * i) for i in range(n_crops_per_side)]
        crop_box_y0 = [int((crop_h - overlap) * i) for i in range(n_crops_per_side)]
        for x0, y0 in product(crop_box_x0, crop_box_y0):
            crop_boxes.append([x0, y0, min(x0 + crop_w, im_w), min(y0 + crop_h, im_h)])
            layer_idxs.append(i_layer + 1)
    return crop_boxes, layer_idxs


def _xywh(b) -> List[int]:
    return [int(b[0]), int(b[1]), int(b[2]) - int(b[0]), int(b[3]) - int(b[1])]


class SamAutomaticMaskGenerator:
    def __init__(self, model, points_per_side: Optional[int] = 32, points_per_batch: int = 64, pred_iou_thresh: float = 0.88,
                 stability_score_thresh: float = 0.95, stability_score_offset: float = 1.0, box_nms_thresh: float = 0.7,
                 crop_n_layers: int = 0, crop_nms_thresh: float = 0.7, crop_overlap_ratio: float = 512 / 1500,
                 crop_n_points_downscale_factor: int = 1, point_grids: Optional[List[np.ndarray]] = None,
                 min_mask_region_area: int = 0, output_mode: str = "binary_mask") -> None:
        """model: a Sam3PointPromptSegmenter (the SAM3 ViT one or one from build_efficientsam3_point_segmenter).  The
        arguments are the reference's (automatic_mask_generator.py:53-96); output_mode is 'binary_mask', 'uncompressed_rle'
        or 'coco_rle' (which needs pycocotools)."""
        assert (points_per_side is None) != (point_grids is None), "Exactly one of points_per_side or point_grid must be provided."
        if points_per_side is not None:
            self.point_grids = build_all_layer_point_grids(points_per_side, crop_n_layers, crop_n_points_downscale_factor)
        elif point_grids is not None:
            self.point_grids = point_grids
        else:
            raise ValueError("Can't have both points_per_side and point_grid be None.")
        assert output_mode in ["binary_mask", "uncompressed_rle", "coco_rle"], f"Unknown output_mode {output_mode}."
        if output_mode == "coco_rle":
            from pycocotools import mask as mask_utils  # type: ignore # noqa: F401
        if min_mask_region_area > 0:
            raise NotImplementedError("min_mask_region_area > 0 is not supported: the reference removes small regions with "
                                      "OpenCV on the host, and its keep-the-largest-island rule is not es3_fill_small_components'")
        # the reference's AMG predictor fills no holes: the default max_hole_area of the interactive predictor must not apply
        self.predictor = SAM3InteractiveImagePredictor(model, mask_threshold=0.0, max_hole_area=0.0, max_sprinkle_area=0.0)
        self.points_per_batch = points_per_batch
        self.pred_iou_thresh = pred_iou_thresh
        self.stability_score_thresh = stability_score_thresh
        self.stability_score_offset = stability_score_offset
        self.box_nms_thresh = box_nms_thresh
        self.crop_n_layers = crop_n_layers
        self.crop_nms_thresh = crop_nms_thresh
        self.crop_overlap_ratio = crop_overlap_ratio
        self.crop_n_points_downscale_factor = crop_n_points_downscale_factor
        self.min_mask_region_area = min_mask_region_area
        self.output_mode = output_mode

    @property
    def device(self):
        return self.predictor.device

    @torch.no_grad()
    def generate(self, image: np.ndarray) -> List[Dict[str, Any]]:
        """image: HWC uint8.  -> one record per mask, best first: segmentation (bool [H,W] ndarray or an RLE dict), area,
        bbox (XYWH), predicted_iou, point_coords, stability_score, crop_box (XYWH) -- the reference's keys and order."""
        orig_size = tuple(image.shape[:2])
        crop_boxes, layer_idxs = generate_crop_boxes(orig_size, self.crop_n_layers, self.crop_overlap_ratio)
        crops = [self._process_crop(image, cb, li, orig_size) for cb, li in zip(crop_boxes, layer_idxs)]
        sizes = [c["n"] for c in crops]
        dev = self.device
        boxes = torch.cat([c["box"] for c in crops])
        if len(crop_boxes) > 1:
            # prefer masks from smaller crops: 1 / box_area(crop_box) in fp32, as torch divides 1 by the int64 areas
            areas = torch.tensor([(c["crop_box"][2] - c["crop_box"][0]) * (c["crop_box"][3] - c["crop_box"][1]) for c in crops],
                                 dtype=torch.float32)
            scores = torch.repeat_interleave(1 / areas, torch.tensor(sizes)).to(dev)
            keep, cnt = ops.box_nms(boxes, scores, self.crop_nms_thresh)
            order = keep[:int(cnt.item())].long().cpu()
        else:
            order = torch.arange(sizes[0])
        return self._records(crops, order, orig_size)

    # ---- model side: the one seam a test substitutes ---------------------------------------------------------------------
    def _decode_crop(self, cropped_im: np.ndarray, points: np.ndarray):
        """Encode the crop and yield (low-res logits [P,3,Hl,Wl] fp32, iou [P,3] fp32) on the device for each batch of
        `points` ([n,2] crop pixels, float64), in order.  Each batch must be consumed before the next is requested: a
        graph replay overwrites its outputs."""
        self.predictor.set_image(cropped_im)
        seg = self.predictor.model
        h, w = cropped_im.shape[:2]
        coords = host_transform_coords(torch.as_tensor(points, dtype=torch.float), True, (h, w), seg.image_size).to(self.device)
        labels = torch.ones((len(points), 1), dtype=torch.int32, device=self.device)
        for b in range(0, len(points), self.points_per_batch):
            sl = slice(b, b + self.points_per_batch)
            low, iou, _ = seg.decode_prompts(0, (coords[sl, None, :], labels[sl]), multimask_output=True, obj_gate=False)
            yield low, iou
        self.predictor.reset_predictor()

    # ---- one crop ------------------------------------------------------------------------------------------------------
    def _process_crop(self, image, crop_box, crop_layer_idx, orig_size):
        x0, y0, x1, y1 = crop_box
        cropped_im = image[y0:y1, x0:x1, :]
        h, w = cropped_im.shape[:2]
        points = self.point_grids[crop_layer_idx] * np.array([w, h])[None, :]
        arena, base = None, 0
        for low, iou in self._decode_crop(cropped_im, points):
            if arena is None:
                arena = self._arena(len(points) * low.shape[1], low.shape[-2], low.shape[-1])
            ops.amg_mask_stats(low.float(), iou.float(), crop_box, orig_size, arena, self.predictor.mask_threshold,
                               self.stability_score_offset, self.pred_iou_thresh, self.stability_score_thresh, point_base=base)
            base += low.shape[0]
        n = int(arena.count.item())                      # the one read of the crop's survivors
        assert n <= arena.cap, (n, arena.cap)
        keep, cnt = ops.box_nms(arena.box[:n], arena.iou[:n], self.box_nms_thresh)
        keep = keep[:int(cnt.item())].long()
        off = torch.tensor([x0, y0, x0, y0], dtype=torch.int32, device=arena.box.device)
        pts = arena.point[keep].long().cpu().numpy()
        return dict(crop_box=list(crop_box), n=int(keep.numel()), low=arena.low[keep], box=arena.box[keep] + off,
                    iou=arena.iou[keep], stab=arena.stab[keep],
                    points=points[pts] + np.array([x0, y0])[None, :])   # uncrop_points: float64 + int offset

    def _arena(self, cap, Hl, Wl):
        a = getattr(self, "_arena_buf", None)
        if a is None or a.cap < cap or (a.Hi, a.Wi) != (Hl, Wl) or a.low.device != self.device:
            a = self._arena_buf = ops.AmgArena(cap, Hl, Wl, self.device)
        return a.reset()

    # ---- encoding and records ------------------------------------------------------------------------------------------
    def _encode(self, low, crop_box, orig_size):
        """RLE counts (lists), areas and (binary_mask) bool masks of the masks low [k,Hl,Wl] of one crop."""
        H, W = orig_size
        binary = self.output_mode == "binary_mask"
        pos, n_trans, area, binm = ops.amg_rle(low, crop_box, orig_size, self.predictor.mask_threshold, binary=binary)
        n = n_trans.cpu().numpy()
        over = np.nonzero(n > pos.shape[1])[0]
        pos = pos.cpu().numpy()
        extra = {}
        if len(over) and not binary:     # a mask with more transitions than the default buffer: once more at its size
            p2, _, _, _ = ops.amg_rle(low[torch.as_tensor(over, device=low.device)], crop_box, orig_size,
                                      self.predictor.mask_threshold, cap=int(n[over].max()))
            extra = dict(zip(over.tolist(), p2.cpu().numpy()))
        counts = None
        if not binary:
            counts = []
            for i in range(len(n)):
                row = extra[i] if i in extra else pos[i]
                counts.append(np.diff(np.concatenate([[0], row[:n[i]], [H * W]])).tolist())
        return counts, area.cpu().numpy(), (binm.bool().cpu().numpy() if binary else None)

    def _records(self, crops, order, orig_size):
        H, W = orig_size
        starts = np.cumsum([0] + [c["n"] for c in crops])
        order = order.numpy()
        which = np.searchsorted(starts, order, side="right") - 1
        enc = {}
        for ci, c in enumerate(crops):
            sel = order[which == ci] - starts[ci]
            if len(sel):
                counts, area, binm = self._encode(c["low"][torch.as_tensor(sel, device=c["low"].device)], c["crop_box"], orig_size)
                for j, s in enumerate(sel.tolist()):
                    enc[(ci, s)] = (counts[j] if counts is not None else None, int(area[j]), binm[j] if binm is not None else None)
        host = [dict(box=c["box"].cpu().numpy(), iou=c["iou"].cpu().numpy(), stab=c["stab"].cpu().numpy()) for c in crops]
        anns = []
        for g, ci in zip(order.tolist(), which.tolist()):
            i = g - int(starts[ci])
            counts, area, binm = enc[(ci, i)]
            if self.output_mode == "binary_mask":
                seg = binm
            else:
                seg = {"size": [H, W], "counts": counts}
                if self.output_mode == "coco_rle":
                    seg = coco_encode_rle(seg)
            anns.append({
                "segmentation": seg,
                "area": area,
                "bbox": _xywh(host[ci]["box"][i]),
                "predicted_iou": float(host[ci]["iou"][i]),
                "point_coords": [crops[ci]["points"][i].tolist()],
                "stability_score": float(host[ci]["stab"][i]),
                "crop_box": _xywh(crops[ci]["crop_box"]),
            })
        return anns


def coco_encode_rle(uncompressed_rle: Dict[str, Any]) -> Dict[str, Any]:
    """An uncompressed column-major RLE as pycocotools' compressed RLE, counts as a str."""
    from pycocotools import mask as mask_utils  # type: ignore
    h, w = uncompressed_rle["size"]
    rle = mask_utils.frPyObjects(uncompressed_rle, h, w)
    rle["counts"] = rle["counts"].decode("utf-8")
    return rle
