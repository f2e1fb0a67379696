"""Automatic mask generation: the SAM1 utilities the reference generator imports, its post-processing in eager torch, a
stable-tie NMS, and a seeded synthetic decoder.

sam3/sam3/model/student_sam/automatic_mask_generator.py imports `.utils.amg`, which the reference does not ship
(student_sam/utils/ holds __init__.py and common.py only).  Its semantics are those of the published SAM1
segment_anything/utils/amg.py; each function below is restated from them and cites its call site in the reference generator
(automatic_mask_generator.py, "AMG:<line>").  `generate` runs the generator's post-processing (AMG:197-322) on decoder outputs
given by a callable, so the native generator can be compared with it on any decoder.

The synthetic decoder makes Gaussian-bump logits around each point whose bilinear resize to the crop is exact in fp32 in any
evaluation order (see synthetic_decoder), so a record computed on the CPU and one computed on the GPU can be compared bit for
bit.
"""
from __future__ import annotations

import math
import zlib
from copy import deepcopy
from itertools import product
from typing import Any, Dict, List, Tuple

import numpy as np
import torch
import torch.nn.functional as F


# ------------------------------------------------------------------------------------------------------ MaskData (AMG:204-246)
class MaskData:
    """A structure for storing masks and their related data in batched format (AMG:204, 243, 288)."""

    def __init__(self, **kwargs) -> None:
        for v in kwargs.values():
            assert isinstance(v, (list, np.ndarray, torch.Tensor)), "MaskData only supports list, numpy arrays, and torch tensors."
        self._stats = dict(**kwargs)

    def __setitem__(self, key: str, item: Any) -> None:
        assert isinstance(item, (list, np.ndarray, torch.Tensor)), "MaskData only supports list, numpy arrays, and torch tensors."
        self._stats[key] = item

    def __delitem__(self, key: str) -> None:
        del self._stats[key]

    def __getitem__(self, key: str) -> Any:
        return self._stats[key]

    def items(self):
        return self._stats.items()

    def filter(self, keep: torch.Tensor) -> None:
        for k, v in self._stats.items():
            if v is None:
                self._stats[k] = None
            elif isinstance(v, torch.Tensor):
                self._stats[k] = v[torch.as_tensor(keep, device=v.device)]
            elif isinstance(v, np.ndarray):
                self._stats[k] = v[keep.detach().cpu().numpy()]
            elif isinstance(v, list) and keep.dtype == torch.bool:
                self._stats[k] = [a for i, a in enumerate(v) if keep[i]]
            elif isinstance(v, list):
                self._stats[k] = [v[i] for i in keep]
            else:
                raise TypeError(f"MaskData key {k} has an unsupported type {type(v)}.")

    def cat(self, new_stats: "MaskData") -> None:
        for k, v in new_stats.items():
            if k not in self._stats or self._stats[k] is None:
                self._stats[k] = deepcopy(v)
            elif isinstance(v, torch.Tensor):
                self._stats[k] = torch.cat([self._stats[k], v], dim=0)
            elif isinstance(v, np.ndarray):
                self._stats[k] = np.concatenate([self._stats[k], v], axis=0)
            elif isinstance(v, list):
                self._stats[k] = self._stats[k] + deepcopy(v)
            else:
                raise TypeError(f"MaskData key {k} has an unsupported type {type(v)}.")

    def to_numpy(self) -> None:
        for k, v in self._stats.items():
            if isinstance(v, torch.Tensor):
                self._stats[k] = v.detach().cpu().numpy()


# ------------------------------------------------------------------------------------------------------ utilities
def is_box_near_crop_edge(boxes, crop_box, orig_box, atol: float = 20.0):
    """AMG:313.  Whether a box touches (within atol) a crop edge that is not an image edge."""
    crop_box_torch = torch.as_tensor(crop_box, dtype=torch.float, device=boxes.device)
    orig_box_torch = torch.as_tensor(orig_box, dtype=torch.float, device=boxes.device)
    boxes = uncrop_boxes_xyxy(boxes, crop_box).float()
    near_crop_edge = torch.isclose(boxes, crop_box_torch[None, :], atol=atol, rtol=0)
    near_image_edge = torch.isclose(boxes, orig_box_torch[None, :], atol=atol, rtol=0)
    near_crop_edge = torch.logical_and(near_crop_edge, ~near_image_edge)
    return torch.any(near_crop_edge, dim=1)


def box_xyxy_to_xywh(box_xyxy):
    """AMG:187, 191."""
    box_xywh = deepcopy(box_xyxy)
    box_xywh[2] = box_xywh[2] - box_xywh[0]
    box_xywh[3] = box_xywh[3] - box_xywh[1]
    return box_xywh


def batch_iterator(batch_size: int, *args):
    """AMG:244."""
    assert len(args) > 0 and all(len(a) == len(args[0]) for a in args), "Batched iteration must have inputs of all the same size."
    n_batches = len(args[0]) // batch_size + int(len(args[0]) % batch_size != 0)
    for b in range(n_batches):
        yield [arg[b * batch_size:(b + 1) * batch_size] for arg in args]


def mask_to_rle_pytorch(tensor: torch.Tensor) -> List[Dict[str, Any]]:
    """AMG:319.  Masks [B,H,W] bool -> uncompressed RLEs in column-major order (a zero-length first run when pixel 0 is set)."""
    b, h, w = tensor.shape
    tensor = tensor.permute(0, 2, 1).flatten(1)
    diff = tensor[:, 1:] ^ tensor[:, :-1]
    change_indices = diff.nonzero()
    out = []
    for i in range(b):
        cur_idxs = change_indices[change_indices[:, 0] == i, 1]
        cur_idxs = torch.cat([
            torch.tensor([0], dtype=cur_idxs.dtype, device=cur_idxs.device),
            cur_idxs + 1,
            torch.tensor([h * w], dtype=cur_idxs.dtype, device=cur_idxs.device),
        ])
        btw_idxs = cur_idxs[1:] - cur_idxs[:-1]
        counts = [] if tensor[i, 0] == 0 else [0]
        counts.extend(btw_idxs.detach().cpu().tolist())
        out.append({"size": [h, w], "counts": counts})
    return out


def rle_to_mask(rle: Dict[str, Any]) -> np.ndarray:
    """AMG:177.  Uncompressed RLE -> bool [H,W]."""
    h, w = rle["size"]
    mask = np.empty(h * w, dtype=bool)
    idx = 0
    parity = False
    for count in rle["counts"]:
        mask[idx:idx + count] = parity
        idx += count
        parity ^= True
    mask = mask.reshape(w, h)
    return mask.transpose()


def area_from_rle(rle: Dict[str, Any]) -> int:
    """AMG:186."""
    return sum(rle["counts"][1::2])


def calculate_stability_score(masks: torch.Tensor, mask_threshold: float, threshold_offset: float) -> torch.Tensor:
    """AMG:301.  IoU of the masks thresholded at thr + offset and thr - offset; int16 row sums, then int32."""
    intersections = (masks > (mask_threshold + threshold_offset)).sum(-1, dtype=torch.int16).sum(-1, dtype=torch.int32)
    unions = (masks > (mask_threshold - threshold_offset)).sum(-1, dtype=torch.int16).sum(-1, dtype=torch.int32)
    return intersections / unions


def build_point_grid(n_per_side: int) -> np.ndarray:
    offset = 1 / (2 * n_per_side)
    points_one_side = np.linspace(offset, 1 - offset, n_per_side)
    points_x = np.tile(points_one_side[None, :], (n_per_side, 1))
    points_y = np.tile(points_one_side[:, None], (1, n_per_side))
    points = np.stack([points_x, points_y], axis=-1).reshape(-1, 2)
    return points


def build_all_layer_point_grids(n_per_side: int, n_layers: int, scale_per_layer: int) -> List[np.ndarray]:
    """AMG:102."""
    points_by_layer = []
    for i in range(n_layers + 1):
        n_points = int(n_per_side / (scale_per_layer ** i))
        points_by_layer.append(build_point_grid(n_points))
    return points_by_layer


def generate_crop_boxes(im_size: Tuple[int, ...], n_layers: int, overlap_ratio: float) -> Tuple[List[List[int]], List[int]]:
    """AMG:199."""
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
            box = [x0, y0, min(x0 + crop_w, im_w), min(y0 + crop_h, im_h)]
            crop_boxes.append(box)
            layer_idxs.append(i_layer + 1)
    return crop_boxes, layer_idxs


def uncrop_boxes_xyxy(boxes: torch.Tensor, crop_box: List[int]) -> torch.Tensor:
    """AMG:260."""
    x0, y0, _, _ = crop_box
    offset = torch.tensor([[x0, y0, x0, y0]], device=boxes.device)
    if len(boxes.shape) == 3:
        offset = offset.unsqueeze(1)
    return boxes + offset


def uncrop_points(points: torch.Tensor, crop_box: List[int]) -> torch.Tensor:
    """AMG:261."""
    x0, y0, _, _ = crop_box
    offset = torch.tensor([[x0, y0]], device=points.device)
    if len(points.shape) == 3:
        offset = offset.unsqueeze(1)
    return points + offset


def uncrop_masks(masks: torch.Tensor, crop_box: List[int], orig_h: int, orig_w: int) -> torch.Tensor:
    """AMG:318."""
    x0, y0, x1, y1 = crop_box
    if x0 == 0 and y0 == 0 and x1 == orig_w and y1 == orig_h:
        return masks
    pad_x, pad_y = orig_w - (x1 - x0), orig_h - (y1 - y0)
    pad = (x0, pad_x - x0, y0, pad_y - y0)
    return torch.nn.functional.pad(masks, pad, value=0)


def batched_mask_to_box(masks: torch.Tensor) -> torch.Tensor:
    """AMG:310.  XYXY boxes (inclusive max) around bool masks [..., H, W]; [0,0,0,0] for an empty mask."""
    if torch.numel(masks) == 0:
        return torch.zeros(*masks.shape[:-2], 4, device=masks.device)
    shape = masks.shape
    h, w = shape[-2:]
    if len(shape) > 2:
        masks = masks.flatten(0, -3)
    else:
        masks = masks.unsqueeze(0)
    in_height, _ = torch.max(masks, dim=-1)
    in_height_coords = in_height * torch.arange(h, device=in_height.device)[None, :]
    bottom_edges, _ = torch.max(in_height_coords, dim=-1)
    in_height_coords = in_height_coords + h * (~in_height)
    top_edges, _ = torch.min(in_height_coords, dim=-1)
    in_width, _ = torch.max(masks, dim=-2)
    in_width_coords = in_width * torch.arange(w, device=in_width.device)[None, :]
    right_edges, _ = torch.max(in_width_coords, dim=-1)
    in_width_coords = in_width_coords + w * (~in_width)
    left_edges, _ = torch.min(in_width_coords, dim=-1)
    empty_filter = (right_edges < left_edges) | (bottom_edges < top_edges)
    out = torch.stack([left_edges, top_edges, right_edges, bottom_edges], dim=-1)
    out = out * (~empty_filter).unsqueeze(-1)
    if len(shape) > 2:
        out = out.reshape(*shape[:-2], 4)
    else:
        out = out[0]
    return out


def coco_encode_rle(uncompressed_rle: Dict[str, Any]) -> Dict[str, Any]:
    """AMG:175 (coco_rle).  Imported by the reference generator; pycocotools is not installed here."""
    from pycocotools import mask as mask_utils  # type: ignore
    h, w = uncompressed_rle["size"]
    rle = mask_utils.frPyObjects(uncompressed_rle, h, w)
    rle["counts"] = rle["counts"].decode("utf-8")
    return rle


def remove_small_regions(mask, area_thresh, mode):
    """AMG:345 (min_mask_region_area > 0 only), imported by the reference generator; not restated."""
    raise NotImplementedError("min_mask_region_area > 0 is not restated")


# ------------------------------------------------------------------------------------------------------ NMS with a defined tie order
def nms_stable(boxes: torch.Tensor, scores: torch.Tensor, iou_threshold: float) -> torch.Tensor:
    """torchvision.ops.batched_nms with one category (AMG:214, 251), equal scores taken in index order (a stable descending
    sort; NaN first, as torch.sort).  IoU in fp32 as torchvision's CPU kernel: inter / (area_i + area_j - inter), areas
    (x2 - x1)(y2 - y1), suppression when IoU > iou_threshold (compared in double)."""
    b = boxes.detach().cpu().float()
    s = scores.detach().cpu().float()
    order = torch.sort(s, descending=True, stable=True).indices
    x1, y1, x2, y2 = b.unbind(1)
    areas = (x2 - x1) * (y2 - y1)
    suppressed = torch.zeros(len(s), dtype=torch.bool)
    keep = []
    for i in order.tolist():
        if suppressed[i]:
            continue
        keep.append(i)
        w = (torch.minimum(x2[i], x2) - torch.maximum(x1[i], x1)).clamp_min(0)
        h = (torch.minimum(y2[i], y2) - torch.maximum(y1[i], y1)).clamp_min(0)
        inter = w * h
        ovr = inter / (areas[i] + areas - inter)
        suppressed |= ovr.double() > iou_threshold
    return torch.tensor(keep, dtype=torch.int64, device=boxes.device)


# ------------------------------------------------------------------------------------------------------ post-processing
def bilinear_upsample(low: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """F.interpolate(bilinear, align_corners=False), the reference's upsampling of low-res logits (predictor.py:178-262)."""
    return F.interpolate(low, (h, w), mode="bilinear", align_corners=False)


def generate(image_size, decode, point_grids, points_per_batch=64, pred_iou_thresh=0.88, stability_score_thresh=0.95,
             stability_score_offset=1.0, box_nms_thresh=0.7, crop_n_layers=0, crop_nms_thresh=0.7, crop_overlap_ratio=512 / 1500,
             output_mode="binary_mask", mask_threshold=0.0, upsample=bilinear_upsample, nms=nms_stable):
    """SamAutomaticMaskGenerator.generate (AMG:136-322) with min_mask_region_area = 0, on decoder outputs:
    decode(crop_box, points [P,2] float64 crop pixels, crop (h, w)) -> (low-res logits [P,3,Hl,Wl] fp32, iou [P,3] fp32);
    upsample(low [P,3,Hl,Wl], h, w) -> logits at the crop size.  -> the reference's records."""
    orig_size = tuple(image_size)
    crop_boxes, layer_idxs = generate_crop_boxes(orig_size, crop_n_layers, crop_overlap_ratio)
    data = MaskData()
    for crop_box, layer_idx in zip(crop_boxes, layer_idxs):
        x0, y0, x1, y1 = crop_box
        cropped_im_size = (y1 - y0, x1 - x0)
        points_scale = np.array(cropped_im_size)[None, ::-1]
        points_for_image = point_grids[layer_idx] * points_scale
        crop_data = MaskData()
        for (points,) in batch_iterator(points_per_batch, points_for_image):
            low, iou = decode(crop_box, points, cropped_im_size)
            masks = upsample(low, *cropped_im_size)
            b = _process_batch(masks, iou, points, crop_box, orig_size, pred_iou_thresh, stability_score_thresh,
                               stability_score_offset, mask_threshold)
            crop_data.cat(b)
        keep_by_nms = nms(crop_data["boxes"].float(), crop_data["iou_preds"], box_nms_thresh)
        crop_data.filter(keep_by_nms)
        crop_data["boxes"] = uncrop_boxes_xyxy(crop_data["boxes"], crop_box)
        crop_data["points"] = uncrop_points(crop_data["points"], crop_box)
        crop_data["crop_boxes"] = torch.tensor([crop_box for _ in range(len(crop_data["rles"]))])
        data.cat(crop_data)
    if len(crop_boxes) > 1:
        cb = data["crop_boxes"]
        scores = 1 / ((cb[:, 2] - cb[:, 0]) * (cb[:, 3] - cb[:, 1]))      # 1 / box_area(crop_boxes)
        keep_by_nms = nms(data["boxes"].float(), scores.to(data["boxes"].device), crop_nms_thresh)
        data.filter(keep_by_nms)
    data.to_numpy()
    return records(data, output_mode)


def _process_batch(masks, iou, points, crop_box, orig_size, pred_iou_thresh, stability_score_thresh, stability_score_offset,
                   mask_threshold):
    """AMG:266-322 after predict_torch."""
    orig_h, orig_w = orig_size
    data = MaskData(masks=masks.flatten(0, 1), iou_preds=iou.flatten(0, 1),
                    points=torch.as_tensor(points.repeat(masks.shape[1], axis=0)))
    if pred_iou_thresh > 0.0:
        data.filter(data["iou_preds"] > pred_iou_thresh)
    data["stability_score"] = calculate_stability_score(data["masks"], mask_threshold, stability_score_offset)
    if stability_score_thresh > 0.0:
        data.filter(data["stability_score"] >= stability_score_thresh)
    data["masks"] = data["masks"] > mask_threshold
    data["boxes"] = batched_mask_to_box(data["masks"])
    keep_mask = ~is_box_near_crop_edge(data["boxes"], crop_box, [0, 0, orig_w, orig_h])
    if not torch.all(keep_mask):
        data.filter(keep_mask)
    data["masks"] = uncrop_masks(data["masks"], crop_box, orig_h, orig_w)
    data["rles"] = mask_to_rle_pytorch(data["masks"])
    del data["masks"]
    return data


def records(mask_data, output_mode):
    """AMG:173-195."""
    assert output_mode in ("binary_mask", "uncompressed_rle"), output_mode
    if output_mode == "binary_mask":
        segs = [rle_to_mask(rle) for rle in mask_data["rles"]]
    else:
        segs = mask_data["rles"]
    anns = []
    for idx in range(len(segs)):
        anns.append({
            "segmentation": segs[idx],
            "area": area_from_rle(mask_data["rles"][idx]),
            "bbox": box_xyxy_to_xywh(mask_data["boxes"][idx]).tolist(),
            "predicted_iou": mask_data["iou_preds"][idx].item(),
            "point_coords": [mask_data["points"][idx].tolist()],
            "stability_score": mask_data["stability_score"][idx].item(),
            "crop_box": box_xyxy_to_xywh(mask_data["crop_boxes"][idx]).tolist(),
        })
    return anns


# ------------------------------------------------------------------------------------------------------ synthetic decoder
def synthetic_low_res_size(n: int) -> int:
    """The low-res side for a crop side n: n / 2 for even n (a 2x upsample, weights 1/4 and 3/4), 2 n for odd n (a 2x
    downsample, weights 1/2).  With logits on a 1/64 grid below 128 in magnitude every product and sum of the bilinear resize
    is exact in fp32, so the resized logits are the same in any evaluation order, FMA or not."""
    return n // 2 if n % 2 == 0 else 2 * n


def synthetic_decoder(points: np.ndarray, crop_hw, seed: int = 0):
    """A seeded stand-in for the SAM decoder: points [P,2] (x, y in crop pixels) -> (low-res logits [P,3,Hl,Wl] fp32,
    iou [P,3] fp32).  Each point's three masks are Gaussian bumps around it with their own radius, steepness and noise,
    a pure function of (seed, point, crop size), so batching does not change them.  Some masks are empty (stability 0 / 0 =
    NaN), some reach the crop or image edge, mask 2 sometimes repeats mask 0 (a duplicate box), and the IoU predictions are
    distinct values in [0.6, 1)."""
    h, w = crop_hw
    Hl, Wl = synthetic_low_res_size(h), synthetic_low_res_size(w)
    ys = (np.arange(Hl) + 0.5) * (h / Hl) - 0.5            # low-res cell centres in crop pixels
    xs = (np.arange(Wl) + 0.5) * (w / Wl) - 0.5
    P = len(points)
    low = np.empty((P, 3, Hl, Wl), dtype=np.float32)
    iou = np.empty((P, 3), dtype=np.float32)
    for p in range(P):
        px, py = float(points[p][0]), float(points[p][1])
        key = repr((seed, round(px, 6), round(py, 6), int(h), int(w))).encode()
        rng = np.random.default_rng(zlib.crc32(key))
        d2 = (ys[:, None] - py) ** 2 + (xs[None, :] - px) ** 2
        for k in range(3):
            r = rng.uniform(1.5, 0.12 * min(h, w)) * (1.0 + 0.7 * k)
            amp = rng.uniform(10.0, 120.0)                  # the edge's steepness: stability rises with it
            noise = rng.uniform(-0.5, 0.5, size=(Hl, Wl))
            v = amp * (np.exp(-d2 / (2 * r * r)) - 0.5) + noise
            if rng.uniform() < 0.08:                          # an empty mask
                v = -np.abs(v) - 2.0
            low[p, k] = np.clip(np.round(v * 64.0) / 64.0, -100.0, 100.0)
        if rng.uniform() < 0.15:
            low[p, 2] = low[p, 0]
        iou[p] = rng.uniform(0.6, 1.0, size=3)
    return torch.from_numpy(low), torch.from_numpy(iou)
