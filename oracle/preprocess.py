"""Oracle: stage-1 image preparation (TEST INFRASTRUCTURE ONLY).
Restates what SA1BDataset.__getitem__ does to a decoded image (stage1/data/sa1b_dataset.py:68-69, 163-170, 216-227):
ResizeLongestSide.apply_image_torch (stage1/data/transforms.py:48-54, get_preprocess_shape :79-85) on the fp32 image,
img_size_before_pad = the resized shape, then norm ((x - mean) / std, :216-219) and pad (zeros bottom / right to S x S, :221-227).
The mean / std defaults are DATA.MEAN / DATA.STD (stage1/config.py:19-20)."""
import torch
import torch.nn.functional as F

MEAN = (123.675, 116.28, 103.53)
STD = (58.395, 57.12, 57.375)


def get_preprocess_shape(oldh, oldw, long_side_length):
    scale = long_side_length * 1.0 / max(oldh, oldw)
    newh, neww = oldh * scale, oldw * scale
    return int(newh + 0.5), int(neww + 0.5)


def prepare_image(img_hwc_u8, img_size, mean=MEAN, std=STD):
    """HWC uint8 RGB -> ([3, S, S] fp32, (3, h', w'))."""
    x = img_hwc_u8.permute(2, 0, 1)[None].float()
    h, w = get_preprocess_shape(x.shape[2], x.shape[3], img_size)
    x = F.interpolate(x, (h, w), mode="bilinear", align_corners=False, antialias=True).squeeze(0)
    size = tuple(x.shape)
    x = (x - torch.tensor(mean).view(-1, 1, 1)) / torch.tensor(std).view(-1, 1, 1)
    x = F.pad(x, (0, img_size - w, 0, img_size - h))
    return x, size
