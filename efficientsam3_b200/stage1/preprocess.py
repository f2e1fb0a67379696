"""Stage-1 image preparation on the device, from decoded uint8 images.

The reference builds every stage-1 input on the CPU inside SA1BDataset.__getitem__ (stage1/data/sa1b_dataset.py:163-170, 216-227):
ResizeLongestSide.apply_image_torch (transforms.py:48-54) -- F.interpolate(bilinear, align_corners=False, antialias=True) of the fp32
0..255 image, longest side to IMG_SIZE -- then (x - DATA.MEAN) / DATA.STD and zero padding bottom and right to IMG_SIZE x IMG_SIZE.
`prepare_images` does the same for a whole ragged batch in two native launches (es3_prepare_images_u8), so the loader only decodes.

`pack_images` lays a batch out as one flat uint8 tensor plus its sizes; used as (part of) a DataLoader `collate_fn`, the
`pin_memory=True` loader pins it and one host-to-device copy moves the batch.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from .. import ops

MEAN = (123.675, 116.28, 103.53)   # DATA.MEAN (stage1/config.py:19)
STD = (58.395, 57.12, 57.375)      # DATA.STD (stage1/config.py:20)


def get_preprocess_shape(h: int, w: int, S: int) -> tuple[int, int]:
    """ResizeLongestSide.get_preprocess_shape (transforms.py:79-85): (h', w') with the longest side scaled to S, int(x + 0.5)."""
    scale = S * 1.0 / max(h, w)
    return int(h * scale + 0.5), int(w * scale + 0.5)


@dataclass
class PackedImages:
    """A batch of HWC uint8 RGB images back to back in `data` (flat uint8), image b of `sizes[b] = (h, w)` (int64 [B,2], CPU)."""
    data: torch.Tensor
    sizes: torch.Tensor

    def pin_memory(self):
        """Called by a `pin_memory=True` DataLoader on each collated batch."""
        return PackedImages(self.data.pin_memory(), self.sizes)

    def __len__(self):
        return self.sizes.shape[0]

    def table(self) -> torch.Tensor:
        """int64 [B,3] CPU rows (byte offset, h, w), the layout es3_prepare_images_u8 reads."""
        n = self.sizes[:, 0] * self.sizes[:, 1] * 3
        off = torch.cumsum(n, 0) - n
        return torch.cat([off[:, None], self.sizes], 1).contiguous()


def _check_image(img, i):
    if not torch.is_tensor(img):
        raise TypeError(f"image {i}: expected a torch.Tensor, got {type(img).__name__}")
    if img.dtype != torch.uint8:
        raise ops._lib.Es3Error(f"image {i}: expected uint8, got {img.dtype}")
    if img.dim() != 3 or img.shape[2] != 3:
        raise ops._lib.Es3Error(f"image {i}: expected HWC with 3 channels, got shape {tuple(img.shape)}")
    if img.shape[0] < 1 or img.shape[1] < 1:
        raise ops._lib.Es3Error(f"image {i}: empty image of shape {tuple(img.shape)}")
    if not img.is_contiguous():
        raise ops._lib.Es3Error(f"image {i}: expected a contiguous HWC tensor (strides {img.stride()})")


def pack_images(images) -> PackedImages:
    """Decoded HWC uint8 RGB images (any sizes, one device) -> PackedImages, `data` on that device."""
    images = list(images)
    if not images:
        raise ops._lib.Es3Error("pack_images: no images")
    for i, img in enumerate(images):
        _check_image(img, i)
    sizes = torch.tensor([[img.shape[0], img.shape[1]] for img in images], dtype=torch.int64)
    return PackedImages(torch.cat([img.reshape(-1) for img in images]), sizes)


def is_uint8_batch(samples) -> bool:
    """True for the batches prepare_images takes: PackedImages, or a list / tuple of uint8 image tensors."""
    if isinstance(samples, PackedImages):
        return True
    return isinstance(samples, (list, tuple)) and len(samples) > 0 and torch.is_tensor(samples[0]) and samples[0].dtype == torch.uint8


def prepare_images(images_or_packed, img_size: int, mean=MEAN, std=STD, device=None, out=None):
    """SA1BDataset's image preparation on the device for a batch of decoded HWC uint8 RGB images (a list, or PackedImages).
    Returns (x fp32 [B,3,S,S] CUDA, img_size_before_pad int64 [B,3] CPU rows (3, h', w')), S = img_size.
    Every check runs on the host before anything is copied or launched."""
    packed = images_or_packed if isinstance(images_or_packed, PackedImages) else pack_images(images_or_packed)
    table = packed.table()
    if packed.data.dtype != torch.uint8 or packed.data.dim() != 1:
        raise ops._lib.Es3Error(f"prepare_images: PackedImages.data must be flat uint8, got {packed.data.dtype} {tuple(packed.data.shape)}")
    ops.image_table_ws_floats(table, packed.data.numel(), img_size)
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    src = packed.data.to(device, non_blocking=True)
    x = ops.prepare_images_u8(src, table, img_size, mean, std, out=out)
    hw = torch.tensor([get_preprocess_shape(int(h), int(w), img_size) for h, w in packed.sizes.tolist()], dtype=torch.int64)
    return x, torch.cat([torch.full((hw.shape[0], 1), 3, dtype=torch.int64), hw], 1)
