"""Tile-boundary geometry of the wgmma MBConv kernels (mbconv_tc, mbconv_tc_s2), all five instantiations, against the same
op-by-op fp32 statement as test_ops_gpu.py::test_mbconv_fused.

The kernels decide which expand rows lie inside the image once per tile, and send the padding rows of the expand's last
64-row block to a scratch row of the pixel-major tile.  These cases put that bookkeeping under load: images smaller than one
tile, H and W of 1 mod the tile (a one-pixel edge tile in each direction), and batches large enough that every persistent
CTA runs several tiles from different images, with partial edge tiles among them.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (Cin, Mid, Cout, stride); output tiles are 8 x 16 (stride 1) and 4 x 16 (stride 2)
BLOCKS = [(32, 128, 32, 1), (64, 256, 64, 1), (16, 64, 32, 2), (32, 128, 64, 2), (64, 256, 128, 2)]

# (B, H, W) per stride
GEOMETRY = {
    1: [(2, 3, 5), (2, 1, 37), (2, 1, 1), (2, 17, 33), (2, 9, 17), (24, 37, 37)],
    2: [(2, 3, 5), (2, 1, 37), (2, 1, 1), (2, 17, 33), (2, 18, 34), (40, 37, 37)],
}

CASES = [(*blk, *geo) for blk in BLOCKS for geo in GEOMETRY[blk[3]]]


@pytest.mark.parametrize("cin,mid,cout,stride,B,H,W", CASES)
def test_mbconv_tc_tile_geometry(cuda, cin, mid, cout, stride, B, H, W):
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(cin + mid + 7 * H + W + B)
    bf = lambda t: t.to(torch.bfloat16).to(cuda)
    x = bf(torch.randn(B, H, W, cin, generator=g))
    w1 = bf(torch.randn(mid, cin, generator=g) / math.sqrt(cin))
    s1 = (torch.rand(mid, generator=g) + 0.5).to(cuda); b1 = (torch.randn(mid, generator=g) * 0.2).to(cuda)
    wdw = (torch.randn(mid, 1, 3, 3, generator=g) / 3).to(cuda); b2 = (torch.randn(mid, generator=g) * 0.2).to(cuda)
    w3 = bf(torch.randn(cout, mid, generator=g) / math.sqrt(mid))
    s3 = (torch.rand(cout, generator=g) + 0.5).to(cuda); b3 = (torch.randn(cout, generator=g) * 0.2).to(cuda)
    res = stride == 1
    y = ops.mbconv_fused(x, w1, s1, b1, wdw.reshape(mid, 9).t().contiguous(), b2, w3, s3, b3, stride, res, "hswish", impl="tc")
    assert y is not None
    xn = x.float().permute(0, 3, 1, 2)
    e = F.hardswish(F.conv2d(xn, w1.float()[:, :, None, None]) * s1.view(1, -1, 1, 1) + b1.view(1, -1, 1, 1))
    e = e.to(torch.bfloat16).float()
    d = F.hardswish(F.conv2d(e, wdw, b2, stride=stride, padding=1, groups=mid)).to(torch.bfloat16).float()
    ref = F.conv2d(d, w3.float()[:, :, None, None]) * s3.view(1, -1, 1, 1) + b3.view(1, -1, 1, 1)
    if res:
        ref = ref + xn
    ref = ref.permute(0, 2, 3, 1)
    assert y.shape == ref.shape
    scale = ref.abs().max().item() + 1e-12
    # per image, so that a tile written for the wrong image (or not at all) cannot hide behind another image's scale
    for i in range(B):
        err = (y[i].float() - ref[i]).abs().max().item() / scale
        assert err <= 1e-2, f"image {i}: max err / scale = {err:.3e}"
