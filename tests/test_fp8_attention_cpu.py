"""The FP8 attention without a GPU: its power-of-two quantisation rule (tests/emu_fp8_attention.py, the definition the kernel's codes
are held to), the ViT switch, the host-side validation of ops.attention_fp8, and the kernel's register budget."""
from __future__ import annotations

import re
import shutil
import subprocess

import pytest
import torch

from emu_fp8 import E4M3
from emu_fp8_attention import dequantized, key_tile, merge_out, pow2_exponent, pow2_scale, quantize_blocks, split_qkv


# ---------------------------------------------------------------------------------------------- the quantisation definition
def test_pow2_scale_rule():
    amax = torch.tensor([448.0, 449.0, 1.0, 0.0, 2.0 ** -140, 896.0, 897.0, 3e38, 447.99])
    assert pow2_exponent(amax).tolist() == [0, 1, -8, 0, -126, 1, 2, 120, 0]
    s = pow2_scale(amax)
    assert (amax / s <= 448).all() and ((amax / s > 224) | (amax == 0) | (amax < 1e-30)).all()
    assert s[3].item() == 1.0                              # the all-zero block


def test_round_trip_and_saturation_free():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(300, 64, generator=g) * torch.exp2(torch.randint(-8, 9, (300, 1), generator=g).float())
    x = x.to(torch.bfloat16).float()
    q, s = quantize_blocks(x, -1)
    assert q.dtype == E4M3 and s.shape == (300, 1)
    codes = q.float()
    assert codes.abs().max() <= 448 and (codes.abs().amax(-1) >= 224).all()   # every block's amax lands in [224, 448]: no clipping
    err = (codes * s - x).abs()
    assert (err <= x.abs() * 2.0 ** -4 + s * 2.0 ** -10).all()
    # every scale is a power of two, so the dequantised values need no rounding
    assert torch.equal(torch.frexp(s)[0], torch.full_like(s, 0.5))


def test_zero_block_and_subnormal_codes():
    x = torch.zeros(3, 64)
    x[1, 5] = 300.0                                        # s = 1: 300 rounds to 288
    x[1, 6] = 300.0 * 2.0 ** -16                           # below e4m3's smallest normal (2^-6): a subnormal code
    x[2, :] = 2.0 ** -134                                  # below the clamp: s = 2^-126, values 2^-8 -> subnormal code 0x02
    q, s = quantize_blocks(x, -1)
    u = q.view(torch.uint8)
    assert s[0].item() == 1.0 and (u[0] == 0).all()
    assert s[1].item() == 1.0 and q[1, 5].float().item() == 288.0
    assert 0 < u[1, 6].item() < 0x08
    assert s[2].item() == 2.0 ** -126 and (u[2] == 0x02).all()


def test_token_order_and_tiles():
    B, H, W, C, win = 2, 6, 4, 128, 2
    qkv = torch.arange(B * H * W * 3 * C, dtype=torch.float32).reshape(B * H * W, 3 * C)
    q, k, v = split_qkv(qkv, B, H, W, C, win)
    assert q.shape == (B, 6, 2, 4, 64)
    # window (1, 1) of image 1, token (1, 0) inside it = image row 3, column 2; head 1 starts at column 64
    assert q[1, 3, 1, 2, 0].item() == qkv[1 * H * W + 3 * W + 2, 64].item()
    assert v[0, 0, 0, 3, 0].item() == qkv[W + 1, 2 * C].item()
    assert torch.equal(merge_out(q, B, H, W, C, win), qkv[:, :C])
    assert torch.equal(merge_out(split_qkv(qkv, B, H, W, C, 0)[1], B, H, W, C, 0), qkv[:, C:2 * C])
    assert key_tile(576) == 96 and key_tile(5184) == 96 and key_tile(1600) == 128 and key_tile(64) == 128


def test_v_blocks_are_per_key_tile_and_channel():
    B, H, W, C = 1, 24, 24, 64
    g = torch.Generator().manual_seed(1)
    qkv = torch.randn(B * H * W, 3 * C, generator=g)
    qkv[5, 2 * C + 7] = 1024.0                             # key 5 (tile 0), channel 7: only that (tile, channel) block scales
    _, _, vd = dequantized(qkv, B, H, W, C, 0)
    v = qkv[:, 2 * C:].double()
    assert vd[0, 0, 0, 5, 7].item() == 1024.0
    assert (vd[0, 0, 0, 128:, 7] - v[128:, 7]).abs().max() < 2.0 ** -4 * 4    # other tiles of channel 7 keep their own scale
    assert ((vd[0, 0, 0, :96, 7] - v[:96, 7]).abs() <= 2.0).all()              # tile 0 (96 keys), channel 7: s = 4


# ---------------------------------------------------------------------------------------------- switch and host validation
def _small_vit():
    from efficientsam3_b200.model.vitdet import create_sam3_vit_backbone
    return create_sam3_vit_backbone(img_size=336, depth=1, global_att_blocks=(), embed_dim=256, num_heads=4)


def test_switch_semantics():
    from efficientsam3_b200.stage1.model import SAM3ImageTeacherEncoder
    vit = _small_vit()
    assert vit._fp8 is False and vit._fp8_attn is False
    assert vit.enable_fp8(attention=True) is vit and vit._fp8 and vit._fp8_attn
    vit._plan_key = ("cached",)
    vit.enable_fp8()
    assert vit._fp8 and not vit._fp8_attn and vit._plan_key is None
    vit._plan_key = ("cached",)
    vit.enable_fp8(True, attention=True)
    assert vit._plan_key is None
    with pytest.raises(ValueError):
        vit.enable_fp8(False, attention=True)
    assert vit._fp8 and vit._fp8_attn                      # a refused call changes nothing
    vit.enable_fp8(False)
    assert not vit._fp8 and not vit._fp8_attn
    t = SAM3ImageTeacherEncoder(embed_size=24, vit_overrides=dict(img_size=336, depth=1, global_att_blocks=()))
    trunk = t.sam3.backbone.vision_backbone.trunk
    assert t.enable_fp8(attention=True) is t and trunk._fp8 and trunk._fp8_attn
    t.enable_fp8()
    assert trunk._fp8 and not trunk._fp8_attn
    with pytest.raises(ValueError):
        t.enable_fp8(False, attention=True)
    t.enable_fp8(attention=True)
    with pytest.raises(ValueError):                        # still no CPU path with the switch on
        trunk.forward_tokens(torch.zeros(1, 3, 336, 336))


def _bad_calls():
    from efficientsam3_b200 import ops
    bf = torch.bfloat16
    good = dict(B=1, H=24, W=24, C=128, num_heads=2, win=0, scale=0.125)
    qkv = torch.zeros(576, 384, dtype=bf)

    def call(x=qkv, **kw):
        return lambda: ops.attention_fp8(x, **dict(good, **kw))
    return {
        "fp32 qkv": call(qkv.float()),
        "fp16 qkv": call(qkv.half()),
        "e4m3 qkv": call(qkv.float().to(E4M3)),
        "non-contiguous": call(torch.zeros(576, 400, dtype=bf)[:, :384]),
        "transposed": call(torch.zeros(384, 576, dtype=bf).t()),
        "head_dim 32": call(num_heads=4),
        "head_dim 128": call(num_heads=1),
        "window does not divide H": call(win=7),
        "window does not divide W": call(torch.zeros(24 * 30, 384, dtype=bf), W=30, win=12),
        "shape mismatch": call(torch.zeros(575, 384, dtype=bf)),
        "negative window": call(win=-1),
        "zero scale": call(scale=0.0),
        "negative scale": call(scale=-0.125),
        "nan scale": call(scale=float("nan")),
    }


@pytest.mark.parametrize("case", list(_bad_calls()))
def test_wrapper_rejects_before_launch(case):
    from efficientsam3_b200 import ops
    n0 = ops.launch_count
    with pytest.raises(ValueError):
        _bad_calls()[case]()
    assert ops.launch_count == n0


def test_valid_call_on_cpu_raises_no_fallback():
    from efficientsam3_b200 import ops
    from efficientsam3_b200._lib import Es3Error
    n0 = ops.launch_count
    with pytest.raises(Es3Error):
        ops.attention_fp8(torch.zeros(576, 384, dtype=torch.bfloat16), 1, 24, 24, 128, 2, 24, 0.125)
    assert ops.launch_count == n0


# ---------------------------------------------------------------------------------------------- register budget
def test_fp8_attention_compiles_without_spills_or_serialised_wgmma(tmp_path):
    """-Xptxas -v of attention_fp8.cu for sm_90a: neither key-tile instantiation (BN = 96, 128) spills or keeps a stack frame,
    and ptxas does not serialise its wgmma."""
    from efficientsam3_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        nvcc = None
    if nvcc is None or not shutil.which(nvcc):
        pytest.skip("nvcc not available")
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "attention_fp8.cu"), "-o", str(tmp_path / "a.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    text = r.stdout + r.stderr
    rows, name = [], None
    for line in text.splitlines():
        m = re.search(r"Function properties for (\w+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name is not None:
            rows.append((name, *map(int, m.groups())))
            name = None
    attn = [r for r in rows if "attn_fp8_kernel" in r[0]]
    assert len(attn) == 2, rows
    bad = [r for r in rows if r[1] or r[2] or r[3]]
    assert not bad, f"(kernel, stack, spill stores, spill loads) = {bad}"
    assert "wgmma.mma_async instructions are serialized" not in text
    assert "C7512" not in text and "C7510" not in text
