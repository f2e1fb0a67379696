"""The FP8 teacher linears without a GPU: the block-scaled e4m3 quantisation rule (tests/emu_fp8.py, the definition the kernels are
held to bit for bit), the ViT switch and the host-side validation of the ops wrappers, and the FP8 GEMM's register budget."""
from __future__ import annotations

import re
import shutil
import subprocess

import pytest
import torch

from emu_fp8 import E4M3, block_scale, dequant_rows, dequant_weight, e4m3_rn_satfinite, quantize_rows, quantize_weight


def _codes(x):
    return e4m3_rn_satfinite(torch.tensor(x, dtype=torch.float32)).view(torch.uint8).tolist()


# ---------------------------------------------------------------------------------------------- the quantisation definition
def test_e4m3_rounding_and_saturation():
    # 448 is the largest finite e4m3 (0x7E); anything above saturates instead of becoming NaN (0x7F)
    assert _codes([448.0, 500.0, 1e30, -1e30]) == [0x7E, 0x7E, 0x7E, 0xFE]
    # round to nearest even: 1 + 2^-4 lies halfway between 1 (0x38) and 1.125 (0x39)
    assert _codes([1.0625, 1.0625 + 2 ** -20, 1.1875]) == [0x38, 0x39, 0x3A]
    # subnormals: 2^-9 is the smallest (0x01); half of it rounds to even (0), three quarters up
    assert _codes([2.0 ** -9, 2.0 ** -10, 0.75 * 2.0 ** -9, 7 * 2.0 ** -9]) == [0x01, 0x00, 0x01, 0x07]
    assert _codes([2.0 ** -6]) == [0x08]                   # the smallest normal


def test_scale_rule():
    assert block_scale(torch.tensor([0.0]))[0].item() == 1.0
    amax = torch.tensor([448.0, 1.0, 3e-30, 7.0])
    assert torch.equal(block_scale(amax), amax / 448.0)
    x = torch.zeros(2, 256)
    x[0, 3], x[0, 200], x[1, 130] = -5.0, 2.0, 0.25
    q, s = quantize_rows(x)
    assert s.tolist() == [[torch.tensor(5.0 / 448).item(), torch.tensor(2.0 / 448).item()], [1.0, torch.tensor(0.25 / 448).item()]]
    assert q.view(torch.uint8)[0, 3].item() == 0xFE and q.view(torch.uint8)[0, 200].item() == 0x7E   # each block's amax -> +-448
    assert (q.view(torch.uint8)[1, :128] == 0).all()         # the all-zero block: scale 1, codes 0


def test_block_layouts_round_trip():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 384, generator=g) * torch.tensor([1.0, 100.0, 1e-3]).repeat_interleave(128)
    q, s = quantize_rows(x)
    assert q.dtype == E4M3 and s.shape == (5, 3)
    assert ((dequant_rows(q, s) - x).abs() <= x.abs() * 2 ** -4 + s.repeat_interleave(128, 1) * 2 ** -10).all()
    w = torch.randn(200, 256, generator=g)
    qw, sw = quantize_weight(w)
    assert qw.shape == (200, 256) and sw.shape == (2, 2)
    assert sw[1, 0].item() == (w[128:, :128].abs().amax() / 448.0).item()      # the ragged row block's amax: rows < N only
    assert ((dequant_weight(qw, sw) - w).abs() <= w.abs() * 2 ** -4 + sw.repeat_interleave(128, 0)[:200].repeat_interleave(128, 1) * 2 ** -10).all()


# ---------------------------------------------------------------------------------------------- switch and host validation
def _small_vit():
    from efficientsam3_b200.model.vitdet import create_sam3_vit_backbone
    return create_sam3_vit_backbone(img_size=336, depth=1, global_att_blocks=(), embed_dim=256, num_heads=4)


def test_switch_is_opt_in_and_forwards():
    from efficientsam3_b200.stage1.model import SAM3ImageTeacherEncoder
    vit = _small_vit()
    assert vit._fp8 is False
    assert vit.enable_fp8() is vit and vit._fp8 is True
    assert vit.enable_fp8(False)._fp8 is False
    t = SAM3ImageTeacherEncoder(embed_size=24, vit_overrides=dict(img_size=336, depth=1, global_att_blocks=()))
    assert t.enable_fp8() is t and t.sam3.backbone.vision_backbone.trunk._fp8 is True
    with pytest.raises(ValueError):                    # still no CPU path with the switch on
        t.sam3.backbone.vision_backbone.trunk.forward_tokens(torch.zeros(1, 3, 336, 336))


def test_switch_invalidates_the_plan():
    vit = _small_vit()
    vit._plan_key = ("cached",)
    vit.enable_fp8()
    assert vit._plan_key is None


def _bad_calls():
    from efficientsam3_b200 import ops
    bf, f32 = torch.bfloat16, torch.float32
    a, sa = torch.zeros(64, 256, dtype=E4M3), torch.ones(64, 2)
    w, sw = torch.zeros(128, 256, dtype=E4M3), torch.ones(1, 2)
    return {
        "K % 128": lambda: ops.gemm_fp8(torch.zeros(64, 200, dtype=E4M3), torch.ones(64, 2), torch.zeros(128, 200, dtype=E4M3), sw),
        "N % 128": lambda: ops.gemm_fp8(a, sa, torch.zeros(96, 256, dtype=E4M3), sw),
        "K mismatch": lambda: ops.gemm_fp8(a, sa, torch.zeros(128, 384, dtype=E4M3), torch.ones(1, 3)),
        "lda misaligned": lambda: ops.gemm_fp8(torch.zeros(64, 264, dtype=E4M3)[:, :256], sa, w, sw),
        "A column stride": lambda: ops.gemm_fp8(torch.zeros(256, 64, dtype=E4M3).t(), sa, w, sw),
        "A dtype": lambda: ops.gemm_fp8(a.view(torch.uint8), sa, w, sw),
        "sa shape": lambda: ops.gemm_fp8(a, torch.ones(64, 1), w, sw),
        "sa dtype": lambda: ops.gemm_fp8(a, sa.to(bf), w, sw),
        "sw shape": lambda: ops.gemm_fp8(a, sa, w, torch.ones(2, 2)),
        "sa strided": lambda: ops.gemm_fp8(a, torch.ones(64, 4)[:, :2], w, sw),
        "bias shape": lambda: ops.gemm_fp8(a, sa, w, sw, torch.zeros(64)),
        "bias dtype": lambda: ops.gemm_fp8(a, sa, w, sw, torch.zeros(128, dtype=bf)),
        "e4m3 out without gelu": lambda: ops.gemm_fp8(a, sa, w, sw, out_dtype=E4M3),
        "bf16 out with gelu": lambda: ops.gemm_fp8(a, sa, w, sw, act="gelu"),
        "relu": lambda: ops.gemm_fp8(a, sa, w, sw, act="relu", out_dtype=f32),
        "fp16 out": lambda: ops.gemm_fp8(a, sa, w, sw, out_dtype=torch.float16),
        "residual with bf16 out": lambda: ops.gemm_fp8(a, sa, w, sw, residual=torch.zeros(64, 128)),
        "residual shape": lambda: ops.gemm_fp8(a, sa, w, sw, residual=torch.zeros(64, 64), out_dtype=f32),
        "residual dtype": lambda: ops.gemm_fp8(a, sa, w, sw, residual=torch.zeros(64, 128, dtype=bf), out_dtype=f32),
        "rope with fp32 out": lambda: ops.gemm_fp8(a, sa, w, sw, rope=(torch.zeros(64, 32, 2), 128, 8, 8, 0), out_dtype=f32),
        "rope table shape": lambda: ops.gemm_fp8(a, sa, w, sw, rope=(torch.zeros(63, 32, 2), 128, 8, 8, 0)),
        "rope cols": lambda: ops.gemm_fp8(a, sa, w, sw, rope=(torch.zeros(64, 32, 2), 64, 8, 8, 0)),
        "quantize C % 128": lambda: ops.quantize_e4m3(torch.zeros(4, 200, dtype=bf)),
        "quantize dtype": lambda: ops.quantize_e4m3(torch.zeros(4, 256, dtype=f32)),
        "quantize row stride": lambda: ops.quantize_e4m3(torch.zeros(4, 258, dtype=bf)[:, :256]),
        "layernorm C": lambda: ops.layernorm_e4m3(torch.zeros(4, 512), torch.ones(512), torch.zeros(512)),
        "layernorm gamma": lambda: ops.layernorm_e4m3(torch.zeros(4, 1024), torch.ones(512), torch.zeros(1024)),
        "layernorm dtype": lambda: ops.layernorm_e4m3(torch.zeros(4, 1024, dtype=bf), torch.ones(1024), torch.zeros(1024)),
        "pack K % 128": lambda: ops.pack_weight_e4m3(torch.zeros(128, 200)),
        "pack dtype": lambda: ops.pack_weight_e4m3(torch.zeros(128, 256, dtype=torch.float16)),
    }


@pytest.mark.parametrize("case", list(_bad_calls()))
def test_wrappers_reject_bad_shapes_before_launch(case):
    from efficientsam3_b200 import ops
    n0 = ops.launch_count
    with pytest.raises(ValueError):
        _bad_calls()[case]()
    assert ops.launch_count == n0


def test_valid_shapes_on_cpu_raise_no_fallback():
    from efficientsam3_b200 import ops
    from efficientsam3_b200._lib import Es3Error
    a, w = torch.zeros(64, 256, dtype=E4M3), torch.zeros(128, 256, dtype=E4M3)
    with pytest.raises(Es3Error):
        ops.gemm_fp8(a, torch.ones(64, 2), w, torch.ones(1, 2), torch.zeros(128))
    with pytest.raises(Es3Error):
        ops.quantize_e4m3(torch.zeros(4, 256, dtype=torch.bfloat16))


# ---------------------------------------------------------------------------------------------- register budget
def test_fp8_gemm_compiles_without_spills_or_serialised_wgmma(tmp_path):
    """-Xptxas -v of gemm_fp8.cu for sm_90a: no instantiation of the FP8 GEMM spills or keeps a stack frame (the main and the
    per-block partial accumulators are 128 fp32 registers a thread), and ptxas does not serialise its wgmma."""
    from efficientsam3_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        nvcc = None
    if nvcc is None or not shutil.which(nvcc):
        pytest.skip("nvcc not available")
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "gemm_fp8.cu"), "-o", str(tmp_path / "gemm_fp8.o")]
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
    gemm = [r for r in rows if "gemm_fp8_kernel" in r[0]]
    assert len(gemm) == 4, rows                             # bf16 / fp32 / fp32+GELU / e4m3+GELU epilogues
    bad = [r for r in rows if r[1] or r[2] or r[3]]
    assert not bad, f"(kernel, stack, spill stores, spill loads) = {bad}"
    assert "wgmma.mma_async instructions are serialized" not in text
