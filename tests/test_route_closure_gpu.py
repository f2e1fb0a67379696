"""Route closure: the es3_* calls real model paths make (tests/es3_recorder.py records them) select only kernel instantiations
that some fp64 table row runs.  Each test hands its recorded calls to routes.assert_closed, which keys every call, requires a key
function for every entry point reached and looks the key up in the tables of the files tests/routes.py lists for its entry point;
the extra assertions pin routes a model is expected to reach.  The last test checks that the GEMM tile rules routes.py restates
from gemm_tc.cu select the instantiations the library launches."""
import json
import os
import re
import subprocess
import sys

import pytest

from es3_recorder import (STUDENTS, TEXT_ROUTES, backbone_calls, eval_forward_calls, image_epoch_calls, module_api_calls,
                          point_segmenter, predictor_calls, segmenter_set_image_calls, teacher_calls, text_epoch_calls, text_step_calls,
                          text_teacher_calls, training_step_calls)
from routes import KEYS, assert_closed, conv3x3_num_kb, gemm_bn, gemm_stages, pick_bn

# What every stage-1 update reaches: the loss backward scaled by the device loss scale, the norm of a 16-byte-aligned arena whose
# length is a multiple of 4 and far below the grid cap, and AdamW clipped at CLIP_GRAD with a dynamic scale and the decay group
# ending inside the arena
STAGE1_UPDATE = {("es3_grad_norm", False, False), ("es3_adamw_flat", True, True, False, True)}

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------------- image students
@pytest.mark.parametrize("step", ["eval", "train", "train frozen BN"])
@pytest.mark.parametrize("name", STUDENTS)
def test_route_closure_student(cuda, monkeypatch, name, step):
    """The eval forward of `name` at 1024^2 (batch 2), or one native training step (1024^2, embed 64, batch 1) with batch-statistics
    or frozen BatchNorm: each is recorded once and checked against the forward, backward and every other covering table.  The eval
    forward of efficientvit_b1 runs both Cin-128 MBConv blocks (its stage-3 blocks and stage-4 opener), that of efficientvit_b0 the
    stride-1 one (its stage-4 blocks)."""
    if step != "eval":
        assert_closed(training_step_calls(cuda, monkeypatch, name, step == "train frozen BN"), f"{name} {step}")
        return
    calls = eval_forward_calls(cuda, monkeypatch, name)
    cin128 = {KEYS[n](a) for n, a in calls if n == "es3_mbconv_bf16" and a[13] == 128}
    expected = {"efficientvit_b1": {("es3_mbconv_bf16", 128, 512, 128, 1), ("es3_mbconv_bf16", 128, 512, 256, 2)},
                "efficientvit_b0": {("es3_mbconv_bf16", 128, 512, 128, 1)}}.get(name)
    if expected is not None:
        assert cin128 == expected, f"{name}: Cin-128 MBConv routes {sorted(cin128)}, expected {sorted(expected)}"
    assert_closed(calls, f"{name} {step}")


# The strict route keys the code says these students reach at 1024^2, spelled as the recorded calls spell them: EfficientViT-B1's
# stage-3 LiteMLA runs at HW 4096 (two chunks) with head dim 16, B2's with head dim 32; RepViT's SqueezeExcite runs fc1 with ReLU and
# fc2 with the sigmoid gate (bias, no scale, no residual) and gates the map; TinyViT's window attention has the relative bias and
# pad_row and is windowed.
STRICT_PINNED = {
    "efficientvit_b1": {("es3_litemla_attn_f32", 16, True), ("es3_litemla_attn_f32", 16, False)},
    "efficientvit_b2": {("es3_litemla_attn_f32", 32, True), ("es3_litemla_attn_f32", 32, False)},
    "repvit_m1_1": {("es3_sgemm_f32", 1, False, False, True, False), ("es3_sgemm_f32", 6, False, False, True, False),
                    ("es3_scale_channels_f32",)},
    "tiny_vit_11m": {("es3_attention_f32", 32, True, True, True)},
}


@pytest.mark.parametrize("name", STUDENTS)
def test_route_closure_student_strict(cuda, monkeypatch, name):
    """The eval forward of `name` at 1024^2 (batch 2) inside ops.strict_precision(): every strict kernel call keyed and covered by
    the strict student kernels' tables (tests/test_strict_kernels_gpu.py) or the ViT file's strict tables."""
    reached = assert_closed(eval_forward_calls(cuda, monkeypatch, name, strict=True), f"{name} strict")
    assert reached and not [k for k in reached if "bf16" in k[0]], f"{name} strict reaches bf16 kernels"
    missing = STRICT_PINNED.get(name, set()) - reached
    assert not missing, f"{name} strict: expected routes not reached: {sorted(missing, key=repr)}"


# ----------------------------------------------------------------------------------------------------------- stage-1 iterations
@pytest.mark.parametrize("name", ["efficientvit_b1", "repvit_m1_1", "tiny_vit_5m"])
def test_route_closure_image_epoch(cuda, monkeypatch, name):
    """stage1.train.train_one_epoch, one student per family: decoded uint8 images of two sizes prepared on the device, the KD loss
    on padded masks with the stored fp16 embeddings, the backward with batch-statistics BatchNorm, two iterations accumulated into
    one FlatAdamW update (dynamic loss scale, clipped)."""
    reached = assert_closed(image_epoch_calls(cuda, monkeypatch, name), f"{name} train_one_epoch")
    pinned = STAGE1_UPDATE | {("es3_prepare_images_u8",), ("es3_kd_loss_fwd", True), ("es3_kd_loss_bwd", True)}
    missing = pinned - reached
    assert not missing, f"{name} train_one_epoch: expected routes not reached: {sorted(missing, key=repr)}"


@pytest.mark.parametrize("backbone", ["MobileCLIP-S0", "MobileCLIP-S1"])
def test_route_closure_text_epoch(cuda, monkeypatch, backbone):
    """stage1.train.train_text_one_epoch: S0 with batch-statistics BatchNorm (the path it takes by default) and S1, masked loss with
    consistency, two iterations accumulated into one FlatAdamW update."""
    reached = assert_closed(text_epoch_calls(cuda, monkeypatch, backbone), f"{backbone} train_text_one_epoch")
    pinned = STAGE1_UPDATE | ({("es3_repmixer_bn_fwd",)} if backbone == "MobileCLIP-S0" else set())
    missing = pinned - reached
    assert not missing, f"{backbone} train_text_one_epoch: expected routes not reached: {sorted(missing, key=repr)}"


# ----------------------------------------------------------------------------------------------------------- text encoders
@pytest.mark.parametrize("route", TEXT_ROUTES, ids=[r[0] for r in TEXT_ROUTES])
def test_route_closure_text(cuda, monkeypatch, route):
    """The native text training steps of es3_recorder.TEXT_ROUTES: S0 with frozen BN, S1, B, S3 at contexts 32, 77 and 128, the
    77-entry table at 32 and at 128, masked and plain loss with consistency, and a batch of 512 x 77 tokens (LayerNorm backward over
    more than 592 x 64 rows)."""
    reached = assert_closed(text_step_calls(cuda, monkeypatch, *route[1:]), route[0])
    if route[1] == "MobileCLIP-S0":
        assert {("es3_repmixer_bf16",), ("es3_repmixer_tm_bwd",)} <= reached
    if route[0] == "B ctx 128":
        assert ("es3_attention_causal_bf16", 2) in reached
    if route[0] == "S3 batch 512":
        assert any(k[0] == "es3_layernorm_bwd_f32" and k[3] for k in reached)


def test_route_closure_sam3_teacher(cuda, monkeypatch):
    """The SAM3 text teacher's eval forward (width 1024, 16 heads, causal)."""
    assert ("es3_attention_causal_bf16", 1) in assert_closed(text_teacher_calls(cuda, monkeypatch), "SAM3 text teacher")


# ----------------------------------------------------------------------------------------------------------- SAM heads
@pytest.mark.parametrize("kind", ["vit", "student"])
def test_route_closure_predictor(cuda, monkeypatch, kind):
    """SAM3InteractiveImagePredictor and Sam3PointPromptSegmenter.predict_batch (object-gated) on the ViT override and the EV-B1
    student: points, box, box + points, point + mask, mask only, 12 points; multimask and return_logits on and off."""
    reached = assert_closed(predictor_calls(point_segmenter(kind, cuda), monkeypatch), f"predictor {kind}")
    assert ("es3_attn_few_keys", True) in reached                        # 12 points + 6 output tokens + the pad point: two tiles
    assert ("es3_hyper_masks", True, 3, 1) in reached and ("es3_bilinear_nchw_f32", False, True) in reached


def test_route_closure_strict(cuda, monkeypatch):
    from efficientsam3_b200 import ops
    seg = point_segmenter("student", cuda)
    with ops.strict_precision():
        reached = assert_closed(predictor_calls(seg, monkeypatch), "predictor strict")
    assert ("es3_attn_few_keys_f32", True) in reached and any(k[0] == "es3_ln_rows_gelu_f32" for k in reached)


def test_route_closure_module_api(cuda, monkeypatch):
    """PromptEncoder / MaskDecoder / TwoWayTransformer as test_decoder_gpu builds them: points, boxes and a mask prompt."""
    assert_closed(module_api_calls(cuda, monkeypatch), "module API")


# ----------------------------------------------------------------------------------------------------------- SAM3 ViT trunk
def test_route_closure_teacher(cuda, monkeypatch):
    """SAM3ImageTeacherEncoder at 1008 px, one windowed and one global block, B = 2: both reach attn_tc_kernel<96>, and the global
    block's QKV projection (N = 3072, K = 1024, bias, bf16 out) takes the RoPE epilogue's 128-wide tile with the 4-stage ring."""
    reached = assert_closed(teacher_calls(cuda, monkeypatch, False), "teacher 1008")
    assert {("es3_attention_bf16", "tc", 96, True), ("es3_attention_bf16", "tc", 96, False)} <= reached
    assert ("es3_gemm_bf16_ex", 128, 4, None, False, True, None, False, "bf16", "global", False) in reached


def test_route_closure_teacher_strict(cuda, monkeypatch):
    reached = assert_closed(teacher_calls(cuda, monkeypatch, True), "teacher 1008 strict")
    assert ("es3_attention_f32", 64, False, False, True) in reached and ("es3_attention_f32", 64, False, False, False) in reached


# The FP8 teacher's routes: QKV to bf16 with windowed and global RoPE, proj and fc2 to fp32 on the fp32 residual stream, fc1 to e4m3
# with GELU, and norm1 / norm2 (C = 1024) to e4m3.
FP8_TEACHER_PINNED = {("es3_gemm_fp8", "bf16", None, False, "window"), ("es3_gemm_fp8", "bf16", None, False, "global"),
                      ("es3_gemm_fp8", "f32", None, True, None), ("es3_gemm_fp8", "e4m3", "gelu", False, None),
                      ("es3_layernorm_f32_e4m3", 8)}


@pytest.mark.parametrize("fp8", ["linear", "attention"])
def test_route_closure_teacher_fp8(cuda, monkeypatch, fp8):
    """The teacher of test_route_closure_teacher with enable_fp8(True, attention=fp8 == "attention"): the four linear layers on
    es3_gemm_fp8; with FP8 attention, L = 576 (24-windows) and L = 5184 (global) both on the 96-key tile."""
    reached = assert_closed(teacher_calls(cuda, monkeypatch, False, fp8=fp8), f"teacher 1008 fp8 {fp8}")
    pinned = set(FP8_TEACHER_PINNED)
    if fp8 == "attention":
        pinned |= {("es3_attention_fp8", 96, True), ("es3_attention_fp8", 96, False)}
    missing = pinned - reached
    assert not missing, f"fp8 {fp8}: expected routes not reached: {sorted(missing, key=repr)}"
    assert (fp8 == "attention") == any(k[0] == "es3_attention_fp8" for k in reached)


@pytest.mark.parametrize("which", ["336", "vit_small_112"])
def test_route_closure_backbone(cuda, monkeypatch, which):
    """create_sam3_vit_backbone with tests/test_vit_gpu.py's 336 configuration and the vit_small_112 fixture's."""
    assert_closed(backbone_calls(cuda, monkeypatch, which), f"ViT backbone {which}")


def test_route_closure_segmenter(cuda, monkeypatch):
    """Sam3PointPromptSegmenter (one windowed block) through the interactive predictor's set_image."""
    reached = assert_closed(segmenter_set_image_calls(cuda, monkeypatch), "segmenter set_image")
    assert ("es3_attention_bf16", "tc", 96, True) in reached


# ----------------------------------------------------------------------------------------------------------- the restated tile rules
# One call per gemm_tc_kernel<BN, STAGES, ACT> instantiation an entry point can launch, each through a different branch of pick_bn,
# the RoPE override or the stage rule where one exists.  gemm: (N, K, act, bn_hint, rope); conv3x3: (W, C, N, act, bn_hint);
# convt2x2: (Cin, Cout, act).
GEMM_PICKS = [(384, 128, None, 0, False), (192, 1024, None, 0, True), (64, 64, "relu", 256, False), (1056, 512, "relu", 0, False),
              (400, 64, "hswish", 0, False), (160, 512, "hswish", 0, False), (64, 128, "gelu", 128, False),
              (4736, 1024, "gelu", 0, False), (96, 256, None, 0, False), (192, 512, "relu", 0, False), (32, 64, "hswish", 64, False),
              (512, 256, "gelu", 0, False), (96, 512, None, 0, False), (48, 64, "relu", 0, False), (256, 1024, "hswish", 32, False),
              (40, 200, "gelu", 0, False)]
CONV_PICKS = [(16, 64, 256, None, 0), (23, 32, 160, "relu", 0), (48, 8, 64, "hswish", 128), (32, 96, 1024, "gelu", 0),
              (64, 64, 192, None, 0), (16, 256, 64, "relu", 0), (8, 32, 256, "hswish", 64), (36, 64, 320, "gelu", 0),
              (32, 16, 96, None, 0), (24, 64, 32, "relu", 0), (16, 128, 128, "hswish", 32), (40, 8, 32, "gelu", 0)]
CONVT_PICKS = [(64, 32, None), (256, 64, None), (128, 64, "relu"), (192, 32, "relu"), (32, 256, "hswish"), (1024, 512, "hswish"),
               (128, 32, "gelu"), (512, 256, "gelu")]

_PICK_SCRIPT = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
from efficientsam3_b200 import ops
ops.PW_SMALL = False
dev = torch.device("cuda:0")
kind, rows = sys.argv[2], json.loads(sys.argv[3])
bf = lambda *s: torch.zeros(*s, device=dev, dtype=torch.bfloat16)
for r in rows:
    if kind == "gemm":
        N, K, act, bn, rope = r
        tab = torch.zeros(16, 32, 2, device=dev)
        ops.gemm(bf(32, K), bf(N, K), act=act, bn_hint=bn, rope=(tab, 128, 4, 4, 0) if rope else None)
    elif kind == "conv3x3":
        W, C, N, act, bn = r
        ops.conv3x3(bf(1, 5, W, C), bf(N, 9 * C), act=act, bn_hint=bn)
    else:
        Cin, Cout, act = r
        ops.convt2x2(bf(1, 3, 5, Cin), bf(4 * Cout, Cin), act=act)
    torch.cuda.synchronize()
"""


def _expected_picks(kind):
    from efficientsam3_b200.ops import ACT
    if kind == "gemm":
        rows = GEMM_PICKS
        bns = [(gemm_bn(N, K, act, "global" if rope else None, bn), -(-K // 64), act) for N, K, act, bn, rope in rows]
    elif kind == "conv3x3":
        rows = CONV_PICKS
        bns = [(pick_bn(N, bn), conv3x3_num_kb(C), act) for W, C, N, act, bn in rows]
    else:
        rows = CONVT_PICKS
        bns = [(pick_bn(4 * Cout, 0), -(-Cin // 64), act) for Cin, Cout, act in rows]
    return rows, [(bn, gemm_stages(bn, kb), ACT[act]) for bn, kb, act in bns]


@pytest.mark.parametrize("kind", ["gemm", "conv3x3", "convt2x2"])
def test_restated_tile_rules_match_the_launches(cuda, kind):
    """tests/routes.py restates pick_bn, the RoPE override, the stage rule and the conv geometry of gemm_tc.cu.  A fresh process with
    ES3_DEBUG_OCCUPANCY=1 runs one call per expected instantiation; gemm_tc.cu reports each instantiation's template arguments on
    its first launch, so the reported lines must be the expected (BN, STAGES, ACT) list, in call order."""
    rows, want = _expected_picks(kind)
    assert len(set(want)) == len(want), f"{kind}: two calls expect the same instantiation"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, ES3_DEBUG_OCCUPANCY="1")
    p = subprocess.run([sys.executable, "-c", _PICK_SCRIPT, root, kind, json.dumps(rows)], env=env, cwd=root, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, f"{kind}: the launch process exited with {p.returncode}:\n{p.stderr[-4000:]}"
    got = [tuple(int(v) for v in m) for m in re.findall(r"gemm_tc_kernel<BN=(\d+),STAGES=(\d+),ACT=(\d+),CPR=\d+>", p.stderr)]
    assert got == want, f"{kind}: launched {got}, the restated rules expect {want}"
