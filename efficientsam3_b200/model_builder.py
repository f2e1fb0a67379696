"""EfficientSAM3 image encoder = student trunk + projection head + SAM3 FPN neck, H100-native.  Mirrors the module tree
(attribute names -> state_dict keys) the reference builds in `_create_student_vision_backbone`
(sam3/sam3/model_builder.py:789-941):

    Sam3DualViTDetNeck( trunk = ListWrapper( ImageStudentEncoder( <Family>TrunkWrapper(backbone), 1024 ch, 72 x 72 ) ) )

    keys:  trunk.model.backbone.model.*   the student backbone      (same module classes as stage 1)
           trunk.model.head.{0,1,3}.*     the 1024-channel projection head (model_builder.py:764-787)
           convs.* / sam2_convs.*         the SimpleFPN branches (necks.py:13-125)

so a merged EfficientSAM3 checkpoint (`detector.backbone.vision_backbone.` + these keys, model_builder.py:584-630) loads
unchanged.  Everything runs on the kernels the stage-1 student and the FPN already use; this file is composition only.
`build_efficientsam3_point_segmenter` puts the SAM heads on top (the SAM-1-task use of EfficientSAM3,
efficientsam3_examples/efficientsam3_for_sam1_task_example.py:161-198).  Out of scope: the detector / text side of
`build_efficientsam3_image_model` (SURVEY.md section 2).  The text encoders of `_create_text_encoder` /
`_create_student_text_encoder` (model_builder.py:487-556) are `create_text_encoder` / `create_student_text_encoder`."""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops
from .model.necks import Sam3DualViTDetNeck
from .stage1.model import EfficientViTAdapter, ImageStudentEncoder, RepViTAdapter, TinyViTAdapter

EFFICIENTVIT = ("b0", "b1", "b2")
REPVIT = {"m0.9": "repvit_m0_9", "m0_9": "repvit_m0_9", "m1.1": "repvit_m1_1", "m1_1": "repvit_m1_1", "m2.3": "repvit_m2_3",
          "m2_3": "repvit_m2_3"}
TINYVIT = {"5m": "tiny_vit_5m_224", "11m": "tiny_vit_11m_224", "21m": "tiny_vit_21m_224"}


class EfficientViTTrunkWrapper(EfficientViTAdapter):
    """model_builder.py:817-828."""

    def __init__(self, model):
        super().__init__(model)
        self.channel_list = [model.width_list[-1]]


class RepViTTrunkWrapper(RepViTAdapter):
    """model_builder.py:846-871 (classifier removed: no parameters under `model.classifier`)."""

    def __init__(self, model, out_channels):
        super().__init__(model, out_channels)
        if hasattr(model, "classifier"):
            delattr(model, "classifier")
        self.channel_list = [out_channels]


class TinyViTTrunkWrapper(TinyViTAdapter):
    """model_builder.py:893-911 (built with num_classes=0: `head` / `norm_head` are parameter-free Identities)."""

    def __init__(self, model, img_size):
        nn.Module.__init__(self)
        self.model = model
        self.out_channels = model.layers[-1].dim
        H, W = model.patches_resolution
        for _ in range(model.num_layers - 1):
            H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        self.final_hw = (H, W)
        self.channel_list = [self.out_channels]


class ListWrapper(nn.Module):
    """model_builder.py:925-933: the neck expects a list of feature maps."""

    def __init__(self, model):
        super().__init__()
        self.model = model
        self.channel_list = model.channel_list

    def forward(self, x):
        return [self.model(x)]

    def forward_nhwc(self, x):
        """[B,3,S,S] fp32 -> [B,72,72,1024] bf16 NHWC for Sam3DualViTDetNeck.forward_nhwc."""
        if ops.precision() == "strict":      # fp32 NHWC stream for the strict neck / heads (layout change only)
            return self.model(x).permute(0, 2, 3, 1).contiguous()
        return ops.nchw_f32_to_nhwc(self.model(x))


def create_student_vision_backbone(backbone_type: str, model_name: str, enable_inst_interactivity: bool = True,
                                   img_size: int = 1008, embed_size: int = 72) -> Sam3DualViTDetNeck:
    """`_create_student_vision_backbone(backbone_type, model_name, enable_inst_interactivity=...)` (model_builder.py:789-941);
    backbone_type in {"efficientvit", "repvit", "tinyvit"}.  (The reference fixes img_size 1008 / embed 72; they are arguments
    here only so that tests can run the TinyViT variant at small sizes.)"""
    if backbone_type == "efficientvit":
        from .backbones import efficientvit
        if model_name not in EFFICIENTVIT:
            raise ValueError(f"Unknown EfficientViT model: {model_name}")
        trunk = EfficientViTTrunkWrapper(getattr(efficientvit, f"efficientvit_backbone_{model_name}")())
    elif backbone_type == "repvit":
        from .backbones import repvit
        if model_name not in REPVIT:
            raise ValueError(f"Unknown RepViT model: {model_name}")
        model = getattr(repvit, REPVIT[model_name])(pretrained=False, num_classes=0, distillation=False)
        trunk = RepViTTrunkWrapper(model, repvit._make_divisible(model.cfgs[-1][2], 8))
    elif backbone_type == "tinyvit":
        from .backbones import tiny_vit
        if model_name not in TINYVIT:
            raise ValueError(f"Unknown TinyViT model: {model_name}")
        trunk = TinyViTTrunkWrapper(getattr(tiny_vit, TINYVIT[model_name])(pretrained=False, img_size=img_size, num_classes=0), img_size)
    else:
        raise ValueError(f"Unknown backbone type: {backbone_type}")
    student = ImageStudentEncoder(backbone=trunk, in_channels=trunk.channel_list[0], embed_dim=1024, embed_size=embed_size,
                                  img_size=img_size)
    student.channel_list = [1024]
    return Sam3DualViTDetNeck(trunk=ListWrapper(student), position_encoding=None, d_model=256, scale_factors=[4.0, 2.0, 1.0, 0.5],
                              add_sam2_neck=enable_inst_interactivity)


def build_efficientsam3_point_segmenter(backbone_type: str, model_name: str, image_size: int = 1008):
    """Sam3PointPromptSegmenter (batched SAM heads + predictor API) over an EfficientSAM3 student encoder instead of the
    SAM3 ViT trunk: `SAM3InteractiveImagePredictor(build_efficientsam3_point_segmenter("efficientvit", "b1"))`."""
    from .model.sam1_task import Sam3PointPromptSegmenter
    return Sam3PointPromptSegmenter(image_size=image_size, vision_backbone=create_student_vision_backbone(
        backbone_type, model_name, enable_inst_interactivity=True, img_size=image_size, embed_size=image_size // 14))


def create_text_encoder(bpe_path: str):
    """`_create_text_encoder(bpe_path)` (model_builder.py:487-496): the SAM3 text encoder, width 1024, 16 heads, 24 layers,
    32-entry positional table, resizer to d_model 256."""
    from .model.text_encoder_ve import VETextEncoder
    from .model.tokenizer_ve import SimpleTokenizer
    return VETextEncoder(tokenizer=SimpleTokenizer(bpe_path=bpe_path), d_model=256, width=1024, heads=16, layers=24)


def create_student_text_encoder(bpe_path: str, backbone_type: str, context_length: int = 32):
    """`_create_student_text_encoder(bpe_path, backbone_type, context_length)` (model_builder.py:499-556): the MobileCLIP
    student with a `context_length`-entry table, projector to d_model 256."""
    from .model.text_encoder_student import TextStudentEncoder
    from .stage1.model import text_student_cfg
    cfg = text_student_cfg(backbone_type)
    cfg["context_length"] = context_length
    return TextStudentEncoder(cfg=cfg, context_length=context_length, output_dim=256, bpe_path=bpe_path)
