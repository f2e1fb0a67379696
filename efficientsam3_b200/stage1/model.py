"""Drop-in for the reference `stage1/model.py` (image path): same builder / class names, same
state_dict keys, forward on libes3.so.

  build_image_student_model(config)   stage1/model.py:30-39
  ImageStudentEncoder                 stage1/model.py:188-211   (head.0/1/3 keys preserved)
  EfficientViTAdapter                 stage1/model.py:327-335
  _build_backbone                     stage1/model.py:386-417
  build_text_student_model(config)    stage1/model.py:42-165    (TextStudentEncoder, model/text_encoder_student.py)
  build_text_teacher_model(config)    stage1/model.py:178-185
  SAM3TextTeacherEncoder              stage1/model.py:252-284   (VETextEncoder, model/text_encoder_ve.py)

`config` needs MODEL.BACKBONE, DATA.IMG_SIZE, DISTILL.EMBED_DIM, DISTILL.EMBED_SIZE (yacs CfgNode or any
attribute namespace); the text builders read MODEL.BACKBONE / PRETRAINED / RESUME, DISTILL.EMBED_DIM / CONTEXT_LENGTH /
POS_EMBED_TABLE_SIZE and, for string input, the CLIP vocabulary path MODEL.BPE_PATH (the reference uses its bundled copy).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from ..backbones.efficientvit import (efficientvit_backbone_b0, efficientvit_backbone_b1,
                                      efficientvit_backbone_b2)
from ..nn_utils import NativePlanMixin, bn_scale_bias, conv3x3_weight, params_fingerprint, pw_weight, pw_weight_scaled


def build_image_student_model(config):
    backbone_name = config.MODEL.BACKBONE.lower()
    backbone, out_channels = _build_backbone(backbone_name, config.DATA.IMG_SIZE)
    return ImageStudentEncoder(backbone=backbone, in_channels=out_channels, embed_dim=config.DISTILL.EMBED_DIM,
                               embed_size=config.DISTILL.EMBED_SIZE, img_size=config.DATA.IMG_SIZE)


class ImageStudentEncoder(nn.Module, NativePlanMixin):
    def __init__(self, backbone, in_channels, embed_dim, embed_size, img_size):
        super().__init__()
        self.backbone = backbone
        self.embed_size = embed_size
        self.img_size = img_size
        # parameter containers; keys head.0.weight, head.1.{weight,bias,running_*}, head.3.{weight,bias}
        self.head = nn.Sequential(
            nn.Conv2d(in_channels, embed_dim, kernel_size=1, bias=False),
            nn.BatchNorm2d(embed_dim),
            nn.GELU(),
            nn.Conv2d(embed_dim, embed_dim, kernel_size=3, padding=1),
        )

    def _build_plan(self):
        dev = self.head[0].weight.device
        s, b = bn_scale_bias(self.head[1], None, self.head[0].out_channels, dev)
        return dict(w0=pw_weight_scaled(self.head[0], s), b0=b, w3=conv3x3_weight(self.head[3]),
                    b3=self.head[3].bias.detach().float().contiguous())

    def forward(self, x):
        if self.training:
            return self._forward_train(x)
        with torch.no_grad():
            if ops.precision() == "strict":           # fp32 activations / weights / accumulation (strict.py, csrc/strict_f32.cu)
                from ..strict import student_forward
                return student_forward(self, x)
            if self._graphs is not None and x.is_cuda:
                return self._forward_graphed(x)
            return self._forward_eval(x)

    # ---- CUDA-graph replay of the eval plan ----------------------------------------------------------------------------------
    # The eval forward is a fixed sequence of ~60 kernels whose arguments depend only on (input address, shape, packed weights).
    # Launching it kernel by kernel costs host time per step, which the device hides on one GPU but which becomes the limiter
    # when 8 ranks share one host.  With
    # `enable_cuda_graphs()` the sequence is captured once per (input buffer, shape) and replayed with ONE launch.
    _graphs = None
    graph_launches_per_step = 0

    def enable_cuda_graphs(self, enabled: bool = True, max_graphs: int = 4):
        """Replay the eval forward from a CUDA graph.  A graph is bound to the ADDRESS of its input tensor (feed a small rotating set
        of input buffers, as a double-buffered loader does) and to the current parameter values; it is re-captured when either moves.
        The returned tensor is the graph's own output buffer: it is overwritten by the next replay for the same input buffer."""
        self._graphs = {} if enabled else None
        self._graph_max = max_graphs
        return self

    def forward_uncaptured(self, x):
        with torch.no_grad():
            return self._forward_eval(x)

    def _forward_graphed(self, x):
        key = (x.data_ptr(), tuple(x.shape), x.dtype)
        fp = params_fingerprint(self)
        ent = self._graphs.get(key)
        if ent is None or ent["fp"] != fp:
            self._forward_eval(x)                      # un-captured pass: packs weights, sizes workspaces, configures kernels
            torch.cuda.synchronize(x.device)
            graph = torch.cuda.CUDAGraph()
            n0 = ops.launch_count
            with torch.cuda.graph(graph):              # private memory pool per graph: outputs of different graphs never alias
                out = self._forward_eval(x)
            ent = dict(graph=graph, out=out, fp=fp, x=x, launches=ops.launch_count - n0)   # holds x: the graph reads its address
            self._graphs.pop(key, None)
            while len(self._graphs) >= self._graph_max:
                self._graphs.pop(next(iter(self._graphs)))
            self._graphs[key] = ent
            self.graph_launches_per_step = ent["launches"]
        ent["graph"].replay()
        return ent["out"]

    def _forward_train(self, x):
        """Train-mode forward recorded as ONE autograd node (StudentTrainFunction): batch-statistics BatchNorm (or frozen
        BN modules, set_bn_state), backward on the kernels of train_bwd.cu.  Built for all nine students (EfficientViT b0 / b1 / b2, RepViT m0_9 / m1_1 / m2_3, TinyViT 5m / 11m / 21m)."""
        if not isinstance(self.backbone, (EfficientViTAdapter, RepViTAdapter, TinyViTAdapter)):
            raise NotImplementedError(
                "train-mode forward / backward is built for the nine students of the reference builder (EfficientViT, RepViT, "
                f"TinyViT adapters); {type(self.backbone).__name__} is eval-only.  Call .eval() first.")
        params = [p for p in self.parameters()]
        return StudentTrainFunction.apply(self, x, *params)

    def _forward_eval(self, x):
        if x.dtype in (torch.bfloat16, torch.float16):
            # half-width image batches (half the host->device bytes).  The first kernel of every student rounds the image to bf16
            # operands anyway (tensor-core stem), so a bf16 batch gives the results of its fp32 original for the fused EV-M stem.
            x = x.float()
        feats = self.backbone.forward_nhwc(x)          # [B,h,w,Cin] bf16
        p = self._plan()
        B, h, w, cin = feats.shape
        y = ops.gemm(feats.view(-1, cin), p["w0"], bias=p["b0"], act="gelu")       # BN scale folded into w0 (nn_utils.pw_weight_scaled)
        y = ops.conv3x3(y.view(B, h, w, -1), p["w3"], bias=p["b3"])
        if h != self.embed_size or w != self.embed_size:
            return ops.bilinear_nhwc_to_nchw(y, self.embed_size, self.embed_size)
        return ops.nhwc_to_nchw_f32(y)


class StudentTrainFunction(torch.autograd.Function):
    """preds = model(samples) with a native backward: forward runs the training graph (backbones/efficientvit_train.py) and
    keeps it; backward(d preds) walks it in reverse and returns one fp32 gradient per parameter, so `loss.backward()`,
    `p.grad`, DDP's gradient hooks and GradScaler work exactly as with the reference nn.Module."""

    @staticmethod
    def forward(ctx, module, x, *params):
        from ..backbones.efficientvit_train import EfficientViTTrainGraph, HeadTrainUnit
        ctx.module = module
        from ..backbones.repvit_train import RepViTTrainGraph
        from ..backbones.tinyvit_train import TinyViTTrainGraph
        if not (x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            raise ValueError("expected an fp32 NCHW image batch [B,3,H,W]")
        for m in module.modules():          # packed eval-mode weights go stale once parameters / running stats move
            if isinstance(m, NativePlanMixin):
                m._plan_key = None
        if isinstance(module.backbone, RepViTAdapter):
            body = RepViTTrainGraph(module.backbone.model)
        elif isinstance(module.backbone, TinyViTAdapter):
            body = TinyViTTrainGraph(module.backbone.model)
        else:
            body = EfficientViTTrainGraph(module.backbone.model)
        head = HeadTrainUnit(module.head, module.embed_size)
        out = head.forward(body.forward(x))
        ctx.graph = (body, head)
        ctx.params = params
        return out

    @staticmethod
    def backward(ctx, dout):
        if ctx.graph is None:
            raise RuntimeError("the native student keeps its saved activations for ONE backward pass (retain_graph / double backward "
                               "are not supported): run the forward again")
        body, head = ctx.graph
        ctx.graph = None
        from ..backbones.efficientvit_train import GradSink
        grads = GradSink()
        arena = getattr(ctx.module, "_es3_grad_arena", None)       # set by stage1.optim.FlatAdamW(direct_grads=True)
        grads.direct = arena is not None
        d = head.backward(dout, grads)
        if arena is not None:
            arena.head_grads_ready()                               # the head's weights (2/3 of EV-M's parameters) are final: exchange them now
        body.backward(d, grads)
        return (None, None) + tuple(grads.get(p) for p in ctx.params)


TEXT_STUDENT_DEFAULT_CFG = {   # stage1/model.py:46-59
    "context_length": 77, "vocab_size": 49408, "dim": 512, "ffn_multiplier_per_layer": 4.0, "n_heads_per_layer": 8,
    "n_transformer_layers": 12, "norm_layer": "layer_norm_fp32", "causal_masking": False, "model_name": "base",
    "embed_dropout": 0.0, "no_scale_embedding": False, "no_pos_embedding": False}

TEXT_STUDENT_VARIANTS = {      # stage1/model.py:61-96; any other name keeps the default cfg (no error, as in the reference)
    "MobileCLIP-S0": dict(dim=512, n_transformer_layers=4, n_heads_per_layer=8, model_name="mct", ffn_multiplier_per_layer=4.0),
    **{n: dict(dim=512, n_transformer_layers=12, n_heads_per_layer=8, model_name="base")
       for n in ("MobileCLIP-S1", "MobileCLIP2-S0", "MobileCLIP2-S2")},
    "MobileCLIP-B": dict(dim=512, n_transformer_layers=12, n_heads_per_layer=8, model_name="base", causal_masking=True),
    **{n: dict(dim=768, n_transformer_layers=12, n_heads_per_layer=12, model_name="base")
       for n in ("MobileCLIP2-S3", "MobileCLIP2-S4", "MobileCLIP2-L")},
}


def text_student_cfg(backbone: str) -> dict:
    cfg = dict(TEXT_STUDENT_DEFAULT_CFG)
    cfg.update(TEXT_STUDENT_VARIANTS.get(backbone, {}))
    return cfg


def build_text_student_model(config, logger=None):
    """stage1/model.py:42-165.  MODEL.PRETRAINED: a student checkpoint or a full MobileCLIP checkpoint (its `text_encoder.*`
    keys are renamed to `encoder.*`), loaded with strict=False; a load failure only warns, as in the reference."""
    from ..model.text_encoder_student import TextStudentEncoder
    cfg = text_student_cfg(config.MODEL.BACKBONE)
    context_length = getattr(config.DISTILL, "CONTEXT_LENGTH", 32)
    table = getattr(config.DISTILL, "POS_EMBED_TABLE_SIZE", 0)
    cfg["context_length"] = context_length if table in (None, 0) else table
    model = TextStudentEncoder(cfg=cfg, context_length=context_length, output_dim=config.DISTILL.EMBED_DIM,
                               bpe_path=getattr(config.MODEL, "BPE_PATH", None))
    if logger:
        logger.info(f"Text encoder context_length: {context_length}")
        logger.info(f"Text encoder pos_embed_table_size: {cfg['context_length']}")
    path = getattr(config.MODEL, "PRETRAINED", None)
    if path:
        try:
            sd = torch.load(path, map_location="cpu")
            if "text_encoder.embedding_layer.weight" in sd:
                sd = {k.replace("text_encoder.", "encoder.", 1): v for k, v in sd.items() if k.startswith("text_encoder.")}
            missing, unexpected = model.load_state_dict(sd, strict=False)
            if logger:
                logger.info(f"Loaded pretrained weights: {len(missing)} missing, {len(unexpected)} unexpected keys")
        except Exception as e:   # the reference continues from random initialisation (stage1/model.py:158-163)
            msg = f"Failed to load pretrained weights: {e}"
            if logger:
                logger.error(msg)
                logger.warning("Continuing with random initialization...")
            else:
                print(f"Warning: {msg}")
    return model


def build_text_teacher_model(config):
    """stage1/model.py:178-185."""
    checkpoint = getattr(config.MODEL, "RESUME", None) or None
    return SAM3TextTeacherEncoder(checkpoint_path=checkpoint, context_length=getattr(config.DISTILL, "CONTEXT_LENGTH", 32),
                                  bpe_path=getattr(config.MODEL, "BPE_PATH", None))


class SAM3TextTeacherEncoder(nn.Module):
    """stage1/model.py:252-284: the frozen SAM3 text encoder -> memory [Seq, B, 256] fp32.  Only the language backbone is
    instantiated, under the reference's key prefix `sam3.backbone.language_backbone.`; checkpoints with the `detector.` prefix
    load too.  It is built with its 32-entry positional table (VETextEncoder's default) and tokenises at `context_length`."""

    def __init__(self, checkpoint_path=None, context_length=32, bpe_path=None, ve_overrides=None):
        super().__init__()
        from ..model.text_encoder_ve import VETextEncoder
        from ..model.tokenizer_ve import SimpleTokenizer
        self.context_length = context_length
        kw = dict(d_model=256, width=1024, heads=16, layers=24)      # model_builder.py:487-496
        kw.update(ve_overrides or {})
        tok = SimpleTokenizer(bpe_path=bpe_path) if bpe_path is not None else None
        self.sam3 = _Holder()
        self.sam3.backbone = _Holder()
        self.sam3.backbone.language_backbone = VETextEncoder(tokenizer=tok, **kw)
        if checkpoint_path:
            sd = torch.load(checkpoint_path, map_location="cpu")
            sd = sd.get("model", sd)
            sd = {("sam3." + k[len("detector."):] if k.startswith("detector.") else k): v for k, v in sd.items()}
            own = set(self.state_dict().keys())
            self.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=False)
        for p in self.parameters():
            p.requires_grad = False
        self.eval()
        self.sam3.backbone.language_backbone.context_length = context_length

    def train(self, mode: bool = True):  # frozen teacher: always eval
        return super().train(False)

    @torch.no_grad()
    def forward(self, text, device=None):
        _, memory, _ = self.sam3.backbone.language_backbone(text, input_boxes=None, device=device)
        return memory[:self.context_length] if memory.shape[0] > self.context_length else memory

    # CUDA-graph replay of the eval forward: the VETextEncoder's (StagedGraphMixin), which this module calls
    def enable_cuda_graphs(self, enabled: bool = True, max_graphs: int = 4):
        """Replay the forward from CUDA graphs, one per (batch, context length); the returned memory is the graph's output buffer,
        overwritten by the next replay of the same shape.  Returns self."""
        self.sam3.backbone.language_backbone.enable_cuda_graphs(enabled, max_graphs)
        return self

    @property
    def graph_launches_per_step(self):
        return self.sam3.backbone.language_backbone.graph_launches_per_step

    @torch.no_grad()
    def forward_uncaptured(self, text, device=None):
        _, memory, _ = self.sam3.backbone.language_backbone.forward_uncaptured(text, input_boxes=None, device=device)
        return memory[:self.context_length] if memory.shape[0] > self.context_length else memory


def build_image_teacher_model(config):
    """stage1/model.py:168-175.  `config.MODEL.RESUME` (optional) is a reference SAM3 checkpoint."""
    checkpoint = getattr(config.MODEL, "RESUME", None) or None
    teacher = SAM3ImageTeacherEncoder(checkpoint_path=checkpoint, embed_size=config.DISTILL.EMBED_SIZE)
    teacher.img_size = config.DATA.IMG_SIZE
    return teacher


class _Holder(nn.Module):
    """Attribute container that reproduces the reference's key prefix `sam3.backbone.vision_backbone.trunk.`"""


class SAM3ImageTeacherEncoder(nn.Module):
    """stage1/model.py:214-249: frozen SAM3 ViT trunk -> [B,1024,72,72].  Only the trunk is instantiated (the
    reference builds the whole SAM3 model and then uses nothing else on this path); a full reference checkpoint
    loads with strict=False through the preserved key prefix."""

    def __init__(self, checkpoint_path=None, embed_size=64, vit_overrides=None):
        super().__init__()
        from ..model.vitdet import create_sam3_vit_backbone
        self.embed_size = embed_size
        self.sam3 = _Holder()
        self.sam3.backbone = _Holder()
        self.sam3.backbone.vision_backbone = _Holder()
        self.sam3.backbone.vision_backbone.trunk = create_sam3_vit_backbone(**(vit_overrides or {}))
        if checkpoint_path:
            sd = torch.load(checkpoint_path, map_location="cpu")
            sd = sd.get("model", sd)
            # reference checkpoints prefix the image model with "detector." (model_builder.py:584-630)
            sd = {("sam3." + k[len("detector."):] if k.startswith("detector.") else k): v for k, v in sd.items()}
            own = set(self.state_dict().keys())
            self.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=False)
        for p in self.parameters():
            p.requires_grad = False
        self.eval()
        self.img_size = 1008

    def train(self, mode: bool = True):  # frozen teacher: always eval (stage1/model.py:226-227)
        return super().train(False)

    @torch.no_grad()
    def forward(self, x):
        feats = self.sam3.backbone.vision_backbone.trunk(x)[-1]
        if feats.shape[-1] != self.embed_size or feats.shape[-2] != self.embed_size:
            # stage1/model.py:241-248 (bilinear, align_corners=False); a no-op in the shipped configs (EMBED_SIZE 72)
            feats, _ = ops.bilinear_nchw(feats, self.embed_size, self.embed_size)
        return feats

    def enable_fp8(self, enabled: bool = True, attention: bool = False):
        """Run the trunk's linear layers as block-scaled e4m3 GEMMs, and with attention=True its attention as FP8 flash attention
        too (ViT.enable_fp8; off by default).  Returns self."""
        self.sam3.backbone.vision_backbone.trunk.enable_fp8(enabled, attention=attention)
        return self


class RepViTAdapter(nn.Module):
    """stage1/model.py:287-296."""

    def __init__(self, model, out_channels):
        super().__init__()
        self.model = model
        self.out_channels = out_channels

    def forward(self, x):
        return ops.nhwc_to_nchw_f32(self.model.forward_nhwc(x))

    def forward_nhwc(self, x):
        return self.model.forward_nhwc(x)


class TinyViTAdapter(nn.Module):
    """stage1/model.py:299-324 (head / norm_head replaced by Identity)."""

    def __init__(self, model, img_size):
        super().__init__()
        self.model = model
        self.out_channels = self.model.norm_head.normalized_shape[0]
        self.model.head = nn.Identity()
        self.model.norm_head = nn.Identity()
        H, W = self.model.patches_resolution
        for _ in range(self.model.num_layers - 1):
            H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        self.final_hw = (H, W)

    def forward(self, x):
        return ops.nhwc_to_nchw_f32(self.model.forward_nhwc(x))

    def forward_nhwc(self, x):
        return self.model.forward_nhwc(x)


class EfficientViTAdapter(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model
        self.out_channels = self.model.width_list[-1]

    def forward(self, x):
        return self.model(x)["stage_final"]

    def forward_nhwc(self, x):
        return self.model.forward_nhwc(x)


def _build_backbone(name, img_size):
    if name.startswith("efficientvit"):
        fn = {"efficientvit_b0": efficientvit_backbone_b0, "efficientvit_b1": efficientvit_backbone_b1,
              "efficientvit_b2": efficientvit_backbone_b2}[name]
        adapter = EfficientViTAdapter(fn())
        return adapter, adapter.out_channels
    if name in ("repvit_m0_9", "repvit_m1_1", "repvit_m2_3"):
        from ..backbones import repvit
        model = getattr(repvit, name)(pretrained=False, num_classes=0, distillation=False)
        out_channels = repvit._make_divisible(model.cfgs[-1][2], 8)
        return RepViTAdapter(model, out_channels), out_channels
    if name in ("tiny_vit_5m", "tiny_vit_11m", "tiny_vit_21m"):
        from ..backbones import tiny_vit
        adapter = TinyViTAdapter(getattr(tiny_vit, name + "_224")(pretrained=False, img_size=img_size), img_size)
        return adapter, adapter.out_channels
    raise ValueError(f"Unsupported backbone {name}")
