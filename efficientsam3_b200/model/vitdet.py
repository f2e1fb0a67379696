"""SAM3 ViT trunk (the stage-1 teacher encoder), H100-native.  Mirrors the reference module tree of
`sam3/sam3/model/vitdet.py` for the configuration family SAM3 builds (model_builder.py:70-97): same
constructor arguments, same state_dict keys (`pos_embed`, `patch_embed.proj.weight`, `ln_pre.*`,
`blocks.N.{norm1,norm2}.*`, `blocks.N.attn.{qkv,proj}.*`, `blocks.N.attn.freqs_cis`, `blocks.N.mlp.{fc1,fc2}.*`).

Device path per block (all libes3.so):
  LayerNorm (fp32 residual stream -> bf16)              es3_layernorm_f32
  qkv Linear + bias + 2-D axial RoPE in the epilogue     es3_gemm_bf16_ex (wgmma)
  windowed / global softmax attention, no partition copy es3_attention_bf16
  proj Linear + bias + fp32 residual                     es3_gemm_bf16_ex
  LayerNorm, fc1 + GELU(erf), fc2 + fp32 residual        es3_layernorm_f32, es3_gemm_bf16_ex x2
Patch embedding = es3_im2col_patch + GEMM; tiled abs-pos add is fused into ln_pre.
Eval-mode only (the teacher is frozen: stage1/model.py:225-227).

ViT.enable_fp8() (off by default; the strict precision mode ignores it) moves the four linear layers to block-scaled e4m3
(gemm_fp8.cu): norm1 / norm2 write e4m3 (es3_layernorm_f32_e4m3), the attention output is quantised (es3_quantize_bf16_e4m3),
fc1's epilogue writes fc2's e4m3 operand, and the weights are packed once per parameter version (es3_pack_weight_e4m3).  Patch
embedding, the LayerNorm statistics, RoPE, attention and the fp32 residual stream stay as above.
ViT.enable_fp8(attention=True) moves attention to e4m3 as well (es3_attention_fp8: Q, K, V and P quantised on the device).
"""
from __future__ import annotations

import math
from functools import partial
from typing import Callable, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from .. import ops
from ..nn_utils import NativePlanMixin


def compute_axial_cis(dim, end_x, end_y, theta=10000.0, scale_pos=1.0, offset=0):
    """vitdet.py:41-57 -- kept as a complex64 buffer for state_dict compatibility."""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 4)[: (dim // 4)].float() / dim))
    t = torch.arange(end_x * end_y, dtype=torch.float32)
    t_x = (t % end_x).float() * scale_pos + offset
    t_y = torch.div(t, end_x, rounding_mode="floor").float() * scale_pos + offset
    fx, fy = torch.outer(t_x, freqs), torch.outer(t_y, freqs)
    return torch.cat([torch.polar(torch.ones_like(fx), fx), torch.polar(torch.ones_like(fy), fy)], dim=-1)


class PatchEmbed(nn.Module):
    def __init__(self, kernel_size=(16, 16), stride=(16, 16), padding=(0, 0), in_chans=3, embed_dim=768, bias=True):
        super().__init__()
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=kernel_size, stride=stride, padding=padding, bias=bias)


class Attention(nn.Module):
    def __init__(self, dim, num_heads=8, qkv_bias=True, use_rel_pos=False, rel_pos_zero_init=True, input_size=None,
                 cls_token=False, use_rope=False, rope_theta=10000.0, rope_pt_size=None, rope_interp=False):
        super().__init__()
        if use_rel_pos or cls_token or not use_rope:
            raise NotImplementedError("native ViT attention covers the SAM3 configuration: rope, no rel-pos, no cls token")
        self.num_heads, self.head_dim = num_heads, dim // num_heads
        self.scale = self.head_dim ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.input_size = input_size
        rope_pt_size = input_size if rope_pt_size is None else rope_pt_size
        scale_pos = rope_pt_size[0] / input_size[0] if rope_interp else 1.0
        self.register_buffer("freqs_cis", compute_axial_cis(self.head_dim, input_size[0], input_size[1], rope_theta,
                                                            scale_pos))


class Mlp(nn.Module):
    """timm.layers.Mlp parameter layout (fc1, fc2); GELU(erf) in between."""

    def __init__(self, in_features, hidden_features, act_layer=nn.GELU, drop=(0.0, 0.0)):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.fc2 = nn.Linear(hidden_features, in_features)


class Block(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=True, drop_path=0.0, norm_layer=nn.LayerNorm,
                 act_layer=nn.GELU, use_rel_pos=False, rel_pos_zero_init=True, window_size=0, input_size=None,
                 use_rope=False, rope_pt_size=None, rope_tiled=False, rope_interp=False, use_ve_rope=False,
                 cls_token=False, dropout=0.0, init_values=None):
        super().__init__()
        if init_values:
            raise NotImplementedError("LayerScale is not used by SAM3 (init_values=None)")
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, use_rel_pos=use_rel_pos,
                              rel_pos_zero_init=rel_pos_zero_init,
                              input_size=input_size if window_size == 0 else (window_size, window_size),
                              use_rope=use_rope, rope_pt_size=rope_pt_size, rope_interp=rope_interp, cls_token=cls_token)
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio), act_layer=act_layer, drop=(dropout, 0.0))
        self.window_size = window_size


def _lin(linear: nn.Linear):
    return (linear.weight.detach().to(torch.bfloat16).contiguous(),
            linear.bias.detach().float().contiguous() if linear.bias is not None else None)


def _lin8(linear: nn.Linear):
    w = linear.weight.detach()
    return (*ops.pack_weight_e4m3(w if w.dtype in (torch.bfloat16, torch.float32) else w.float()),
            linear.bias.detach().float().contiguous() if linear.bias is not None else None)


class ViT(nn.Module, NativePlanMixin):
    def __init__(self, img_size=1024, patch_size=16, in_chans=3, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4.0,
                 qkv_bias=True, drop_path_rate=0.0, norm_layer: Union[Callable[..., nn.Module], str] = "LayerNorm",
                 act_layer=nn.GELU, use_abs_pos=True, tile_abs_pos=True, rel_pos_blocks=(2, 5, 8, 11),
                 rel_pos_zero_init=True, window_size=14, global_att_blocks=(2, 5, 8, 11), use_rope=False,
                 rope_pt_size=None, use_interp_rope=False, pretrain_img_size=224, pretrain_use_cls_token=True,
                 retain_cls_token=True, dropout=0.0, return_interm_layers=False, init_values=None, ln_pre=False,
                 ln_post=False, bias_patch_embed=True, compile_mode=None, use_act_checkpoint=True):
        super().__init__()
        if retain_cls_token or not (use_abs_pos and tile_abs_pos) or not ln_pre or ln_post or return_interm_layers \
                or (not isinstance(rel_pos_blocks, bool) and len(rel_pos_blocks) > 0) or rel_pos_blocks is True \
                or bias_patch_embed or in_chans != 3:
            raise NotImplementedError("native ViT covers the SAM3 trunk configuration (model_builder.py:70-97)")
        if isinstance(norm_layer, str):
            norm_layer = partial(getattr(nn, norm_layer), eps=1e-5)
        self.img_size, self.patch_size, self.embed_dim, self.num_heads = img_size, patch_size, embed_dim, num_heads
        self.window_size = window_size
        self.full_attn_ids = list(global_att_blocks)
        self.pretrain_use_cls_token = pretrain_use_cls_token
        self.patch_embed = PatchEmbed((patch_size, patch_size), (patch_size, patch_size), in_chans=in_chans,
                                      embed_dim=embed_dim, bias=False)
        n_pos = (pretrain_img_size // patch_size) ** 2 + (1 if pretrain_use_cls_token else 0)
        self.pos_embed = nn.Parameter(torch.zeros(1, n_pos, embed_dim))
        nn.init.trunc_normal_(self.pos_embed, std=0.02)
        grid = img_size // patch_size
        self.blocks = nn.ModuleList()
        for i in range(depth):
            self.blocks.append(Block(
                dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, norm_layer=norm_layer,
                act_layer=act_layer, window_size=0 if i in global_att_blocks else window_size, input_size=(grid, grid),
                use_rope=use_rope,
                rope_pt_size=(window_size, window_size) if rope_pt_size is None else (rope_pt_size, rope_pt_size),
                rope_interp=use_interp_rope, dropout=dropout, init_values=init_values))
        self.channel_list = [embed_dim]
        self.ln_pre = norm_layer(embed_dim)
        self.ln_post = nn.Identity()
        for m in self.modules():  # vitdet.py:789-796
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)

    _fp8 = False
    _fp8_attn = False

    def enable_fp8(self, enabled: bool = True, attention: bool = False):
        """Run qkv, proj, fc1 and fc2 as block-scaled e4m3 GEMMs (off by default; ignored in the strict precision mode).  The
        weights are packed to e4m3 on the next forward and again whenever a parameter changes.  attention=True also runs every
        block's attention as FP8 flash attention (ops.attention_fp8); it needs enabled=True.  Returns self."""
        if attention and not enabled:
            raise ValueError("enable_fp8: attention=True needs the FP8 linear layers (enabled=True)")
        self._fp8 = bool(enabled)
        self._fp8_attn = bool(attention)
        self._plan_key = None
        return self

    def _build_plan(self):
        P, C = self.patch_size, self.embed_dim
        kp = (3 * P * P + 7) // 8 * 8
        dev = self.pos_embed.device
        wpe = torch.zeros((C, kp), device=dev, dtype=torch.bfloat16)
        wpe[:, : 3 * P * P] = self.patch_embed.proj.weight.detach().reshape(C, -1).to(torch.bfloat16)
        tab = self.pos_embed.detach()[0, 1:] if self.pretrain_use_cls_token else self.pos_embed.detach()[0]
        blocks = []
        for blk in self.blocks:
            blocks.append(dict(
                n1=(blk.norm1.weight.detach().float().contiguous(), blk.norm1.bias.detach().float().contiguous(), blk.norm1.eps),
                n2=(blk.norm2.weight.detach().float().contiguous(), blk.norm2.bias.detach().float().contiguous(), blk.norm2.eps),
                qkv=_lin(blk.attn.qkv), proj=_lin(blk.attn.proj), fc1=_lin(blk.mlp.fc1), fc2=_lin(blk.mlp.fc2),
                rope=torch.view_as_real(blk.attn.freqs_cis.detach().to(torch.complex64)).float().contiguous(),
                win=blk.window_size, scale=blk.attn.scale))
            if self._fp8:
                blocks[-1].update(qkv8=_lin8(blk.attn.qkv), proj8=_lin8(blk.attn.proj), fc1_8=_lin8(blk.mlp.fc1),
                                  fc2_8=_lin8(blk.mlp.fc2))
        return dict(kp=kp, wpe=wpe, pos=tab.float().contiguous(), pos_size=int(math.isqrt(tab.shape[0])),
                    ln_pre=(self.ln_pre.weight.detach().float().contiguous(), self.ln_pre.bias.detach().float().contiguous(),
                            self.ln_pre.eps), blocks=blocks)

    @torch.no_grad()
    def forward_tokens(self, x: torch.Tensor):
        """x [B,3,S,S] fp32 CUDA -> fp32 tokens [B*h*w, C] after the last block, plus (B, h, w)."""
        self._require_eval("ViT.forward")
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            raise ValueError("expected a CUDA fp32 NCHW image batch; the native path has no CPU fallback")
        B, _, S, S2 = x.shape
        assert S == S2 and S % self.patch_size == 0
        h = w = S // self.patch_size
        # the reference asserts on the RoPE table shape for any other size (SURVEY.md D2, vitdet.py:60-65)
        assert h == self.img_size // self.patch_size, f"ViT built for {self.img_size}px inputs, got {S}"
        if ops.precision() == "strict":               # fp32 operands / accumulation end to end (strict.py, csrc/strict_f32.cu)
            from ..strict import vit_tokens
            return vit_tokens(self, x)
        p = self._plan()
        C, heads = self.embed_dim, self.num_heads
        cols = ops.im2col_patch(x, self.patch_size, p["kp"])
        tok = ops.gemm(cols, p["wpe"], out_dtype=torch.float32)
        g, b_, eps = p["ln_pre"]
        _, xs = ops.layernorm(tok, g, b_, eps, pos=p["pos"], pos_size=p["pos_size"], H=h, W=w, out_bf16=False, out_f32=True)
        if self._fp8:
            for bp in p["blocks"]:
                q, s = ops.layernorm_e4m3(xs, *bp["n1"])
                qkv = ops.gemm_fp8(q, s, *bp["qkv8"], rope=(bp["rope"], 2 * C, h, w, bp["win"]))
                attn = ops.attention_fp8 if self._fp8_attn else ops.attention
                a = attn(qkv, B, h, w, C, heads, bp["win"], bp["scale"])
                xs = ops.gemm_fp8(*ops.quantize_e4m3(a), *bp["proj8"], residual=xs, out_dtype=torch.float32)
                q, s = ops.layernorm_e4m3(xs, *bp["n2"])
                q, s = ops.gemm_fp8(q, s, *bp["fc1_8"], act="gelu", out_dtype=ops.E4M3)
                xs = ops.gemm_fp8(q, s, *bp["fc2_8"], residual=xs, out_dtype=torch.float32)
            return xs, (B, h, w)
        for bp in p["blocks"]:
            y, _ = ops.layernorm(xs, *bp["n1"])
            qkv = ops.gemm(y, bp["qkv"][0], bias=bp["qkv"][1], rope=(bp["rope"], 2 * C, h, w, bp["win"]))
            a = ops.attention(qkv, B, h, w, C, heads, bp["win"], bp["scale"])
            xs = ops.gemm(a, bp["proj"][0], bias=bp["proj"][1], residual=xs, out_dtype=torch.float32)
            y, _ = ops.layernorm(xs, *bp["n2"])
            hdn = ops.gemm(y, bp["fc1"][0], bias=bp["fc1"][1], act="gelu")
            xs = ops.gemm(hdn, bp["fc2"][0], bias=bp["fc2"][1], residual=xs, out_dtype=torch.float32)
        return xs, (B, h, w)

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        xs, (B, h, w) = self.forward_tokens(x)
        return [ops.tokens_f32_to_nchw(xs, B, h, w)]


SAM3_VIT_KWARGS = dict(  # sam3/sam3/model_builder.py:70-97
    img_size=1008, pretrain_img_size=336, patch_size=14, embed_dim=1024, depth=32, num_heads=16, mlp_ratio=4.625,
    norm_layer="LayerNorm", drop_path_rate=0.1, qkv_bias=True, use_abs_pos=True, tile_abs_pos=True,
    global_att_blocks=(7, 15, 23, 31), rel_pos_blocks=(), use_rope=True, use_interp_rope=True, window_size=24,
    pretrain_use_cls_token=True, retain_cls_token=False, ln_pre=True, ln_post=False, return_interm_layers=False,
    bias_patch_embed=False)


def create_sam3_vit_backbone(**overrides):
    kw = dict(SAM3_VIT_KWARGS)
    kw.update(overrides)
    return ViT(**kw)
