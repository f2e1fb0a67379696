"""MobileCLIP text transformer (the stage-1 text students), H100-native.  Mirrors `sam3/sam3/backbones/mobile_clip.py`:
same class names, constructor arguments and state_dict keys (`embedding_layer.weight`,
`positional_embedding.pos_embed.pos_embed`, `transformer.N.pre_norm_mha.{0,1.qkv_proj,1.out_proj}.*`,
`transformer.N.pre_norm_ffn.{0,1,4}.*`, the RepMixerBlock's `token_mixer.{norm,mixer}.*`, `convffn.*`, `layer_scale`,
`final_layer_norm.*`, `projection_layer`).  The nn modules are parameter containers; eval-mode forward only.

Device path (all libes3.so; fp32 residual stream, bf16 GEMM operands, fp32 accumulation / LayerNorm / softmax):
  embedding gather + positional add                      es3_text_embed
  TransformerEncoder: LN, qkv, attention, out_proj + res  es3_layernorm_f32, es3_gemm_bf16_ex,
                      LN, fc1 + GELU, fc2 + res           es3_attention_bf16 (H=1, W=L) | es3_attention_causal_bf16
  RepMixerBlock: folded token mixer + ConvFFN dwconv     es3_repmixer_bf16
                 fc1 + GELU, fc2 x layer_scale + res      es3_gemm_bf16_ex x2
  final LayerNorm (+ projection)                         es3_layernorm_f32 (+ es3_gemm_bf16_ex)
"""
from __future__ import annotations

import math
from typing import List, Optional, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..nn_utils import NativePlanMixin, bn_scale_bias


# ----------------------------------------------------------------------------------------------- parameter containers
class MobileOneBlock(nn.Module):
    """mobile_clip.py:48-244, training-time (un-reparameterised) form; the text encoders build it without SE and act."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 inference_mode=False, use_se=False, use_act=True, use_scale_branch=True, num_conv_branches=1,
                 activation: nn.Module = nn.GELU()):
        super().__init__()
        if inference_mode or use_se:
            raise NotImplementedError("MobileOneBlock: reparameterised (reparam_conv) and SE blocks are not part of the "
                                      "text encoders' native path")
        self.inference_mode, self.groups, self.stride, self.padding = inference_mode, groups, stride, padding
        self.dilation, self.kernel_size = dilation, kernel_size
        self.in_channels, self.out_channels, self.num_conv_branches = in_channels, out_channels, num_conv_branches
        self.se = nn.Identity()
        self.activation = activation if use_act else nn.Identity()
        self.rbr_skip = nn.BatchNorm2d(in_channels) if out_channels == in_channels and stride == 1 else None
        self.rbr_conv = nn.ModuleList([self._conv_bn(kernel_size, padding) for _ in range(num_conv_branches)]) \
            if num_conv_branches > 0 else None
        self.rbr_scale = None
        k0 = kernel_size if isinstance(kernel_size, int) else kernel_size[0]
        if k0 > 1 and use_scale_branch:          # a (1, k) kernel has no scale branch (mobile_clip.py:115-119)
            self.rbr_scale = self._conv_bn(1, 0)

    def _conv_bn(self, kernel_size, padding):
        m = nn.Sequential()
        m.add_module("conv", nn.Conv2d(self.in_channels, self.out_channels, kernel_size=kernel_size, stride=self.stride,
                                       padding=padding, groups=self.groups, bias=False))
        m.add_module("bn", nn.BatchNorm2d(self.out_channels))
        return m


class LayerNormFP32(nn.LayerNorm):
    """mobile_clip.py:250-269 (LayerNorm computed in fp32: the native LayerNorm always is)."""


def get_normalization_layer(norm_type, num_features):
    if norm_type == "layer_norm":
        return nn.LayerNorm(num_features)
    if norm_type == "layer_norm_fp32":
        return LayerNormFP32(num_features)
    raise NotImplementedError(f"Option: {norm_type} not supported.")


class LearnablePositionalEmbedding(nn.Module):
    def __init__(self, num_embeddings, embedding_dim, padding_idx=None, interpolation_mode="bilinear", *args, **kwargs):
        super().__init__()
        self.pos_embed = nn.Parameter(torch.empty(1, 1, num_embeddings, embedding_dim))
        self.embedding_dim, self.num_embeddings = embedding_dim, num_embeddings
        self.padding_idx, self.interpolation_mode = padding_idx, interpolation_mode
        nn.init.trunc_normal_(self.pos_embed, mean=0, std=embedding_dim ** -0.5)
        if padding_idx is not None:
            with torch.no_grad():
                self.pos_embed[:, :, padding_idx, ...] = 0.0

    def table(self, seq_len: int) -> torch.Tensor:
        """[seq_len, D] fp32 as mobile_clip.py:305-317 computes it: the table resized with F.interpolate(bilinear,
        align_corners=False) on [1,1,N,D] when seq_len != N.  Weight preparation on the host (cached in the plan)."""
        pe = self.pos_embed.detach().float().cpu().clone()
        if self.padding_idx is not None:
            pe[:, :, self.padding_idx, ...] = 0.0
        if seq_len != self.num_embeddings:
            pe = F.interpolate(pe, size=(seq_len, self.embedding_dim), mode=self.interpolation_mode)
        return pe.reshape(seq_len, self.embedding_dim).contiguous()


class PositionalEmbedding(nn.Module):
    def __init__(self, num_embeddings, embedding_dim, padding_idx=None, is_learnable=False, interpolation_mode="bilinear",
                 *args, **kwargs):
        super().__init__()
        self.pos_embed = LearnablePositionalEmbedding(num_embeddings, embedding_dim, padding_idx, interpolation_mode)


class MultiHeadAttention(nn.Module):
    """mobile_clip.py:345-424: qkv_proj [q|k|v] x heads, q * head_dim^-0.5, softmax in fp32, out_proj."""

    def __init__(self, embed_dim, num_heads, attn_dropout=0.0, bias=True, output_dim=None, *args, **kwargs):
        super().__init__()
        output_dim = output_dim or embed_dim
        self.qkv_proj = nn.Linear(embed_dim, 3 * embed_dim, bias=bias)
        self.attn_dropout = nn.Dropout(p=attn_dropout)
        self.out_proj = nn.Linear(embed_dim, output_dim, bias=bias)
        self.head_dim = embed_dim // num_heads
        self.scaling = self.head_dim ** -0.5
        self.softmax = nn.Softmax(dim=-1)
        self.num_heads, self.embed_dim = num_heads, embed_dim


class TransformerEncoder(nn.Module):
    """mobile_clip.py:427-491: pre-norm attention and FFN, both residual."""

    def __init__(self, embed_dim, ffn_latent_dim, num_heads=8, attn_dropout=0.0, dropout=0.0, ffn_dropout=0.0,
                 transformer_norm_layer="layer_norm", stochastic_dropout=0.0, *args, **kwargs):
        super().__init__()
        self.pre_norm_mha = nn.Sequential(get_normalization_layer(transformer_norm_layer, embed_dim),
                                          MultiHeadAttention(embed_dim, num_heads, attn_dropout=attn_dropout, bias=True),
                                          nn.Dropout(p=dropout))
        self.pre_norm_ffn = nn.Sequential(get_normalization_layer(transformer_norm_layer, embed_dim),
                                          nn.Linear(embed_dim, ffn_latent_dim, bias=True), nn.GELU(), nn.Dropout(p=ffn_dropout),
                                          nn.Linear(ffn_latent_dim, embed_dim, bias=True), nn.Dropout(p=dropout))
        self.drop_path = nn.Identity()


class ConvFFN(nn.Module):
    """mobile_clip.py:497-542: depthwise (1, k) conv + BN, fc1 (1x1, bias), GELU, fc2."""

    def __init__(self, in_channels, context_size, hidden_channels=None, out_channels=None, act_layer=nn.GELU, drop=0.0):
        super().__init__()
        out_channels = out_channels or in_channels
        hidden_channels = hidden_channels or in_channels
        self.conv = nn.Sequential()
        self.conv.add_module("conv", nn.Conv2d(in_channels, out_channels, kernel_size=(1, int(context_size)),
                                               padding=(0, int(context_size // 2)), groups=in_channels, bias=False))
        self.conv.add_module("bn", nn.BatchNorm2d(out_channels))
        self.fc1 = nn.Conv2d(in_channels, hidden_channels, kernel_size=1)
        self.act = act_layer()
        self.fc2 = nn.Conv2d(hidden_channels, out_channels, kernel_size=1)
        self.drop = nn.Dropout(drop)
        for m in (self.conv.conv, self.fc1, self.fc2):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)


class RepMixer(nn.Module):
    """mobile_clip.py:545-603: x + layer_scale * (mixer(x) - norm(x)); mixer = BN_skip + BN(conv 1xk), norm = BN_skip."""

    def __init__(self, dim, kernel_size=3, use_layer_scale=True, layer_scale_init_value=1e-5, inference_mode=False):
        super().__init__()
        if inference_mode:
            raise NotImplementedError("RepMixer: reparameterised (reparam_conv) checkpoints are not supported")
        self.dim, self.kernel_size, self.inference_mode = dim, kernel_size, inference_mode
        self.norm = MobileOneBlock(dim, dim, (1, kernel_size), padding=(0, kernel_size // 2), groups=dim, use_act=False,
                                   use_scale_branch=False, num_conv_branches=0)
        self.mixer = MobileOneBlock(dim, dim, (1, kernel_size), padding=(0, kernel_size // 2), groups=dim, use_act=False)
        self.use_layer_scale = use_layer_scale
        if use_layer_scale:
            self.layer_scale = nn.Parameter(layer_scale_init_value * torch.ones((dim, 1, 1)), requires_grad=True)


class RepMixerBlock(nn.Module):
    """mobile_clip.py:647-702: x1 = token_mixer(x); x1 + layer_scale * convffn(x1), on [B, C, 1, L]."""

    def __init__(self, dim, kernel_size=11, mlp_ratio=4.0, act_layer=nn.GELU, drop=0.0, drop_path=0.0, use_layer_scale=True,
                 layer_scale_init_value=1e-5, inference_mode=False, *args, **kwargs):
        super().__init__()
        if kernel_size != 11:
            raise NotImplementedError(f"RepMixerBlock: the native kernel is built for the 1x11 convs, got {kernel_size}")
        self.token_mixer = RepMixer(dim, kernel_size=kernel_size, use_layer_scale=use_layer_scale,
                                    layer_scale_init_value=layer_scale_init_value, inference_mode=inference_mode)
        self.convffn = ConvFFN(dim, context_size=kernel_size, hidden_channels=int(dim * mlp_ratio), act_layer=act_layer,
                               drop=drop)
        self.drop_path = nn.Identity()
        self.use_layer_scale = use_layer_scale
        if use_layer_scale:
            self.layer_scale = nn.Parameter(layer_scale_init_value * torch.ones((dim, 1, 1)), requires_grad=True)


# ----------------------------------------------------------------------------------------------- plans and the trunk
def _f32(t):
    return t.detach().float().contiguous()


def _lin(linear: nn.Linear):
    return (linear.weight.detach().to(torch.bfloat16).contiguous(), _f32(linear.bias) if linear.bias is not None else None)


def _bn(bn: nn.BatchNorm2d):
    return bn_scale_bias(bn, None, bn.num_features, bn.weight.device)


def _taps(conv: nn.Conv2d, scale):
    """depthwise (1, 11) weight [C,1,1,11] x per-channel scale -> fp32 [11, C] tap-major."""
    w = conv.weight.detach().float()
    return (w.reshape(w.shape[0], -1) * scale.view(-1, 1)).t().contiguous()


def encoder_layer_plan(blk: TransformerEncoder):
    n1, attn, n2 = blk.pre_norm_mha[0], blk.pre_norm_mha[1], blk.pre_norm_ffn[0]
    return dict(kind="attn", n1=(_f32(n1.weight), _f32(n1.bias), n1.eps), qkv=_lin(attn.qkv_proj), proj=_lin(attn.out_proj),
                n2=(_f32(n2.weight), _f32(n2.bias), n2.eps), fc1=_lin(blk.pre_norm_ffn[1]), fc2=_lin(blk.pre_norm_ffn[4]),
                heads=attn.num_heads, scale=attn.scaling)


def repmixer_plan(blk: RepMixerBlock):
    """Eval-mode RepMixerBlock folded to the es3_repmixer_bf16 taps and the two GEMMs (mobile_clip.py:594-702):
    x1 = x + ls (BN_ms(x) + BN_mc(conv(x)) - BN_ns(x)) = sum_k wm[k] x[l+k-5] + bm,  u = BN_f(conv_f(x1)),
    out = x1 + ls_blk (fc2(gelu(fc1(u))))."""
    tm, ffn = blk.token_mixer, blk.convffn
    dim = tm.dim
    ls = _f32(tm.layer_scale).reshape(-1) if tm.use_layer_scale else torch.ones(dim, device=tm.mixer.rbr_skip.weight.device)
    s_ms, b_ms = _bn(tm.mixer.rbr_skip)
    s_mc, b_mc = _bn(tm.mixer.rbr_conv[0].bn)
    s_ns, b_ns = _bn(tm.norm.rbr_skip)
    wm = _taps(tm.mixer.rbr_conv[0].conv, ls * s_mc)
    wm[tm.kernel_size // 2] += 1.0 + ls * (s_ms - s_ns)
    bm = (ls * (b_ms + b_mc - b_ns)).contiguous()
    s_f, b_f = _bn(ffn.conv.bn)
    lsb = _f32(blk.layer_scale).reshape(-1) if blk.use_layer_scale else torch.ones_like(ls)
    w1 = ffn.fc1.weight.detach().reshape(ffn.fc1.out_channels, -1).to(torch.bfloat16).contiguous()
    w2 = ffn.fc2.weight.detach().reshape(ffn.fc2.out_channels, -1).to(torch.bfloat16).contiguous()
    return dict(kind="repmixer", wm=wm.contiguous(), bm=bm, wf=_taps(ffn.conv.conv, s_f), bf=b_f.contiguous(),
                fc1=(w1, _f32(ffn.fc1.bias)), fc2=(w2, lsb.contiguous(), (lsb * _f32(ffn.fc2.bias)).contiguous()))


def run_layers(layers, x, B, L, causal):
    """The residual trunk on x [B*L, C] fp32 (not modified) -> fp32 [B*L, C]."""
    C = x.shape[1]
    for lp in layers:
        if lp["kind"] == "repmixer":
            x1, u = ops.repmixer(x, B, L, lp["wm"], lp["bm"], lp["wf"], lp["bf"])
            h = ops.gemm(u, lp["fc1"][0], bias=lp["fc1"][1], act="gelu")
            w2, s2, b2 = lp["fc2"]
            x = ops.gemm(h, w2, scale=s2, bias=b2, residual=x1, out_dtype=torch.float32)
            continue
        y, _ = ops.layernorm(x, *lp["n1"])
        qkv = ops.gemm(y, lp["qkv"][0], bias=lp["qkv"][1])
        if causal:
            a = ops.attention_causal(qkv, B, L, C, lp["heads"], lp["scale"])
        else:
            a = ops.attention(qkv, B, 1, L, C, lp["heads"], 0, lp["scale"])
        x = ops.gemm(a, lp["proj"][0], bias=lp["proj"][1], residual=x, out_dtype=torch.float32)
        y, _ = ops.layernorm(x, *lp["n2"])
        h = ops.gemm(y, lp["fc1"][0], bias=lp["fc1"][1], act="gelu")
        x = ops.gemm(h, lp["fc2"][0], bias=lp["fc2"][1], residual=x, out_dtype=torch.float32)
    return x


def check_native(module: nn.Module, what: str, training: bool):
    """The raise paths shared by the text modules: no CPU fallback, eval-mode only, no strict (fp32) mode yet."""
    if training:
        raise NotImplementedError(f"{what}: the text encoders' native path is eval-mode (forward) only; training the text "
                                  "student (backward, batch-statistics BatchNorm) is not built yet.  Call .eval() first.")
    if ops.precision() == "strict":
        raise NotImplementedError(f"{what}: the strict (fp32) precision mode is not built for the text encoders")
    p = next(module.parameters())
    if not p.is_cuda:
        raise RuntimeError(f"{what}: the module is on {p.device}; the native path runs on a CUDA device and has no CPU fallback")
    return p.device


def host_ids(ids: torch.Tensor, vocab: int) -> torch.Tensor:
    """Token ids checked on the host before they reach the device: int64 [B, L], every id in [0, vocab)."""
    if not torch.is_tensor(ids) or ids.dim() != 2 or ids.dtype not in (torch.int64, torch.int32):
        raise ValueError("expected token ids as an integer tensor [B, L]")
    h = ids.detach().to("cpu", torch.int64).contiguous()
    if h.numel() and (int(h.min()) < 0 or int(h.max()) >= vocab):
        raise ValueError(f"token id out of range [0, {vocab}): min {int(h.min())}, max {int(h.max())}")
    return h


class MobileCLIPTextTransformer(nn.Module, NativePlanMixin):
    def __init__(self, cfg: dict, projection_dim: int, skip_embeddings: bool = False, *args, **kwargs) -> None:
        super().__init__()
        if skip_embeddings:
            raise NotImplementedError("MobileCLIPTextTransformer(skip_embeddings=True) is not used by the text students")
        model_dim = cfg["dim"]
        norm_layer = cfg["norm_layer"]
        variant = cfg["model_name"]
        self.vocab_size = cfg["vocab_size"]
        self.projection_dim = projection_dim
        self.skip_embeddings = skip_embeddings
        self.embedding_layer = nn.Embedding(embedding_dim=model_dim, num_embeddings=self.vocab_size)
        self.embed_scale = 1.0 if cfg.get("no_scale_embedding", False) else model_dim ** -0.5   # unused, as in the reference
        self.positional_embedding = None if cfg.get("no_pos_embedding", False) else \
            PositionalEmbedding(num_embeddings=cfg["context_length"], embedding_dim=model_dim)
        self.embedding_dropout = nn.Dropout(p=cfg.get("embed_dropout", 0.0))
        n_layers = cfg["n_transformer_layers"]
        mult = cfg["ffn_multiplier_per_layer"]
        mult = [mult] * n_layers if isinstance(mult, (float, int)) else mult
        ffn_dims = [int(math.ceil(model_dim * m / 16.0) * 16.0) for m in mult]
        heads = cfg["n_heads_per_layer"]
        heads = [heads] * n_layers if isinstance(heads, int) else heads
        enc = [TransformerEncoder(embed_dim=model_dim, num_heads=heads[i], ffn_latent_dim=ffn_dims[i],
                                  transformer_norm_layer=norm_layer) for i in range(n_layers)]
        if variant == "base":
            self.transformer = nn.ModuleList(enc)
        elif variant == "mct":
            self.transformer = nn.ModuleList([RepMixerBlock(dim=model_dim), *enc, RepMixerBlock(dim=model_dim)])
        else:
            raise ValueError("Unrecognized text encoder variant {}".format(variant))
        self.final_layer_norm = get_normalization_layer(num_features=model_dim, norm_type=norm_layer)
        self.projection_layer = nn.Parameter(torch.empty(model_dim, self.projection_dim))
        nn.init.normal_(self.projection_layer, std=model_dim ** -0.5)
        self.model_dim = model_dim
        self.causal_masking = cfg["causal_masking"]

    def resize_pos_embed(self, new_length: int):
        """mobile_clip.py:709-724: truncates the table (a new Parameter) when new_length is shorter; never grows it."""
        if self.positional_embedding is None:
            return
        lpe = self.positional_embedding.pos_embed
        if new_length < lpe.pos_embed.shape[2]:
            lpe.pos_embed = nn.Parameter(lpe.pos_embed.detach()[:, :, :new_length, :].clone())
            lpe.num_embeddings = new_length

    def _build_plan(self):
        fl = self.final_layer_norm
        layers = [repmixer_plan(b) if isinstance(b, RepMixerBlock) else encoder_layer_plan(b) for b in self.transformer]
        return dict(table=_f32(self.embedding_layer.weight), layers=layers, pos={},
                    ln=(_f32(fl.weight), _f32(fl.bias), fl.eps),
                    proj=self.projection_layer.detach().t().to(torch.bfloat16).contiguous())

    def _pos(self, p, L, dev):
        if self.positional_embedding is None:
            return None
        if L not in p["pos"]:
            p["pos"][L] = self.positional_embedding.pos_embed.table(L).to(dev)
        return p["pos"][L]

    @torch.no_grad()
    def embed_tokens(self, ids: torch.Tensor):
        """forward_embedding on validated ids -> fp32 [B*L, C] (token + positional embedding), also the residual stream."""
        dev = check_native(self, "MobileCLIPTextTransformer", self.training)
        h = host_ids(ids, self.vocab_size)
        p = self._plan()
        B, L = h.shape
        x, _ = ops.text_embed(h.to(dev, non_blocking=True), p["table"], self._pos(p, L, dev))
        return x.view(B, L, self.model_dim)

    def forward_embedding(self, text_tokens: torch.Tensor) -> torch.Tensor:
        return self.embed_tokens(text_tokens)

    @torch.no_grad()
    def encode_tokens(self, x: torch.Tensor):
        """The transformer + final LayerNorm on embeddings x [B, L, C] fp32 CUDA -> (fp32 [B*L, C], bf16 [B*L, C])."""
        check_native(self, "MobileCLIPTextTransformer", self.training)
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 3 and x.shape[2] == self.model_dim):
            raise ValueError(f"expected CUDA fp32 embeddings [B, L, {self.model_dim}]; the native path has no CPU fallback")
        B, L, C = x.shape
        p = self._plan()
        xs = run_layers(p["layers"], x.reshape(B * L, C).contiguous(), B, L, self.causal_masking)
        yb, yf = ops.layernorm(xs, *p["ln"], out_bf16=True, out_f32=True)
        return yf, yb

    def encode_text(self, text, key_padding_mask=None, return_all_tokens=False, input_is_embeddings=False, *args, **kwargs):
        if key_padding_mask is not None:
            raise NotImplementedError("MobileCLIPTextTransformer: key_padding_mask is not supported on the native path (no "
                                      "caller passes one: TextStudentEncoder attends over padding tokens)")
        check_native(self, "MobileCLIPTextTransformer", self.training)
        ids = None
        if input_is_embeddings:
            emb = text
        else:
            ids = host_ids(text, self.vocab_size)
            emb = self.embed_tokens(ids)
        B, L, C = emb.shape
        yf, yb = self.encode_tokens(emb)
        if return_all_tokens:
            return yf.view(B, L, C)
        # pooled: EOT token (argmax of the ids) or, for embeddings, the last token (mobile_clip.py:873-882)
        rows = torch.arange(B) * L + (ids.argmax(dim=-1) if ids is not None else L - 1)
        pooled = yb.index_select(0, rows.to(yb.device)).contiguous()
        with torch.no_grad():
            return ops.gemm(pooled, self._plan()["proj"], out_dtype=torch.float32)

    def forward(self, text_tokens, key_padding_mask=None, return_all_tokens=False, input_is_embeddings=False, *args, **kwargs):
        return self.encode_text(text_tokens, key_padding_mask=key_padding_mask, return_all_tokens=return_all_tokens,
                                input_is_embeddings=input_is_embeddings)
