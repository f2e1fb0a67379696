"""MobileCLIP text transformer (the stage-1 text students), H100-native.  Mirrors `sam3/sam3/backbones/mobile_clip.py`:
same class names, constructor arguments and state_dict keys (`embedding_layer.weight`,
`positional_embedding.pos_embed.pos_embed`, `transformer.N.pre_norm_mha.{0,1.qkv_proj,1.out_proj}.*`,
`transformer.N.pre_norm_ffn.{0,1,4}.*`, the RepMixerBlock's `token_mixer.{norm,mixer}.*`, `convffn.*`, `layer_scale`,
`final_layer_norm.*`, `projection_layer`).  The nn modules are parameter containers.  Eval-mode forward for every student;
train-mode forward + backward for the base (TransformerEncoder-only) students and for MobileCLIP-S0 with its RepMixerBlocks'
BatchNorms frozen in .eval() or, after enable_batch_stat_bn(), in train mode (batch statistics): TextStudentTrainGraph at the end of
this file.

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

from .. import ops, sync_bn
from ..nn_utils import NativePlanMixin, StagedGraphMixin, bn_scale_bias, cached_pack


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


def repmixer_fold(blk: RepMixerBlock):
    """The RepMixerBlock's token mixer and ConvFFN conv with their BatchNorms' running statistics folded into es3_repmixer_bf16's
    taps (mobile_clip.py:594-702): x1 = x + ls (BN_ms(x) + BN_mc(conv(x)) - BN_ns(x)) = sum_k wm[k] x[l+k-5] + bm,
    u = BN_f(conv_f(x1)) = sum_k wf[k] x1[l+k-5] + bf.  Also returns the layer scales ls (token mixer) and lsb (block), fp32 [C]."""
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
    return dict(wm=wm.contiguous(), bm=bm, wf=_taps(ffn.conv.conv, s_f), bf=b_f.contiguous(), ls=ls.contiguous(),
                lsb=lsb.contiguous())


def repmixer_plan(blk: RepMixerBlock):
    """Eval-mode RepMixerBlock: the folded taps (repmixer_fold) and the two GEMMs, out = x1 + ls_blk (fc2(gelu(fc1(u))))."""
    ffn = blk.convffn
    f = repmixer_fold(blk)
    lsb = f["lsb"]
    w1 = ffn.fc1.weight.detach().reshape(ffn.fc1.out_channels, -1).to(torch.bfloat16).contiguous()
    w2 = ffn.fc2.weight.detach().reshape(ffn.fc2.out_channels, -1).to(torch.bfloat16).contiguous()
    return dict(kind="repmixer", wm=f["wm"], bm=f["bm"], wf=f["wf"], bf=f["bf"],
                fc1=(w1, _f32(ffn.fc1.bias)), fc2=(w2, lsb, (lsb * _f32(ffn.fc2.bias)).contiguous()))


def repmixer_bns(blk: RepMixerBlock):
    """The block's four BatchNorms in the kernels' order: BN_ms (mixer.rbr_skip), BN_mc (mixer.rbr_conv.0.bn), BN_ns
    (norm.rbr_skip), BN_f (convffn.conv.bn)."""
    tm = blk.token_mixer
    return (tm.mixer.rbr_skip, tm.mixer.rbr_conv[0].bn, tm.norm.rbr_skip, blk.convffn.conv.bn)


def repmixer_bn_pack(blk: RepMixerBlock):
    """The parameters es3_repmixer_bn_* read, cached until the next optimiser step: taps [2, 11, C] (raw w_mc, w_f), aff [9, C]
    (ls_tm, then gamma / beta of repmixer_bns), and fc2's layer scale / bias.  No running statistics: they change every forward."""
    tm, ffn = blk.token_mixer, blk.convffn

    def build():
        one = torch.ones(tm.dim, device=blk.layer_scale.device)
        aff = [_f32(tm.layer_scale).reshape(-1)] + [_f32(t) for bn in repmixer_bns(blk) for t in (bn.weight, bn.bias)]
        lsb, b2 = _f32(blk.layer_scale).reshape(-1), _f32(ffn.fc2.bias)
        return dict(taps=torch.stack([_taps(tm.mixer.rbr_conv[0].conv, one), _taps(ffn.conv.conv, one)]).contiguous(),
                    aff=torch.stack(aff).contiguous(), lsb=lsb.contiguous(), b2=b2, b2s=(lsb * b2).contiguous())
    return cached_pack(blk, "bn_train", blk.layer_scale, build)


def repmixer_bn_forward(blk: RepMixerBlock, x, B, L):
    """The block's prologue with batch-statistics BatchNorm (updates its running buffers): (x1 fp32, u bf16, stats [8, C], pack,
    sync).  sync is None for per-rank statistics; when the block's SyncBatchNorms span several ranks (sync_bn.repmixer_sync_group)
    the statistics are taken over every rank -- es3_repmixer_bn_fwd split at its two finalize points, each rank's (count, mean, M2)
    all-gathered -- and sync = (exchange group, the group's token count) for the backward."""
    p = repmixer_bn_pack(blk)
    bns = repmixer_bns(blk)
    group = sync_bn.repmixer_sync_group(bns)
    if group is None:
        x1, u, _, stats = ops.repmixer_bn_fwd(x, B, L, p["taps"], p["aff"], bns)
        return x1, u, stats, p, None
    group = sync_bn.exchange_group(group, x.is_cuda)
    C = x.shape[1]
    fold = torch.empty((24, C), device=x.device, dtype=torch.float32)
    stats = torch.empty((8, C), device=x.device, dtype=torch.float32)
    taps, aff = p["taps"], p["aff"]
    parts = sync_bn.all_gather_partials(ops.repmixer_bn_stats_partial(x, B, L, taps, fold, 0), group)     # x and c = dw(x)
    total = ops.repmixer_bn_finalize_sync(parts, 0, taps, aff, bns, fold, stats)
    parts = sync_bn.all_gather_partials(ops.repmixer_bn_stats_partial(x, B, L, taps, fold, 1), group)     # f = dw(x1)
    ops.repmixer_bn_finalize_sync(parts, 1, taps, aff, bns, fold, stats)
    x1, u = ops.repmixer(x, B, L, fold[:11], fold[11], fold[12:23], fold[23])
    return x1, u, stats, p, (group, total)


def invalidate_running_folds(enc: "MobileCLIPTextTransformer"):
    """Drop every cached fold of the RepMixerBlocks' running statistics (the eval plan and RepMixerUnit's train_fold).  The
    batch-statistics kernels write the running buffers in place, which torch's _version does not see."""
    enc._plan_key = None
    for b in enc.transformer:
        if isinstance(b, RepMixerBlock):
            b.__dict__.get("_es3_pack_cache", {}).pop("train_fold", None)


def run_layers(layers, x, B, L, causal, bn_blocks=None):
    """The residual trunk on x [B*L, C] fp32 (not modified) -> fp32 [B*L, C].  bn_blocks: the trunk's modules when the
    RepMixerBlocks normalise with batch statistics (their running buffers are updated), else None."""
    C = x.shape[1]
    for i, lp in enumerate(layers):
        if lp["kind"] == "repmixer":
            if bn_blocks is not None:
                x1, u, _, _, _ = repmixer_bn_forward(bn_blocks[i], x, B, L)
            else:
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
        raise NotImplementedError(f"{what}: this module's native path is eval-mode (forward) only; training is built for "
                                  "TextStudentEncoder with a TransformerEncoder (base) trunk.  Call .eval() first.")
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


class MobileCLIPTextTransformer(nn.Module, NativePlanMixin, StagedGraphMixin):
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
        # train-mode RepMixerBlock BatchNorms normalise with batch statistics (TextStudentEncoder.enable_batch_stat_bn); not state
        self.batch_stat_bn = False

    def batch_stat_active(self) -> bool:
        """True when the RepMixerBlocks' BatchNorms are in train mode and batch statistics were asked for (check_trainable
        rejects a mixed train / eval state before this is consulted)."""
        return self.batch_stat_bn and any(m.training for b in self.transformer if isinstance(b, RepMixerBlock)
                                          for m in repmixer_bns(b))

    def batch_stat_synced(self) -> bool:
        """True when the RepMixerBlocks' batch statistics are taken over several ranks (SyncBatchNorm, sync_bn.sync_group)."""
        return any(sync_bn.repmixer_sync_group(repmixer_bns(b)) is not None for b in self.transformer if isinstance(b, RepMixerBlock))

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
        check_native(self, "MobileCLIPTextTransformer", self.training)
        return self._embed(ids)

    def _embed(self, ids):
        h = host_ids(ids, self.vocab_size)
        return self._embed_ids(h.to(next(self.parameters()).device, non_blocking=True))

    def _embed_ids(self, ids):
        """The embedding of ids [B, L] int64 already on the device (validated on the host) -> fp32 [B, L, C]."""
        p = self._plan()
        B, L = ids.shape
        x, _ = ops.text_embed(ids, p["table"], self._pos(p, L, ids.device))
        return x.view(B, L, self.model_dim)

    def forward_embedding(self, text_tokens: torch.Tensor) -> torch.Tensor:
        return self.embed_tokens(text_tokens)

    @torch.no_grad()
    def encode_tokens(self, x: torch.Tensor):
        """The transformer + final LayerNorm on embeddings x [B, L, C] fp32 CUDA -> (fp32 [B*L, C], bf16 [B*L, C])."""
        check_native(self, "MobileCLIPTextTransformer", self.training)
        return self._encode(x)

    def _check_embeddings(self, x):
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 3 and x.shape[2] == self.model_dim):
            raise ValueError(f"expected CUDA fp32 embeddings [B, L, {self.model_dim}]; the native path has no CPU fallback")

    def _encode(self, x):
        self._check_embeddings(x)
        B, L, C = x.shape
        p = self._plan()
        bn_blocks = list(self.transformer) if self.batch_stat_active() else None
        xs = run_layers(p["layers"], x.reshape(B * L, C).contiguous(), B, L, self.causal_masking, bn_blocks)
        if bn_blocks is not None:
            invalidate_running_folds(self)
        yb, yf = ops.layernorm(xs, *p["ln"], out_bf16=True, out_f32=True)
        return yf, yb

    def encode_text(self, text, key_padding_mask=None, return_all_tokens=False, input_is_embeddings=False, *args, **kwargs):
        return self._encode_text(text, key_padding_mask, return_all_tokens, input_is_embeddings, self._graphs is not None)

    @torch.no_grad()
    def _encode_text(self, text, key_padding_mask, return_all_tokens, input_is_embeddings, graphed):
        if key_padding_mask is not None:
            raise NotImplementedError("MobileCLIPTextTransformer: key_padding_mask is not supported on the native path (no "
                                      "caller passes one: TextStudentEncoder attends over padding tokens)")
        dev = check_native(self, "MobileCLIPTextTransformer", self.training)
        # on the host: the ids validated and the pooled rows built (EOT token = argmax of the ids or, for embeddings, the last
        # token, mobile_clip.py:873-882); _encode_on_device runs on device copies of them
        if input_is_embeddings:
            self._check_embeddings(text)
            B, L, _ = text.shape
            host, dev_in, eot = [], [text], L - 1
        else:
            ids = host_ids(text, self.vocab_size)
            B, L = ids.shape
            host, dev_in, eot = [ids], [], ids.argmax(dim=-1)
        if not return_all_tokens:
            host.append(torch.arange(B) * L + eot)

        def run(*inputs):
            return self._encode_on_device(inputs, input_is_embeddings, return_all_tokens)
        if graphed and not self.batch_stat_active():
            key = (B, L, "embeddings" if input_is_embeddings else "ids", bool(return_all_tokens), dev)
            return self._graphed(key, host, dev_in, run)
        return run(*(h.to(dev, non_blocking=True) for h in host), *dev_in)

    def _encode_on_device(self, inputs, input_is_embeddings, return_all_tokens):
        """inputs: (ids [B, L] | embeddings [B, L, C], then the pooled rows [B] unless return_all_tokens), all on the device ->
        fp32 [B, L, C] (return_all_tokens) or the pooled projection fp32 [B, projection_dim]."""
        if input_is_embeddings:
            emb, rows = inputs[-1], (None if return_all_tokens else inputs[0])
        else:
            emb, rows = self._embed_ids(inputs[0]), (None if return_all_tokens else inputs[1])
        B, L, C = emb.shape
        yf, yb = self._encode(emb)
        if return_all_tokens:
            return yf.view(B, L, C)
        pooled = yb.index_select(0, rows).contiguous()
        return ops.gemm(pooled, self._plan()["proj"], out_dtype=torch.float32)

    def forward(self, text_tokens, key_padding_mask=None, return_all_tokens=False, input_is_embeddings=False, *args, **kwargs):
        return self.encode_text(text_tokens, key_padding_mask=key_padding_mask, return_all_tokens=return_all_tokens,
                                input_is_embeddings=input_is_embeddings)

    def forward_uncaptured(self, text_tokens, key_padding_mask=None, return_all_tokens=False, input_is_embeddings=False):
        """forward() launched kernel by kernel, whether or not CUDA graphs are enabled."""
        return self._encode_text(text_tokens, key_padding_mask, return_all_tokens, input_is_embeddings, False)


# ----------------------------------------------------------------------------------------------- training graph (base trunk)
# Train-mode forward + backward of the base students (TransformerEncoder layers only), in the scheme of tinyvit_train.py: units
# with forward(x) / backward(d, grads), wrapped into ONE autograd node by model.text_encoder_student.TextStudentTrainFunction.
# The residual stream and its gradient are fp32 ([B*L, C]); GEMM operands are bf16 with fp32 accumulation.
#   embedding + positional table        es3_text_embed (+ es3_text_pos_resize); grads es3_text_embed_grad, es3_text_pos_grad
#   LayerNorm                           es3_layernorm_f32 / es3_layernorm_bwd_f32 (fp32 dx + the residual gradient, bf16 copy)
#   nn.Linear (+ GELU)                  es3_gemm_bf16_ex [+ es3_affine_act]; grads es3_wgrad_pw, column sums / es3_bn_act_bwd_*,
#                                       es3_gemm_bf16_ex on the cached W^T (nn_utils.cached_pack, invalidated by each optimiser step)
#   attention                           es3_attention_bf16 | es3_attention_causal_bf16 / es3_text_attn_bwd
#   RepMixerBlock (frozen BatchNorm)    es3_repmixer_bf16 + fc1 / fc2 GEMMs; es3_repmixer_ls_bwd, es3_repmixer_ffn_bwd,
#                                       es3_repmixer_tm_bwd (RepMixerUnit)
#   RepMixerBlock (batch-statistics BN) es3_repmixer_bn_fwd + fc1 / fc2 GEMMs; es3_repmixer_ls_bwd, es3_repmixer_bn_ffn_bwd,
#                                       es3_repmixer_bn_tm_bwd (RepMixerBatchStatUnit)
def _grad_of(grads, p):
    from .efficientvit_train import _grad_of as g
    return g(grads, p)


def check_trainable(module: nn.Module, enc: "MobileCLIPTextTransformer", what: str):
    """The raise paths of the training graph: S0-style RepMixerBlocks with a BatchNorm in train mode unless batch statistics were
    enabled (then: a mixed train / eval state, momentum=None, track_running_stats=False), strict precision, CPU modules,
    dropout > 0.  nn.SyncBatchNorm (convert_sync_batchnorm) is a _BatchNorm but not a BatchNorm2d: both follow the same rules."""
    bns = [m for b in enc.transformer if isinstance(b, RepMixerBlock) for m in b.modules()
           if isinstance(m, nn.modules.batchnorm._BatchNorm)]
    if any(m.training for m in bns):
        if not enc.batch_stat_bn:
            raise NotImplementedError(f"{what}: the RepMixerBlocks of MobileCLIP-S0 train with frozen BatchNorm (running "
                                      "statistics) unless batch statistics are enabled.  To train, put every BatchNorm in .eval() "
                                      "after .train() (set_bn_state with TRAIN.EVAL_BN_WHEN_TRAINING does) or call "
                                      "enable_batch_stat_bn() to normalise with batch statistics; for inference, Call .eval() first.")
        if not all(m.training for m in bns):
            raise NotImplementedError(f"{what}: batch-statistics BatchNorm needs every BatchNorm of the RepMixerBlocks in train mode; "
                                      "a mixed train / eval state is not built (set_bn_state freezes all of them)")
        for m in bns:
            if m.momentum is None:
                raise NotImplementedError(f"{what}: BatchNorm momentum=None (a cumulative moving average) is not built for "
                                          "batch-statistics BatchNorm")
            if not m.track_running_stats or m.running_mean is None:
                raise NotImplementedError(f"{what}: batch-statistics BatchNorm is built with track_running_stats=True only")
        for b in enc.transformer:
            if isinstance(b, RepMixerBlock):
                sync_bn.repmixer_sync_group(repmixer_bns(b))     # raises when a block's BNs disagree on their process group
    if ops.precision() == "strict":
        raise NotImplementedError(f"{what}: the strict (fp32) precision mode is not built for the text encoders")
    for m in module.modules():
        if isinstance(m, nn.Dropout) and m.p > 0:
            raise NotImplementedError(f"{what}: dropout p={m.p} in train mode is not built (every shipped text student uses p = 0)")
    p = next(module.parameters())
    if not p.is_cuda:
        raise RuntimeError(f"{what}: the module is on {p.device}; the native path runs on a CUDA device and has no CPU fallback")
    return p.device


class _TextLinear:
    """nn.Linear [+ GELU] on [M, K] bf16 rows."""

    def __init__(self, lin: nn.Linear, act=None):
        self.lin, self.act = lin, act
        self.saved = None

    def _w(self):
        lin = self.lin
        return cached_pack(lin, "text_w", lin.weight, lambda: lin.weight.detach().to(torch.bfloat16).contiguous())

    def _wt(self):
        lin = self.lin
        return cached_pack(lin, "text_wt", lin.weight, lambda: lin.weight.detach().to(torch.bfloat16).t().contiguous())

    def forward(self, x2, residual=None, out_dtype=torch.bfloat16):
        b = self.lin.bias.detach().float().contiguous()
        if self.act is None:
            self.saved = (x2, None, b)
            return ops.gemm(x2, self._w(), bias=b, residual=residual, out_dtype=out_dtype)
        z = ops.gemm(x2, self._w())
        self.saved = (x2, z, b)
        return ops.affine_act(z, None, b, self.act)

    def backward(self, dy, grads, dy_f32=None, out_dtype=torch.bfloat16):
        """dy: bf16 gradient of the output (dy_f32: the same in fp32, for the bias sum).  Returns the input gradient."""
        x2, z, b = self.saved
        self.saved = None
        lin = self.lin
        gb = _grad_of(grads, lin.bias)
        if z is None:
            dz = dy
            if gb is not None:
                if dy_f32 is not None:
                    ops.colsum_f32(dy_f32, gb)
                else:
                    ops.bn_act_bwd(dz, dz, None, None, None, "none", dbeta=gb, apply=False)
        else:
            dz = ops.bn_act_bwd(dy, z, None, b, self.act, "none", dbeta=gb)
        gw = _grad_of(grads, lin.weight)
        if gw is not None:
            ops.wgrad_pw(dz, x2, gw)
        return ops.gemm(dz, self._wt(), out_dtype=out_dtype)


class _TextConv1x1(_TextLinear):
    """A 1x1 nn.Conv2d (ConvFFN.fc1 / fc2, weight [N, K, 1, 1]) as _TextLinear on [M, K] bf16 rows."""

    def _w(self):
        lin = self.lin
        return cached_pack(lin, "text_w", lin.weight,
                           lambda: lin.weight.detach().reshape(lin.out_channels, -1).to(torch.bfloat16).contiguous())

    def _wt(self):
        lin = self.lin
        return cached_pack(lin, "text_wt", lin.weight,
                           lambda: lin.weight.detach().reshape(lin.out_channels, -1).to(torch.bfloat16).t().contiguous())


def _ln_params(ln):
    return ln.weight.detach().float().contiguous(), ln.bias.detach().float().contiguous(), ln.eps


class TextEncoderLayerUnit:
    """TransformerEncoder (mobile_clip.py:469-491): x1 = x + out_proj(attn(qkv(LN1(x)))); x2 = x1 + fc2(gelu(fc1(LN2(x1))))."""

    wants_bf16_grad = True      # fc2's backward takes the bf16 copy of the output gradient

    def __init__(self, blk: TransformerEncoder, causal: bool):
        self.n1, at, self.n2 = blk.pre_norm_mha[0], blk.pre_norm_mha[1], blk.pre_norm_ffn[0]
        if at.head_dim != 64:
            raise NotImplementedError(f"text attention backward is built for head_dim 64, got {at.head_dim}")
        self.heads, self.scale, self.causal = at.num_heads, at.scaling, causal
        self.qkv, self.proj = _TextLinear(at.qkv_proj), _TextLinear(at.out_proj)
        self.fc1, self.fc2 = _TextLinear(blk.pre_norm_ffn[1], "gelu"), _TextLinear(blk.pre_norm_ffn[4])
        self.saved = None

    def forward(self, x, B, L):
        C = x.shape[1]
        y1, _ = ops.layernorm(x, *_ln_params(self.n1))
        qkv = self.qkv.forward(y1)
        if self.causal:
            a = ops.attention_causal(qkv, B, L, C, self.heads, self.scale)
        else:
            a = ops.attention(qkv, B, 1, L, C, self.heads, 0, self.scale)
        x1 = self.proj.forward(a, residual=x, out_dtype=torch.float32)
        y2, _ = ops.layernorm(x1, *_ln_params(self.n2))
        x2 = self.fc2.forward(self.fc1.forward(y2), residual=x1, out_dtype=torch.float32)
        self.saved = (x, x1, qkv, a, B, L)
        return x2

    def backward(self, g, gb, grads, want_bf16=True):
        """g: fp32 gradient of the layer output, gb: its bf16 copy -> (fp32 input gradient, bf16 copy | None)."""
        x, x1, qkv, a, B, L = self.saved
        self.saved = None
        C = x.shape[1]
        dh = self.fc2.backward(gb, grads, dy_f32=g)
        dy2 = self.fc1.backward(dh, grads, out_dtype=torch.float32)
        w2, _, eps2 = _ln_params(self.n2)
        g1, g1b = ops.layernorm_bwd_f32(x1, dy2, w2, eps2, _grad_of(grads, self.n2.weight), _grad_of(grads, self.n2.bias), dres=g,
                                        want_bf16=True)
        da = self.proj.backward(g1b, grads, dy_f32=g1)
        dqkv = ops.text_attn_bwd(qkv, a, da, B, L, C, self.heads, self.scale, self.causal)
        dy1 = self.qkv.backward(dqkv, grads, out_dtype=torch.float32)
        w1, _, eps1 = _ln_params(self.n1)
        return ops.layernorm_bwd_f32(x, dy1, w1, eps1, _grad_of(grads, self.n1.weight), _grad_of(grads, self.n1.bias), dres=g1,
                                     want_bf16=want_bf16)


def _bn_rows(bn: nn.BatchNorm2d):
    """A frozen BatchNorm2d as fp32 [4, C]: scale and shift (as folded for the forward), running mean, 1 / sqrt(running var + eps)."""
    s, b = _bn(bn)
    return torch.stack([s, b, _f32(bn.running_mean), torch.rsqrt(_f32(bn.running_var) + bn.eps)])


class RepMixerUnit:
    """RepMixerBlock (mobile_clip.py:594-702) with frozen BatchNorm (every BN in .eval(): running statistics, so the block is its
    eval function).  Forward: es3_repmixer_bf16 on the taps folded from the current parameters (repmixer_fold, cached until the
    next optimiser step), fc1 + GELU, fc2 x layer scale + residual.  Backward (repmixer_bwd.cu): fc2's output y is recomputed in
    fp32 from the saved hidden h (deriving it as (x2 - x1) / ls_blk would scale x1's rounding by 1 / ls_blk, 1e5 at init);
    es3_repmixer_ls_bwd -> fc2 / GELU / fc1 backward -> es3_repmixer_ffn_bwd -> es3_repmixer_tm_bwd.  The BatchNorms' running
    statistics and num_batches_tracked are read, never written."""

    wants_bf16_grad = False     # the backward reads the fp32 output gradient only

    def __init__(self, blk: RepMixerBlock):
        tm = blk.token_mixer
        if not (blk.use_layer_scale and tm.use_layer_scale):
            raise NotImplementedError("RepMixerBlock training is built for the layer-scaled block of MobileCLIP-S0")
        self.blk, self.tm, self.ffn = blk, tm, blk.convffn
        self.fc1, self.fc2 = _TextConv1x1(self.ffn.fc1, "gelu"), _TextConv1x1(self.ffn.fc2)
        self.saved = None

    def _pack(self):
        blk, tm, ffn = self.blk, self.tm, self.ffn

        def build():
            p = repmixer_fold(blk)
            one = torch.ones_like(p["ls"])
            p["bnp"] = torch.cat([_bn_rows(tm.mixer.rbr_skip), _bn_rows(tm.mixer.rbr_conv[0].bn), _bn_rows(tm.norm.rbr_skip),
                                  p["ls"].view(1, -1)]).contiguous()
            p["bnf"] = _bn_rows(ffn.conv.bn).contiguous()
            p["tm_taps"], p["f_taps"] = _taps(tm.mixer.rbr_conv[0].conv, one), _taps(ffn.conv.conv, one)
            p["b2"] = _f32(ffn.fc2.bias)
            p["b2s"] = (p["lsb"] * p["b2"]).contiguous()
            return p
        return cached_pack(blk, "train_fold", blk.layer_scale, build)

    def prologue(self, x, B, L):
        """(x1 fp32, u bf16, the parameter pack, what the conv + BatchNorm backward needs besides)."""
        p = self._pack()
        return (*ops.repmixer(x, B, L, p["wm"], p["bm"], p["wf"], p["bf"]), p, None)

    def forward(self, x, B, L):
        x1, u, p, bn = self.prologue(x, B, L)
        h = self.fc1.forward(u)
        x2 = ops.gemm(h, self.fc2._w(), scale=p["lsb"], bias=p["b2s"], residual=x1, out_dtype=torch.float32)
        self.saved = (x, x1, h, p, bn, B, L)
        return x2

    def backward(self, g, gb, grads, want_bf16=True):
        """g: fp32 gradient of the block output (gb, its bf16 copy, is not needed) -> (fp32 input gradient, bf16 copy | None)."""
        x, x1, h, p, bn, B, L = self.saved
        self.saved = None
        ffn = self.ffn
        y = ops.gemm(h, self.fc2._w(), bias=p["b2"], out_dtype=torch.float32)
        dy = ops.repmixer_ls_bwd(g, y, p["lsb"], B, L, dls=_grad_of(grads, self.blk.layer_scale),
                                 dbias=_grad_of(grads, ffn.fc2.bias))
        gw2 = _grad_of(grads, ffn.fc2.weight)
        if gw2 is not None:
            ops.wgrad_pw(dy, h, gw2)
        du = self.fc1.backward(ops.gemm(dy, self.fc2._wt()), grads, out_dtype=torch.float32)
        dbn = [_grad_of(grads, t) for b in repmixer_bns(self.blk) for t in (b.weight, b.bias)]
        dst = (_grad_of(grads, ffn.conv.conv.weight), _grad_of(grads, self.tm.mixer.rbr_conv[0].conv.weight),
               _grad_of(grads, self.tm.layer_scale), dbn)
        return self.conv_bn_backward(x, x1, du, g, p, bn, B, L, dst, want_bf16)

    def conv_bn_backward(self, x, x1, du, g, p, bn, B, L, dst, want_bf16):
        """The two depthwise convs and their BatchNorms: du (fc1's input gradient) and g -> the block's input gradient.  dst: the
        gradients of the ConvFFN taps, the token-mixer taps, its layer scale and (gamma, beta) x (BN_ms, BN_mc, BN_ns, BN_f)."""
        d_ftaps, d_mtaps, d_ls, dbn = dst
        e = ops.repmixer_ffn_bwd(x1, du, g, p["f_taps"], p["bnf"], B, L, dtaps=d_ftaps, dgamma=dbn[6], dbeta=dbn[7])
        return ops.repmixer_tm_bwd(x, e, p["tm_taps"], p["bnp"], B, L, dtaps=d_mtaps, dls=d_ls, dbn=dbn[:6], want_bf16=want_bf16)


class RepMixerBatchStatUnit(RepMixerUnit):
    """RepMixerBlock with every BatchNorm in train mode (batch statistics, as nn.BatchNorm2d trains; enable_batch_stat_bn).
    Forward: es3_repmixer_bn_fwd (statistics over the B*L tokens, running buffers and num_batches_tracked updated on the device,
    taps folded on the device, then es3_repmixer_bf16), fc1 + GELU, fc2 x layer scale + residual; the batch statistics are kept
    for the backward.  Backward: as RepMixerUnit, with es3_repmixer_bn_ffn_bwd / es3_repmixer_bn_tm_bwd, which add the two
    mean terms of the BatchNorm input gradient."""

    def __init__(self, blk: RepMixerBlock, enc: "MobileCLIPTextTransformer"):
        super().__init__(blk)
        self.enc = enc

    def prologue(self, x, B, L):
        x1, u, stats, p, sync = repmixer_bn_forward(self.blk, x, B, L)
        invalidate_running_folds(self.enc)
        return x1, u, p, (stats, sync)

    def conv_bn_backward(self, x, x1, du, g, p, bn, B, L, dst, want_bf16):
        (stats, sync), (d_ftaps, d_mtaps, d_ls, dbn), taps, aff = bn, dst, p["taps"], p["aff"]
        if sync is None:
            e = ops.repmixer_bn_ffn_bwd(x1, du, g, taps, aff, stats, B, L, dtaps=d_ftaps, dgamma=dbn[6], dbeta=dbn[7])
            return ops.repmixer_bn_tm_bwd(x, e, taps, aff, stats, B, L, dtaps=d_mtaps, dls=d_ls, dbn=dbn[:6], want_bf16=want_bf16)
        # synchronised: each BN sum is all-gathered and added in rank order; the BNs' gamma / beta gradients stay this rank's own
        group, total = sync
        sums = ops.repmixer_bn_ffn_sums(x1, du, taps, stats, B, L, aff, dgamma=dbn[6], dbeta=dbn[7])
        e = ops.repmixer_bn_ffn_apply(x1, du, g, taps, aff, stats, sync_bn.all_gather_partials(sums, group), total, B, L, dtaps=d_ftaps)
        sums = ops.repmixer_bn_tm_sums(x, e, taps, aff, stats, B, L, dbn=dbn[:6])
        return ops.repmixer_bn_tm_apply(x, e, taps, aff, stats, sync_bn.all_gather_partials(sums, group), total, B, L, dtaps=d_mtaps,
                                        dls=d_ls, want_bf16=want_bf16)


class TextEmbedUnit:
    """forward_embedding (mobile_clip.py:815-823): table[ids] + the positional table, resized N -> L when they differ."""

    def __init__(self, enc: "MobileCLIPTextTransformer"):
        self.emb = enc.embedding_layer
        self.lpe = enc.positional_embedding.pos_embed if enc.positional_embedding is not None else None
        if self.lpe is not None and self.lpe.padding_idx is not None:
            raise NotImplementedError("positional table with a padding_idx is not on the text students' path")
        self.saved = None

    def forward(self, ids_host, dev):
        B, L = ids_host.shape
        table = self.emb.weight.detach()
        pos = None
        if self.lpe is not None:
            N, C = self.lpe.num_embeddings, self.lpe.embedding_dim
            pos = self.lpe.pos_embed.detach().reshape(N, C)
            if N != L:
                pos = ops.text_pos_resize(pos.contiguous(), L)
        x, _ = ops.text_embed(ids_host.to(dev, non_blocking=True), table.contiguous(), pos)
        # the gradient's token grouping is built now, while the ids are on the host, and copied asynchronously
        plan = ops.embed_grad_plan(ids_host, dev) if self.emb.weight.requires_grad else None
        self.saved = (plan, B, L)
        return x

    def backward(self, dx, grads):
        plan, B, L = self.saved
        self.saved = None
        ge = _grad_of(grads, self.emb.weight)
        if ge is not None:
            ops.text_embed_grad(dx, plan, ge)
        if self.lpe is not None:
            gp = _grad_of(grads, self.lpe.pos_embed)
            if gp is not None:
                ops.text_pos_grad(dx, B, L, gp)


class TextStudentTrainGraph:
    """TextStudentEncoder in train mode: embed -> TransformerEncoder layers (and MobileCLIP-S0's RepMixerBlocks, frozen or
    batch-statistics BN) -> final LayerNorm -> projector (fp32 memory)."""

    def __init__(self, student):
        enc = student.encoder
        self.embed = TextEmbedUnit(enc)
        bstat = enc.batch_stat_active()

        def unit(b):
            if isinstance(b, RepMixerBlock):
                return RepMixerBatchStatUnit(b, enc) if bstat else RepMixerUnit(b)
            return TextEncoderLayerUnit(b, enc.causal_masking)
        self.layers = [unit(b) for b in enc.transformer]
        self.fln = enc.final_layer_norm
        self.proj = _TextLinear(student.projector)
        self.saved = None

    def forward(self, ids_host, dev):
        B, L = ids_host.shape
        x0 = self.embed.forward(ids_host, dev)
        x = x0
        for u in self.layers:
            x = u.forward(x, B, L)
        yb, _ = ops.layernorm(x, *_ln_params(self.fln))
        mem = self.proj.forward(yb, out_dtype=torch.float32)
        self.saved = x
        return mem.view(B, L, -1), x0.view(B, L, -1)

    def backward(self, dmem, grads):
        xs = self.saved
        self.saved = None
        dmem = dmem.reshape(-1, dmem.shape[-1]).contiguous()
        dy = self.proj.backward(ops.cast_f32_to_bf16(dmem), grads, dy_f32=dmem, out_dtype=torch.float32)
        w, _, eps = _ln_params(self.fln)
        g, gb = ops.layernorm_bwd_f32(xs, dy, w, eps, _grad_of(grads, self.fln.weight), _grad_of(grads, self.fln.bias),
                                      want_bf16=bool(self.layers) and self.layers[-1].wants_bf16_grad)
        for i in range(len(self.layers) - 1, -1, -1):
            g, gb = self.layers[i].backward(g, gb, grads, want_bf16=i > 0 and self.layers[i - 1].wants_bf16_grad)
        self.embed.backward(g, grads)
