"""Oracle: the text encoders (MobileCLIP students, SAM3 text teacher) -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).

Functional fp32 restatement driven by reference-keyed state_dicts, on token ids (the tokenizer is tested separately):
  LearnablePositionalEmbedding.forward     sam3/sam3/backbones/mobile_clip.py:305-317 (bilinear resize when L != N)
  MultiHeadAttention._forward_impl          mobile_clip.py:373-408 (q * scale, additive causal mask, softmax in fp32)
  TransformerEncoder.forward                mobile_clip.py:469-491 (pre-norm, residual)
  MobileOneBlock / RepMixer / ConvFFN       mobile_clip.py:121-138, 535-603 (BN eval, 1x11 depthwise, no scale branch)
  RepMixerBlock.forward                     mobile_clip.py:685-702 on [B, C, 1, L]
  MobileCLIPTextTransformer.encode_text     mobile_clip.py:815-883 (forward_embedding without embed_scale; argmax pooling)
  TextStudentEncoder.forward                sam3/sam3/model/text_encoder_student.py:40-58
  VETextEncoder / TextTransformer           sam3/sam3/model/text_encoder_ve.py:13-145, 228-250, 286-328 (causal, ln_final,
                                            resizer; the discarded pooled projection is skipped)
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def _ln(x, sd, p, eps=1e-5):
    return F.layer_norm(x, x.shape[-1:], sd[p + ".weight"], sd[p + ".bias"], eps)


def _lin(x, sd, p):
    return F.linear(x, sd[p + ".weight"], sd.get(p + ".bias"))


def _bn(x, sd, p, eps=1e-5):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False, 0.0, eps)


def causal_mask(L, device=None):
    return torch.full((L, L), float("-inf"), device=device).triu_(1)


def mha(x, w_qkv, b_qkv, w_o, b_o, heads, mask=None):
    B, L, C = x.shape
    qkv = F.linear(x, w_qkv, b_qkv).reshape(B, L, 3, heads, -1).transpose(1, 3)   # [B, heads, 3, L, d]
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    q = q * (C // heads) ** -0.5
    a = q @ k.transpose(-1, -2)
    if mask is not None:
        a = a + mask
    a = torch.softmax(a.float(), dim=-1)
    return F.linear((a @ v).transpose(1, 2).reshape(B, L, C), w_o, b_o)


def transformer_encoder(x, sd, p, heads, mask):
    y = _ln(x, sd, p + ".pre_norm_mha.0")
    x = x + mha(y, sd[p + ".pre_norm_mha.1.qkv_proj.weight"], sd[p + ".pre_norm_mha.1.qkv_proj.bias"],
                sd[p + ".pre_norm_mha.1.out_proj.weight"], sd[p + ".pre_norm_mha.1.out_proj.bias"], heads, mask)
    y = F.gelu(_lin(_ln(x, sd, p + ".pre_norm_ffn.0"), sd, p + ".pre_norm_ffn.1"))
    return x + _lin(y, sd, p + ".pre_norm_ffn.4")


def _dw(x, w):
    return F.conv2d(x, w, None, 1, (0, w.shape[-1] // 2), 1, x.shape[1])


def repmixer_block(x, sd, p):
    """x [B, L, C] -> [B, L, C]."""
    t = x.permute(0, 2, 1).unsqueeze(2)                       # [B, C, 1, L]
    tm = p + ".token_mixer"
    mixer = _bn(t, sd, tm + ".mixer.rbr_skip") + _bn(_dw(t, sd[tm + ".mixer.rbr_conv.0.conv.weight"]), sd, tm + ".mixer.rbr_conv.0.bn")
    norm = _bn(t, sd, tm + ".norm.rbr_skip")
    t = t + sd[tm + ".layer_scale"] * (mixer - norm)
    f = p + ".convffn"
    u = _bn(_dw(t, sd[f + ".conv.conv.weight"]), sd, f + ".conv.bn")
    u = F.conv2d(F.gelu(F.conv2d(u, sd[f + ".fc1.weight"], sd[f + ".fc1.bias"])), sd[f + ".fc2.weight"], sd[f + ".fc2.bias"])
    t = t + sd[p + ".layer_scale"] * u
    return t.squeeze(2).permute(0, 2, 1)


def pos_table(pe, L):
    """pe [1, 1, N, D] -> [L, D]."""
    if L != pe.shape[2]:
        pe = F.interpolate(pe, size=(L, pe.shape[3]), mode="bilinear")
    return pe.reshape(L, pe.shape[3])


def mobileclip_embed(sd, ids, prefix="encoder."):
    emb = F.embedding(ids, sd[prefix + "embedding_layer.weight"])
    key = prefix + "positional_embedding.pos_embed.pos_embed"
    return emb + pos_table(sd[key], ids.shape[1]) if key in sd else emb


def mobileclip_encode(sd, x, cfg, prefix="encoder."):
    """Embeddings [B, L, C] -> final-LayerNorm tokens [B, L, C]."""
    mask = causal_mask(x.shape[1], x.device) if cfg["causal_masking"] else None
    n = cfg["n_transformer_layers"] + (2 if cfg["model_name"] == "mct" else 0)
    for i in range(n):
        p = f"{prefix}transformer.{i}"
        if p + ".token_mixer.layer_scale" in sd:
            x = repmixer_block(x, sd, p)
        else:
            x = transformer_encoder(x, sd, p, cfg["n_heads_per_layer"], mask)
    return _ln(x, sd, prefix + "final_layer_norm")


def mobileclip_pooled(sd, ids, cfg, prefix="encoder."):
    """MobileCLIPTextTransformer.forward(ids) (return_all_tokens=False): EOT token (argmax id) @ projection_layer."""
    y = mobileclip_encode(sd, mobileclip_embed(sd, ids, prefix), cfg, prefix)
    return y[torch.arange(ids.shape[0]), ids.argmax(dim=-1)] @ sd[prefix + "projection_layer"]


def text_student(sd, ids, cfg):
    """TextStudentEncoder.forward on ids -> (mask [B,L], memory [L,B,out], input_embeds [L,B,dim])."""
    emb = mobileclip_embed(sd, ids)
    mem = _lin(mobileclip_encode(sd, emb, cfg), sd, "projector")
    return (ids != 0).ne(True), mem.transpose(0, 1), emb.transpose(0, 1)


def ve_text_encoder(sd, ids, heads, prefix=""):
    """VETextEncoder.forward on ids -> (mask, memory [L,B,d_model], inputs_embeds [L,B,width])."""
    e = prefix + "encoder."
    L = ids.shape[1]
    emb = F.embedding(ids, sd[e + "token_embedding.weight"])
    x = emb + sd[e + "positional_embedding"][:L]
    mask = causal_mask(L, x.device)
    i = 0
    while f"{e}transformer.resblocks.{i}.ln_1.weight" in sd:
        p = f"{e}transformer.resblocks.{i}"
        x = x + mha(_ln(x, sd, p + ".ln_1"), sd[p + ".attn.in_proj_weight"], sd[p + ".attn.in_proj_bias"],
                    sd[p + ".attn.out_proj.weight"], sd[p + ".attn.out_proj.bias"], heads, mask)
        x = x + _lin(F.gelu(_lin(_ln(x, sd, p + ".ln_2"), sd, p + ".mlp.c_fc")), sd, p + ".mlp.c_proj")
        i += 1
    mem = _lin(_ln(x, sd, e + "ln_final").transpose(0, 1), sd, prefix + "resizer")
    return (ids != 0).ne(True), mem, emb.transpose(0, 1)


def flops_mobileclip(cfg, B, L, out_dim):
    """Algorithmic FLOPs (2 per multiply-add) of TextStudentEncoder.forward from shapes."""
    C = cfg["dim"]
    F_ = int(math.ceil(C * cfg["ffn_multiplier_per_layer"] / 16.0) * 16)
    M = B * L
    per_attn = 2 * M * C * 3 * C + 2 * M * C * C + 2 * 2 * B * L * L * C + 2 * 2 * M * C * F_
    n = cfg["n_transformer_layers"] * per_attn
    if cfg["model_name"] == "mct":
        n += 2 * (2 * 2 * M * C * 11 + 2 * 2 * M * C * 4 * C)
    return n + 2 * M * C * out_dim


def flops_ve(width, layers, B, L, d_model=256):
    M = B * L
    return layers * (2 * M * width * 4 * width + 2 * 2 * B * L * L * width + 2 * 2 * M * width * 4 * width) + 2 * M * width * d_model
