"""The SAM3 text encoder (the stage-1 text teacher), H100-native.  Mirrors `sam3/sam3/model/text_encoder_ve.py`:
`VETextEncoder`, `TextTransformer`, `Transformer`, `ResidualAttentionBlock` with the same constructor arguments and keys
(`encoder.positional_embedding`, `encoder.text_projection`, `encoder.token_embedding.weight`,
`encoder.transformer.resblocks.N.{attn.in_proj_*, attn.out_proj.*, ln_1, ln_2, mlp.c_fc, mlp.c_proj}`, `encoder.ln_final`,
`resizer`).  Parameter containers only; eval-mode forward on libes3.so:

  token embedding + positional table                   es3_text_embed (the plain rows are returned as inputs_embeds)
  24 x [LN, in_proj, causal attention, out_proj + res,  es3_layernorm_f32, es3_gemm_bf16_ex, es3_attention_causal_bf16
        LN, c_fc + GELU, c_proj + res]
  ln_final, resizer Linear(width -> d_model)            es3_layernorm_f32, es3_gemm_bf16_ex

TextTransformer also computes a pooled projection (`text_projection`) that VETextEncoder discards: it is not computed.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Callable, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from .. import ops
from ..backbones.mobile_clip import check_native, host_ids
from ..nn_utils import NativePlanMixin, StagedGraphMixin


def _f32(t):
    return t.detach().float().contiguous()


class ResidualAttentionBlock(nn.Module):
    def __init__(self, d_model: int, n_head: int, mlp_ratio: float = 4.0, ls_init_value: Optional[float] = None,
                 act_layer: Callable[[], nn.Module] = nn.GELU, norm_layer: Callable[[int], nn.Module] = nn.LayerNorm):
        super().__init__()
        if ls_init_value is not None:
            raise NotImplementedError("ResidualAttentionBlock: LayerScale is not used by the SAM3 text encoder")
        self.attn = nn.MultiheadAttention(d_model, n_head, batch_first=True)
        self.ln_1 = norm_layer(d_model)
        self.ln_2 = norm_layer(d_model)
        self.ls_1 = nn.Identity()
        self.ls_2 = nn.Identity()
        mlp_width = int(d_model * mlp_ratio)
        self.mlp = nn.Sequential(OrderedDict([("c_fc", nn.Linear(d_model, mlp_width)), ("gelu", act_layer()),
                                              ("c_proj", nn.Linear(mlp_width, d_model))]))

    def plan(self):
        a = self.attn
        return dict(kind="attn", n1=(_f32(self.ln_1.weight), _f32(self.ln_1.bias), self.ln_1.eps),
                    qkv=(a.in_proj_weight.detach().to(torch.bfloat16).contiguous(), _f32(a.in_proj_bias)),
                    proj=(a.out_proj.weight.detach().to(torch.bfloat16).contiguous(), _f32(a.out_proj.bias)),
                    n2=(_f32(self.ln_2.weight), _f32(self.ln_2.bias), self.ln_2.eps),
                    fc1=(self.mlp.c_fc.weight.detach().to(torch.bfloat16).contiguous(), _f32(self.mlp.c_fc.bias)),
                    fc2=(self.mlp.c_proj.weight.detach().to(torch.bfloat16).contiguous(), _f32(self.mlp.c_proj.bias)),
                    heads=a.num_heads, scale=a.head_dim ** -0.5)


class Transformer(nn.Module):
    def __init__(self, width: int, layers: int, heads: int, mlp_ratio: float = 4.0, ls_init_value: Optional[float] = None,
                 act_layer: Callable[[], nn.Module] = nn.GELU, norm_layer: Callable[[int], nn.Module] = nn.LayerNorm,
                 compile_mode: Optional[str] = None, use_act_checkpoint: bool = False):
        super().__init__()
        self.width, self.layers = width, layers
        self.grad_checkpointing = use_act_checkpoint
        self.resblocks = nn.ModuleList([ResidualAttentionBlock(width, heads, mlp_ratio, ls_init_value=ls_init_value,
                                                               act_layer=act_layer, norm_layer=norm_layer)
                                        for _ in range(layers)])


class TextTransformer(nn.Module):
    def __init__(self, context_length: int = 77, vocab_size: int = 49408, width: int = 512, heads: int = 8, layers: int = 12,
                 mlp_ratio: float = 4.0, ls_init_value: Optional[float] = None, output_dim: int = 512,
                 no_causal_mask: bool = False, pool_type: str = "none", proj_bias: bool = False, act_layer: Callable = nn.GELU,
                 norm_layer: Callable = nn.LayerNorm, output_tokens: bool = False, use_ln_post: bool = True,
                 compile_mode: Optional[str] = None, use_act_checkpoint: bool = False):
        super().__init__()
        if proj_bias or not use_ln_post:
            raise NotImplementedError("TextTransformer: the native path covers the SAM3 text encoder (ln_final, projection "
                                      "matrix)")
        self.output_tokens = output_tokens
        self.num_pos = self.context_length = context_length
        self.vocab_size, self.width, self.output_dim, self.heads, self.pool_type = vocab_size, width, output_dim, heads, pool_type
        self.token_embedding = nn.Embedding(self.vocab_size, width)
        self.positional_embedding = nn.Parameter(torch.empty(self.num_pos, width))
        nn.init.normal_(self.positional_embedding, std=0.01)
        self.transformer = Transformer(width=width, layers=layers, heads=heads, mlp_ratio=mlp_ratio,
                                       ls_init_value=ls_init_value, act_layer=act_layer, norm_layer=norm_layer)
        self.ln_final = norm_layer(width)
        self.causal = not no_causal_mask
        self.text_projection = nn.Parameter(torch.empty(width, output_dim))
        nn.init.normal_(self.text_projection, std=width ** -0.5)


class VETextEncoder(nn.Module, NativePlanMixin, StagedGraphMixin):
    def __init__(self, d_model: int, tokenizer: Callable, width: int = 1024, heads: int = 16, layers: int = 24,
                 context_length: int = 32, vocab_size: int = 49408, use_ln_post: bool = True, compile_mode: Optional[str] = None,
                 use_act_checkpoint: bool = True):
        super().__init__()
        self.context_length = context_length
        self.use_ln_post = use_ln_post
        self.tokenizer = tokenizer
        self.encoder = TextTransformer(context_length=self.context_length, vocab_size=vocab_size, width=width, heads=heads,
                                       layers=layers, output_tokens=True, use_ln_post=use_ln_post)
        self.resizer = nn.Linear(self.encoder.width, d_model)

    def _build_plan(self):
        e = self.encoder
        return dict(table=_f32(e.token_embedding.weight), pos=_f32(e.positional_embedding),
                    layers=[blk.plan() for blk in e.transformer.resblocks],
                    ln=(_f32(e.ln_final.weight), _f32(e.ln_final.bias), e.ln_final.eps),
                    resizer=(self.resizer.weight.detach().to(torch.bfloat16).contiguous(), _f32(self.resizer.bias)))

    def forward(self, text: Union[List[str], Tuple[torch.Tensor, torch.Tensor, dict]], input_boxes: Optional[List] = None,
                device: torch.device = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        return self._forward(text, input_boxes, self._graphs is not None)

    def forward_uncaptured(self, text, input_boxes=None, device=None):
        """forward() launched kernel by kernel, whether or not CUDA graphs are enabled."""
        return self._forward(text, input_boxes, False)

    @torch.no_grad()
    def _forward(self, text, input_boxes, graphed):
        if not (torch.is_tensor(text) or isinstance(text[0], str)):
            # already encoded (text_encoder_ve.py:315-321)
            assert input_boxes is None or len(input_boxes) == 0, "Can't replace boxes in text if it's already encoded"
            mask, memory, tokenized = text
            return mask, memory, tokenized["inputs_embeds"].transpose(0, 1)
        assert input_boxes is None or len(input_boxes) == 0, "not supported"
        dev = check_native(self, "VETextEncoder", self.training)
        if torch.is_tensor(text):
            ids = host_ids(text, self.encoder.vocab_size)
        else:
            if self.tokenizer is None:
                raise ValueError("VETextEncoder: string input needs a tokenizer (SimpleTokenizer(bpe_path=...))")
            ids = self.tokenizer(text, context_length=self.context_length)
            ids = host_ids(ids, self.encoder.vocab_size)
        B, L = ids.shape
        if L > self.encoder.num_pos:
            raise ValueError(f"VETextEncoder: {L} tokens exceed the {self.encoder.num_pos}-entry positional table")
        if graphed:
            memory, emb = self._graphed((B, L, "ids", True, dev), [ids], [], self._forward_ids)
        else:
            memory, emb = self._forward_ids(ids.to(dev, non_blocking=True))
        mask = (ids != 0).bool().ne(1)
        return mask.to(dev), memory.transpose(0, 1), emb.transpose(0, 1)

    def _forward_ids(self, ids):
        """ids [B, L] on the device -> (memory fp32 [B, L, d_model], inputs_embeds fp32 [B, L, width])."""
        from ..backbones.mobile_clip import run_layers
        B, L = ids.shape
        p = self._plan()
        C = self.encoder.width
        x, emb = ops.text_embed(ids, p["table"], p["pos"][:L], emb="plain")
        xs = run_layers(p["layers"], x, B, L, causal=self.encoder.causal)
        yb, _ = ops.layernorm(xs, *p["ln"])
        w, b = p["resizer"]
        memory = ops.gemm(yb, w, bias=b, out_dtype=torch.float32).view(B, L, -1)
        return memory, emb.view(B, L, C)
