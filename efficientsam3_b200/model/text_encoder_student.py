"""Drop-in for `sam3/sam3/model/text_encoder_student.py` `TextStudentEncoder`: tokenizer -> MobileCLIP text transformer ->
projector Linear(dim -> output_dim), forward on libes3.so.  Keys: `encoder.*` (MobileCLIPTextTransformer), `projector.*`.

forward(text) returns (pad_mask [B, L] bool, True = padding id 0; memory [L, B, output_dim] fp32; input_embeds [L, B, dim]
fp32 = token + positional embedding), the reference's sequence-first layout as transposed views.  Padding tokens take part
in attention, as in the reference (no key_padding_mask is passed), so a caption's output depends on the context length
but not on the other captions of the batch.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from ..backbones.mobile_clip import MobileCLIPTextTransformer, check_native, host_ids
from ..nn_utils import NativePlanMixin
from .tokenizer_ve import SimpleTokenizer


def _lin(linear: nn.Linear):
    return linear.weight.detach().to(torch.bfloat16).contiguous(), linear.bias.detach().float().contiguous()


class TextStudentEncoder(nn.Module, NativePlanMixin):
    def __init__(self, cfg, context_length, output_dim, bpe_path=None):
        super().__init__()
        self.context_length = context_length
        # the reference defaults to its bundled assets/bpe_simple_vocab_16e6.txt.gz; this package ships no vocabulary
        self.tokenizer = SimpleTokenizer(bpe_path=bpe_path) if bpe_path is not None else None
        self.encoder = MobileCLIPTextTransformer(cfg=cfg, projection_dim=cfg["dim"])
        self.projector = nn.Linear(cfg["dim"], output_dim)

    def set_context_length(self, context_length: int):
        """text_encoder_student.py:31-38: tokenise at the new length; the positional table is truncated (never grown)."""
        self.context_length = context_length
        self.encoder.resize_pos_embed(context_length)

    def _build_plan(self):
        return dict(proj=_lin(self.projector))

    def tokenize(self, text) -> torch.Tensor:
        if torch.is_tensor(text):
            return host_ids(text, self.encoder.vocab_size)
        if self.tokenizer is None:
            raise ValueError("TextStudentEncoder: string input needs a tokenizer; construct it with bpe_path=<CLIP "
                             "bpe_simple_vocab_16e6.txt.gz>")
        return self.tokenizer(text, context_length=self.context_length)

    @torch.no_grad()
    def forward(self, text, input_boxes=None, device=None):
        dev = check_native(self, "TextStudentEncoder", self.training)
        ids = self.tokenize(text)
        mask = (ids != 0).bool().ne(1)                       # True = padding (text_encoder_student.py:56)
        B, L = ids.shape
        emb = self.encoder.embed_tokens(ids)                 # [B, L, dim]: also the trunk's input stream
        _, yb = self.encoder.encode_tokens(emb)
        w, b = self._plan()["proj"]
        memory = ops.gemm(yb, w, bias=b, out_dtype=torch.float32).view(B, L, -1)
        return mask.to(dev), memory.transpose(0, 1), emb.transpose(0, 1)
