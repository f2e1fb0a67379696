"""Drop-in for `sam3/sam3/model/text_encoder_student.py` `TextStudentEncoder`: tokenizer -> MobileCLIP text transformer ->
projector Linear(dim -> output_dim), forward on libes3.so.  Keys: `encoder.*` (MobileCLIPTextTransformer), `projector.*`.

forward(text) returns (pad_mask [B, L] bool, True = padding id 0; memory [L, B, output_dim] fp32; input_embeds [L, B, dim]
fp32 = token + positional embedding), the reference's sequence-first layout as transposed views.  Padding tokens take part
in attention, as in the reference (no key_padding_mask is passed), so a caption's output depends on the context length
but not on the other captions of the batch.

Train mode (base students: every TransformerEncoder trunk; MobileCLIP-S0 once every BatchNorm of its RepMixerBlocks is in .eval(),
i.e. frozen BN as set_bn_state / TRAIN.EVAL_BN_WHEN_TRAINING leaves it) with grad enabled records the forward as ONE autograd
node (TextStudentTrainFunction) whose backward runs the native kernels (backbones/mobile_clip.py TextStudentTrainGraph).  `encoder.projection_layer` is not used here (the reference calls the encoder with return_all_tokens=True):
it gets no gradient, so optimisers skip it (build stage1.optim.FlatAdamW with exclude=TextStudentEncoder.UNUSED_PARAMETERS).
A train-mode module under torch.no_grad() runs the eval path: the base students have no train-time behaviour besides gradients.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from ..backbones.mobile_clip import MobileCLIPTextTransformer, TextStudentTrainGraph, check_native, check_trainable, host_ids
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

    # the reference's TextStudentEncoder never reads this parameter (return_all_tokens=True): it keeps no gradient
    UNUSED_PARAMETERS = ("encoder.projection_layer",)
    # stage1.optim.FlatAdamW may point the backward straight at its gradient arena (GradSink.direct)
    supports_direct_grads = True

    def forward(self, text, input_boxes=None, device=None):
        if self.training:
            dev = check_trainable(self, self.encoder, "TextStudentEncoder")
            if torch.is_grad_enabled():
                return self._forward_train(text, dev)
        else:
            dev = check_native(self, "TextStudentEncoder", self.training)
        with torch.no_grad():
            return self._forward_eval(text, dev)

    def _forward_eval(self, text, dev):
        ids = self.tokenize(text)
        mask = (ids != 0).bool().ne(1)                       # True = padding (text_encoder_student.py:56)
        B, L = ids.shape
        emb = self.encoder._embed(ids)                       # [B, L, dim]: also the trunk's input stream
        _, yb = self.encoder._encode(emb)
        w, b = self._plan()["proj"]
        memory = ops.gemm(yb, w, bias=b, out_dtype=torch.float32).view(B, L, -1)
        return mask.to(dev), memory.transpose(0, 1), emb.transpose(0, 1)

    def trainable_parameters(self):
        """The parameters the training graph produces gradients for (all but UNUSED_PARAMETERS)."""
        skip = set(self.UNUSED_PARAMETERS)
        return [p for n, p in self.named_parameters() if n not in skip and p.requires_grad]

    def _forward_train(self, text, dev):
        ids = self.tokenize(text)                            # checked on the host before anything is launched
        if ids.shape[1] > ops.TEXT_ATTN_BWD_MAX_L:
            raise ValueError(f"TextStudentEncoder: training takes 1..{ops.TEXT_ATTN_BWD_MAX_L} tokens per caption, got "
                             f"{ids.shape[1]}")
        mask = (ids != 0).bool().ne(1)
        memory, emb = TextStudentTrainFunction.apply(self, ids, *self.trainable_parameters())
        return mask.to(dev), memory.transpose(0, 1), emb.transpose(0, 1)


class TextStudentTrainFunction(torch.autograd.Function):
    """memory = student(ids) with a native backward (one node, as stage1.model.StudentTrainFunction): the forward runs the
    training graph and keeps it; the backward walks it in reverse, accumulating straight into FlatAdamW's arena views when the
    optimiser registered itself (GradSink.direct), otherwise returning one fp32 gradient per parameter to autograd (torch AdamW,
    DDP).  Outputs: memory [B, L, out] fp32 and input_embeds [B, L, dim] (no gradient)."""

    @staticmethod
    def forward(ctx, module, ids, *params):
        for m in module.modules():          # packed eval-mode weights go stale once parameters move
            if isinstance(m, NativePlanMixin):
                m._plan_key = None
        graph = TextStudentTrainGraph(module)
        memory, emb = graph.forward(ids, next(module.parameters()).device)
        ctx.graph, ctx.module, ctx.params = graph, module, params
        ctx.mark_non_differentiable(emb)
        return memory, emb

    @staticmethod
    def backward(ctx, dmem, demb):
        if ctx.graph is None:
            raise RuntimeError("the native text student keeps its saved activations for ONE backward pass (retain_graph / double "
                               "backward are not supported): run the forward again")
        graph = ctx.graph
        ctx.graph = None
        from ..backbones.efficientvit_train import GradSink
        grads = GradSink()
        grads.direct = getattr(ctx.module, "_es3_grad_arena", None) is not None
        graph.backward(dmem.float().contiguous(), grads)
        return (None, None) + tuple(grads.get(p) for p in ctx.params)
