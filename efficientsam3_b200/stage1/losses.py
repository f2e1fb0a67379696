"""Stage-1 KD loss and KD steps on the native path: masked MSE + masked cosine between student and teacher embeddings,
stage1/train_image_encoder_stage1.py:205-210, 271-307.  One streaming kernel + a fixed-order final reduction."""
from __future__ import annotations

import torch

from .. import ops


@torch.no_grad()
def kd_loss(preds: torch.Tensor, teacher: torch.Tensor, img_size: int, img_size_before_pad, cosine_weight: float = 1.0):
    """preds, teacher: [B,C,E,E] fp32 CUDA (NCHW, the modules' outputs); img_size_before_pad: sequence of (3, h, w)
    as the reference loader yields it.  Returns (loss, mse, cosine) 0-dim fp32 CUDA tensors."""
    sizes = torch.tensor([[int(s[1]), int(s[2])] for s in img_size_before_pad], dtype=torch.int32, device=preds.device)
    out, _ = ops.kd_loss_fwd(preds, teacher, sizes, img_size, cosine_weight)
    return out[0], out[1], out[2]


@torch.no_grad()
def kd_eval_step(student, teacher_model, images, img_size_before_pad, cosine_weight: float = 1.0):
    """Online teacher -> student -> loss (north-star wording of the stage-1 step, forward only; SURVEY.md D1/N1).
    The teacher embedding is rounded through fp16 as the reference's stored targets are
    (save_embedding_image_stage1.py:89-92: outputs.half())."""
    t = teacher_model(images).half().float()
    s = student(images)
    return kd_loss(s, t, images.shape[-1], img_size_before_pad, cosine_weight)


def kd_train_step(student, optimizer, images, teacher_embeddings, img_size_before_pad, cosine_weight: float = 1.0,
                  clip_grad: float = 5.0, lr: float | None = None, group=None, accumulation_steps: int = 1,
                  update: bool = True):
    """One iteration of the reference's train_one_epoch (stage1/train_image_encoder_stage1.py:185-230), everything on the
    device and on libes3 kernels:

        preds = model(samples)                 train-mode student forward (one autograd node, batch-statistics or frozen BN)
        loss  = masked_mse + COSINE * cosine   es3_kd_loss_fwd            (targets: stored / online teacher embeddings, fp32)
        loss_scaler(loss, optimizer, ...)      es3_kd_loss_bwd -> native student backward -> ONE all-reduce of the flat gradient
                                               arena (data parallel, SURVEY.md section 8e) -> global-norm clip + fused AdamW

    `optimizer` is a stage1.optim.FlatAdamW built on `student` (parameters and gradients live in its flat arenas, so the
    backward accumulates straight into the buffer that is all-reduced).  Gradient accumulation as in the reference
    (TRAIN.ACCUMULATION_STEPS, :212-226): the loss is divided by `accumulation_steps`, gradients add up in the arena, and only
    calls with `update=True` exchange, step and clear it.  Returns the detached (divided) loss, a device scalar -- no host sync.
    """
    from .optim import KDLossFunction
    if not student.training:
        raise RuntimeError("kd_train_step expects student.train() (freeze BN with set_bn_state-style .eval() on the BN modules)")
    sizes = torch.tensor([[int(s[1]), int(s[2])] for s in img_size_before_pad], dtype=torch.int32, device=images.device)
    preds = student(images)
    loss = KDLossFunction.apply(preds, teacher_embeddings, sizes, images.shape[-1], cosine_weight)
    if accumulation_steps != 1:
        loss = loss / accumulation_steps
    if hasattr(optimizer, "begin_backward"):
        optimizer.begin_backward(update, group)              # finished arena ranges may go to NCCL from inside the backward
    (loss * optimizer.loss_scale_tensor[0]).backward()       # GradScaler.scale(loss).backward(): the scale stays on the device
    if update:
        world = optimizer.all_reduce_grads(group)
        optimizer.step(lr=lr, max_norm=clip_grad, world_size=world)
        optimizer.zero_grad()                                # as the reference: clear right after the update (:224-225)
    return loss.detach()


def kd_train_step_online(student, teacher_model, optimizer, images, img_size_before_pad, cosine_weight: float = 1.0,
                         clip_grad: float = 5.0, lr: float | None = None, group=None, teacher_chunk: int = 8,
                         accumulation_steps: int = 1, update: bool = True):
    """The north-star wording of the stage-1 iteration (SURVEY.md D1 / N1): the frozen SAM3 teacher embeds the batch on the
    fly (no embedding store), the student is trained against it.  Targets are rounded through fp16 exactly as the stored
    embeddings are (save_embedding_image_stage1.py:89-92).  The teacher runs in chunks to bound its activation memory."""
    with torch.no_grad():
        t = torch.cat([teacher_model(images[i:i + teacher_chunk]) for i in range(0, images.shape[0], teacher_chunk)], 0)
        t = t.half().float()
    return kd_train_step(student, optimizer, images, t, img_size_before_pad, cosine_weight, clip_grad, lr, group,
                         accumulation_steps=accumulation_steps, update=update)


# ------------------------------------------------------------------------------------------------------------------ text KD
def permute_words(text: str) -> str:
    """train_text_encoder_stage1.py:327-333: shuffle the words of a caption with Python's global `random` (so a seeded run draws
    the reference's permutations)."""
    import random
    words = text.split()
    if len(words) <= 1:
        return text
    random.shuffle(words)
    return " ".join(words)


class TextKDLossFunction(torch.autograd.Function):
    """The text KD loss of train_text_encoder_stage1.py:230-270 as one node on es3_text_kd_loss_* / es3_text_consistency_*:
        loss = mse + cosine_weight * cos                      (masked_text_* with pad given, text_* without)
             + consistency_weight * sum_k mse(mean_L(preds), mean_L(perm_k))
    Returns (loss, mse, cos, consistency terms [K]); only `loss` carries a gradient (into preds and every perm_k)."""

    @staticmethod
    def forward(ctx, preds, teacher, pad, cosine_weight, consistency_weight, *perms):
        out, ws = ops.text_kd_loss_fwd(preds.detach(), teacher, pad, cosine_weight)
        mdiffs, terms = [], []
        for q in perms:                                  # each adds consistency_weight * its value into out[0], in order
            v, md = ops.text_consistency_fwd(preds.detach(), q.detach(), consistency_weight, loss=out)
            mdiffs.append(md)
            terms.append(v)
        cons = torch.cat(terms) if terms else out.new_zeros(0)
        ctx.save_for_backward(preds.detach(), teacher, ws, *mdiffs)
        ctx.pad, ctx.meta = pad, (cosine_weight, consistency_weight, preds.shape[1])
        loss, mse, cos = out[0].clone(), out[1].clone(), out[2].clone()
        ctx.mark_non_differentiable(mse, cos, cons)
        return loss, mse, cos, cons

    @staticmethod
    def backward(ctx, gloss, *_):
        preds, teacher, ws, *mdiffs = ctx.saved_tensors
        cw, kw, L = ctx.meta
        gout = gloss.reshape(1).float().contiguous()
        dp = ops.text_kd_loss_bwd(preds, teacher, ctx.pad, ws, cw, 1.0, None, gout)
        dqs = [ops.text_consistency_bwd(md, L, kw, dp, 1.0, None, gout) for md in mdiffs]
        return (dp, None, None, None, None, *dqs)


@torch.no_grad()
def text_kd_loss(preds: torch.Tensor, teacher: torch.Tensor, pad_mask=None, cosine_weight: float = 1.0):
    """preds, teacher: [B, L, D] fp32 CUDA; pad_mask [B, L] bool (True = padding: the masked loss) or None (plain loss).
    Returns (loss, mse, cos) 0-dim fp32 CUDA tensors (forward only)."""
    pad = pad_mask.to(preds.device).contiguous() if pad_mask is not None else None
    out, _ = ops.text_kd_loss_fwd(preds.contiguous(), teacher.contiguous(), pad, cosine_weight)
    return out[0], out[1], out[2]


def text_kd_train_step(student, optimizer, text, teacher_embeddings, *, cosine_weight: float = 1.0, mask_pad_tokens: bool = False,
                       consistency_weight: float = 0.0, clip_grad: float = 5.0, lr: float | None = None, group=None,
                       accumulation_steps: int = 1, update: bool = True):
    """One iteration of the reference's text train_one_epoch (stage1/train_text_encoder_stage1.py:221-288) on the native path:

        pad_mask, preds = student(text)          train-mode TextStudentEncoder (one autograd node, native backward)
        loss = [masked_]text_mse + COSINE * [masked_]text_cosine_loss
        twice, as the reference does (:244-256, :258-270), when consistency_weight > 0:
            loss += consistency_weight * mse(mean_L(preds), mean_L(student(permute_words(text))))
        loss / ACCUMULATION_STEPS, scaled by the device loss scale, backward -> all-reduce -> clip + AdamW (FlatAdamW)

    `text`: a list of captions (or token ids [B, L] when consistency_weight == 0); `teacher_embeddings`: [B, L, D] fp32 on the
    device.  Returns the detached (divided) loss, a device scalar -- no host synchronisation beyond tokenisation."""
    if not student.training:
        raise RuntimeError("text_kd_train_step expects student.train()")
    pad_mask, memory, _ = student(text)
    preds = memory.transpose(0, 1)                       # [B, L, D] (contiguous: the student's own layout)
    perms = []
    if consistency_weight > 0.0:
        if torch.is_tensor(text) or not all(isinstance(s, str) for s in text):
            raise ValueError("the consistency loss permutes the words of captions: pass the batch as a list of strings")
        for _ in range(2):                               # the reference's block appears twice (:244-256, :258-270)
            _, pm, _ = student([permute_words(s) for s in text])
            perms.append(pm.transpose(0, 1))
    teacher = teacher_embeddings.float().contiguous()
    if teacher.shape != preds.shape:
        raise ValueError(f"teacher embeddings {tuple(teacher.shape)} do not match the student's output {tuple(preds.shape)}")
    loss, _, _, _ = TextKDLossFunction.apply(preds, teacher, pad_mask.contiguous() if mask_pad_tokens else None, float(cosine_weight),
                                             float(consistency_weight), *perms)
    if accumulation_steps != 1:
        loss = loss / accumulation_steps
    if hasattr(optimizer, "begin_backward"):
        optimizer.begin_backward(update, group)
    (loss * optimizer.loss_scale_tensor[0]).backward()
    if update:
        world = optimizer.all_reduce_grads(group)
        optimizer.step(lr=lr, max_norm=clip_grad, world_size=world)
        optimizer.zero_grad()
    return loss.detach()
