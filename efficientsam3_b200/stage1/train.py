"""Drop-in for the loop body of the reference's stage-1 trainer (stage1/train_image_encoder_stage1.py:154-268, 310-314):
`train_one_epoch` with the reference's loader contract -- batches of ((samples, annos), (saved_embeddings, seeds)) as
`build_loader` yields them, teacher embeddings read from the store -- on the native student, KD loss, backward and optimiser.
Logging / TensorBoard / checkpointing stay with the caller (out of scope, SURVEY.md section 2)."""
from __future__ import annotations

import numpy as np
import torch

from .losses import kd_train_step
from .optim import cosine_lr
from .preprocess import MEAN, STD, is_uint8_batch, prepare_images


def set_bn_state(config, model):
    """train_image_encoder_stage1.py:310-314: with TRAIN.EVAL_BN_WHEN_TRAINING every BatchNorm stays in eval mode (the native
    training graph then uses the running statistics and still produces the BN weight / bias gradients)."""
    if config.TRAIN.EVAL_BN_WHEN_TRAINING:
        for m in model.modules():
            if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
                m.eval()


def default_lr_at(config, optimizer, num_steps):
    """The reference's cosine schedule built from config.TRAIN, indexed by update (lr_scheduler.step_update)."""
    accum = int(config.TRAIN.ACCUMULATION_STEPS)
    n_iter = num_steps // accum                      # build_scheduler(config, optimizer, len(loader) // ACCUMULATION_STEPS), :80-84
    total = int(config.TRAIN.EPOCHS * n_iter)
    warm = int(config.TRAIN.WARMUP_EPOCHS * n_iter)
    base = getattr(optimizer, "base_lr", optimizer.lr)     # never optimizer.lr: step(lr=...) overwrites it every update

    def lr_at(t):
        return cosine_lr(t, base, total, config.TRAIN.MIN_LR, warm, config.TRAIN.WARMUP_LR)
    return lr_at


def lr_for_update(idx, epoch, num_steps, accum, lr_at):
    """LR of the update made at iteration `idx` of `epoch`.  The reference applies update u with the LR the PREVIOUS
    `step_update` call left in the optimiser (the scheduler is stepped after optimizer.step(), :216-229); the very first update
    runs at the scheduler's initial value, which is lr_at(0)."""
    prev = idx - accum                               # iteration index of the previous update inside this epoch
    if prev >= 0:
        return lr_at((epoch * num_steps + prev) // accum)
    last = (num_steps // accum) * accum - 1          # last updating iteration of the previous epoch
    if epoch > 0 and last >= 0:
        return lr_at(((epoch - 1) * num_steps + last) // accum)
    return lr_at(0)


def train_one_epoch(config, model, data_loader, optimizer, epoch, lr_at=None, on_step=None):
    """One epoch of stage-1 distillation.  `samples` are the reference's [3,S,S] fp32 images with annos["img_size_before_pad"], or
    decoded HWC uint8 images (a list or stage1.preprocess.PackedImages) that are prepared on the device with DATA.IMG_SIZE /
    DATA.MEAN / DATA.STD, their sizes before padding coming from the preparation.  `optimizer`: stage1.optim.FlatAdamW over `model`.  `lr_at(update_index) -> lr`
    replaces `lr_scheduler.step_update` (default: the reference's cosine schedule built from config.TRAIN).  `on_step(idx, loss)`
    is called after every iteration with the detached device loss (call `.item()` there only when you log: it syncs).
    Returns the list of per-iteration losses (device scalars)."""
    model.train()
    set_bn_state(config, model)
    optimizer.zero_grad()
    num_steps = len(data_loader)
    accum = int(config.TRAIN.ACCUMULATION_STEPS)
    embed_shape = (config.DISTILL.EMBED_DIM, config.DISTILL.EMBED_SIZE, config.DISTILL.EMBED_SIZE)
    if lr_at is None:
        lr_at = default_lr_at(config, optimizer, num_steps)
    cosine_w = float(config.DISTILL.COSINE)
    dev = next(model.parameters()).device
    losses = []
    for idx, ((samples, annos), (saved_embeddings, seeds)) in enumerate(data_loader):
        if is_uint8_batch(samples):
            samples, sizes_before_pad = prepare_images(samples, config.DATA.IMG_SIZE, getattr(config.DATA, "MEAN", MEAN),
                                                       getattr(config.DATA, "STD", STD), device=dev)
        else:
            samples = torch.stack(list(samples), dim=0).to(dev, non_blocking=True)
            sizes_before_pad = annos["img_size_before_pad"]
        saved = torch.from_numpy(np.stack(saved_embeddings, axis=0)).float()
        saved = saved.view(samples.size(0), *embed_shape).to(dev, non_blocking=True)
        update = (idx + 1) % accum == 0
        loss = kd_train_step(model, optimizer, samples, saved, sizes_before_pad, cosine_weight=cosine_w,
                             clip_grad=config.TRAIN.CLIP_GRAD,
                             lr=lr_for_update(idx, epoch, num_steps, accum, lr_at) if update else None,
                             accumulation_steps=accum, update=update)
        losses.append(loss)
        if on_step is not None:
            on_step(idx, loss)
        if getattr(config.DATA, "DEBUG", False):
            break
    return losses


def parse_text_batch(batch):
    """The two batch structures of train_text_encoder_stage1.py:197-209 -> (captions, saved_embeddings, seeds):
    [captions, [embeddings, seeds]] (default collate of DatasetWrapper items) or [(caption, (embedding, seed)), ...]."""
    if isinstance(batch, list) and len(batch) == 2 and isinstance(batch[0], (list, tuple)) and len(batch[0]) > 0 \
            and isinstance(batch[0][0], str):
        return list(batch[0]), batch[1][0], batch[1][1]
    if isinstance(batch, list) and len(batch) > 0 and isinstance(batch[0], tuple):
        return [item[0] for item in batch], [item[1][0] for item in batch], [item[1][1] for item in batch]
    raise ValueError(f"Unexpected batch structure: {type(batch)}")


def train_text_one_epoch(config, model, data_loader, optimizer, epoch, lr_at=None, on_step=None):
    """One epoch of stage-1 text distillation (train_text_encoder_stage1.py:161-288) on the native text student.  `optimizer`:
    stage1.optim.FlatAdamW over `model` (build it with exclude=TextStudentEncoder.UNUSED_PARAMETERS, as the reference's AdamW
    never sees a gradient for encoder.projection_layer).  Reads DISTILL.NUM_EMBED / EMBED_DIM (the stored embeddings' shape),
    MASK_PAD_TOKENS, COSINE and CONSISTENCY_LOSS; TRAIN.ACCUMULATION_STEPS / CLIP_GRAD and the cosine schedule as
    train_one_epoch does.  With TRAIN.EVAL_BN_WHEN_TRAINING (read with a default of False) every BatchNorm goes back to eval mode
    after model.train(), as set_bn_state does, and MobileCLIP-S0 trains with frozen BatchNorm.  Without it, S0 trains with
    batch-statistics BatchNorm once the model opted in (TextStudentEncoder.enable_batch_stat_bn), as the reference's text configs
    run it; otherwise it raises.  The reference's text trainer leaves that call commented out (train_text_encoder_stage1.py:173);
    its text configs all set the key False.
    Returns the list of per-iteration losses (device scalars)."""
    from .losses import text_kd_train_step
    model.train()
    if getattr(config.TRAIN, "EVAL_BN_WHEN_TRAINING", False):
        set_bn_state(config, model)
    optimizer.zero_grad()
    num_steps = len(data_loader)
    accum = int(config.TRAIN.ACCUMULATION_STEPS)
    embed_shape = (config.DISTILL.NUM_EMBED, config.DISTILL.EMBED_DIM)
    if lr_at is None:
        lr_at = default_lr_at(config, optimizer, num_steps)
    masked = bool(getattr(config.DISTILL, "MASK_PAD_TOKENS", False))
    cosine_w = float(config.DISTILL.COSINE)
    consistency_w = float(getattr(config.DISTILL, "CONSISTENCY_LOSS", 0.0))
    dev = next(model.parameters()).device
    losses = []
    for idx, batch in enumerate(data_loader):
        samples, saved_embeddings, _ = parse_text_batch(batch)
        saved = torch.from_numpy(np.stack(saved_embeddings, axis=0)).float()      # stored fp16 -> fp32 (:212-217)
        saved = saved.view(len(samples), *embed_shape).to(dev, non_blocking=True)
        update = (idx + 1) % accum == 0
        loss = text_kd_train_step(model, optimizer, samples, saved, cosine_weight=cosine_w, mask_pad_tokens=masked,
                                  consistency_weight=consistency_w, clip_grad=config.TRAIN.CLIP_GRAD,
                                  lr=lr_for_update(idx, epoch, num_steps, accum, lr_at) if update else None,
                                  accumulation_steps=accum, update=update)
        losses.append(loss)
        if on_step is not None:
            on_step(idx, loss)
        if getattr(getattr(config, "DATA", None), "DEBUG", False):
            break
    return losses
