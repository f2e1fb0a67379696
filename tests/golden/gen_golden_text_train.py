"""Generate the text-student TRAINING fixtures by running the UNMODIFIED reference modules and loss functions (CPU fp32).

    python tests/golden/gen_golden_text_train.py

Needs /root/reference (absent on the GPU box -- fixtures are committed).  For each case the reference TextStudentEncoder is built
in .train() at reduced depth (weights from oracle.weights.fill_state_dict(seed)), and one iteration of the reference's text
train_one_epoch is composed (stage1/train_text_encoder_stage1.py:225-272) with its own loss functions and permute_words, which are
compiled from the AST of that script (it is not importable here: yacs, timm.scheduler, ...; nothing is copied into the repo).
random.seed(seed_p) is set before the iteration, so the permuted captions are the reference's.  One backward pass.  Writes:

  text_train_*.npz   keys, ids, pad mask, teacher (fp16, as stored; upcast to fp32 as the trainer does), the permuted strings and
                     their ids, loss terms (loss, mse, cos, consistency 1, consistency 2), and per-parameter gradient statistics
                     (norm, sum, first 4 entries) of every parameter that receives a gradient
"""
from __future__ import annotations

import ast
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from gen_golden_text import TEXT_CAPTIONS, _text_student, keyshapes  # noqa: E402  (installs the reference shim)
from oracle.weights import fill_state_dict  # noqa: E402

REF_TRAINER = "/root/reference/stage1/train_text_encoder_stage1.py"


def _ref_functions():
    """permute_words, text_mse, text_cosine_loss, masked_text_mse, masked_text_cosine_loss (:327-370) from the reference's source."""
    import torch.nn.functional as F
    tree = ast.parse(open(REF_TRAINER).read())
    ns = {"torch": torch, "F": F, "random": random}
    want = ("permute_words", "text_mse", "text_cosine_loss", "masked_text_mse", "masked_text_cosine_loss")
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in want:
            exec(compile(ast.Module([node], []), REF_TRAINER, "exec"), ns)
    return tuple(ns[k] for k in want)


def gen_text_train(tag, backbone, ctx, seed_w, seed_t, seed_p, masked, cosine, consistency, table=None, layers=None):
    permute_words, text_mse, text_cosine_loss, masked_text_mse, masked_text_cosine_loss = _ref_functions()
    m = _text_student(backbone, ctx, table, None, layers)
    m.load_state_dict(fill_state_dict(m.state_dict(), seed_w))
    m.train()
    samples = list(TEXT_CAPTIONS)
    g = torch.Generator().manual_seed(seed_t)
    teacher16 = (torch.randn(len(samples), m.context_length, 256, generator=g) * 0.5).half()
    saved_embeddings = teacher16.float()                             # stored fp16, upcast (:212-217)
    random.seed(seed_p)
    perm_strings = []
    with torch.enable_grad():
        # :225-242
        pad_mask, preds, _ = m(samples, device="cpu")
        preds = preds.transpose(0, 1)
        if masked:
            valid = (~pad_mask).float()
            mse = masked_text_mse(preds, saved_embeddings, valid)
            cos = masked_text_cosine_loss(preds, saved_embeddings, valid)
        else:
            mse = text_mse(preds, saved_embeddings)
            cos = text_cosine_loss(preds, saved_embeddings)
        loss = mse
        if cosine > 0.0:
            loss = loss + cosine * cos
        # :244-270: the consistency block, twice
        cons = []
        for _ in range(2):
            if consistency > 0.0:
                permuted_samples = [permute_words(s) for s in samples]
                perm_strings.append(permuted_samples)
                _, preds_permuted, _ = m(permuted_samples, device="cpu")
                preds_permuted = preds_permuted.transpose(0, 1)
                c = torch.nn.functional.mse_loss(preds.mean(dim=1), preds_permuted.mean(dim=1))
                loss = loss + consistency * c
                cons.append(c.item())
        loss.backward()
    names, gstat = [], []
    for k, p in m.named_parameters():
        if p.grad is None:                                           # encoder.projection_layer: never used
            continue
        gr = p.grad.reshape(-1).double()
        first = torch.zeros(4, dtype=torch.float64)
        first[:min(4, gr.numel())] = gr[:4]
        names.append(k)
        gstat.append(torch.cat([gr.norm().reshape(1), gr.sum().reshape(1), first]).numpy())
    ids = m.tokenizer(samples, context_length=m.context_length)
    perm_ids = np.stack([m.tokenizer(ps, context_length=m.context_length).numpy() for ps in perm_strings]) if perm_strings \
        else np.zeros((0, len(samples), m.context_length), np.int64)
    cons += [0.0] * (2 - len(cons))
    path = os.path.join(HERE, f"{tag}.npz")
    np.savez_compressed(path, keys=keyshapes(m.state_dict()), ids=ids.numpy(), pad=pad_mask.numpy(), teacher=teacher16.numpy(),
                        perm_strings=np.array(perm_strings if perm_strings else np.zeros((0, len(samples)), "U1")), perm_ids=perm_ids,
                        loss=np.array([loss.item(), mse.item(), cos.item(), *cons]), grad_names=np.array(names),
                        grad_stats=np.stack(gstat), seed_w=seed_w, seed_p=seed_p, ctx=m.context_length, backbone=backbone,
                        table=table or 0, layers=np.array(repr(layers)), masked=int(masked), cosine=cosine, consistency=consistency)
    print(tag, "loss %.6f" % loss.item(), "->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


def main():
    gen_text_train("text_train_s1", "MobileCLIP-S1", 32, seed_w=111, seed_t=211, seed_p=311, masked=True, cosine=2.0,
                   consistency=0.05, layers=dict(n_transformer_layers=2))
    gen_text_train("text_train_b_causal", "MobileCLIP-B", 32, seed_w=112, seed_t=212, seed_p=312, masked=False, cosine=1.0,
                   consistency=0.0, layers=dict(n_transformer_layers=2, causal_masking=True))
    gen_text_train("text_train_768", "MobileCLIP2-L", 32, seed_w=113, seed_t=213, seed_p=313, masked=True, cosine=2.0,
                   consistency=0.0, table=77, layers=dict(dim=768, n_transformer_layers=2, n_heads_per_layer=12))


if __name__ == "__main__":
    main()
