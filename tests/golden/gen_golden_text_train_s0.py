"""Generate the MobileCLIP-S0 TRAINING fixtures (frozen BatchNorm) by running the UNMODIFIED reference modules (CPU fp32).

    python tests/golden/gen_golden_text_train_s0.py

Needs /root/reference (absent on the GPU box -- fixtures are committed).  For each case the reference TextStudentEncoder of
MobileCLIP-S0 is built at n_transformer_layers=1 (trunk: RepMixerBlock, TransformerEncoder, RepMixerBlock; weights and BatchNorm
running statistics from oracle.weights.fill_state_dict(seed)), put in .train(), and then frozen by the reference's own set_bn_state
(train_image_encoder_stage1.py:310-314, compiled from the AST of that script) with TRAIN.EVAL_BN_WHEN_TRAINING = True.  One
iteration of the reference's text train_one_epoch is composed as tests/golden/gen_golden_text_train.py does (same loss functions,
permute_words after random.seed(seed_p), the consistency block twice), and one backward pass runs.  Writes:

  text_train_s0_*.npz   the keys of gen_golden_text_train.py's fixtures, plus the BatchNorms' names, running mean / var and
                        num_batches_tracked after the iteration (frozen BN: equal to the loaded values)
"""
from __future__ import annotations

import ast
import os
import random
import sys
from types import SimpleNamespace as NS

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from gen_golden_text import TEXT_CAPTIONS, _text_student, keyshapes  # noqa: E402  (installs the reference shim)
from gen_golden_text_train import _ref_functions  # noqa: E402
from oracle.weights import fill_state_dict  # noqa: E402

REF_IMAGE_TRAINER = "/root/reference/stage1/train_image_encoder_stage1.py"
S0_LAYERS = dict(model_name="mct", n_transformer_layers=1)


def _ref_set_bn_state():
    tree = ast.parse(open(REF_IMAGE_TRAINER).read())
    ns = {"torch": torch}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name == "set_bn_state":
            exec(compile(ast.Module([node], []), REF_IMAGE_TRAINER, "exec"), ns)
    return ns["set_bn_state"]


def gen_text_train_s0(tag, ctx, seed_w, seed_t, seed_p, masked, cosine, consistency, table=None):
    permute_words, text_mse, text_cosine_loss, masked_text_mse, masked_text_cosine_loss = _ref_functions()
    set_bn_state = _ref_set_bn_state()
    m = _text_student("MobileCLIP-S0", ctx, table, None, S0_LAYERS)
    m.load_state_dict(fill_state_dict(m.state_dict(), seed_w))
    m.train()
    set_bn_state(NS(TRAIN=NS(EVAL_BN_WHEN_TRAINING=True)), m)
    bns = [(n, b) for n, b in m.named_modules() if isinstance(b, torch.nn.modules.batchnorm._BatchNorm)]
    assert bns and not any(b.training for _, b in bns)
    samples = list(TEXT_CAPTIONS)
    g = torch.Generator().manual_seed(seed_t)
    teacher16 = (torch.randn(len(samples), m.context_length, 256, generator=g) * 0.5).half()
    saved_embeddings = teacher16.float()
    random.seed(seed_p)
    perm_strings = []
    with torch.enable_grad():
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
        if p.grad is None:
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
                        grad_stats=np.stack(gstat), seed_w=seed_w, seed_p=seed_p, ctx=m.context_length, backbone="MobileCLIP-S0",
                        table=table or 0, layers=np.array(repr(S0_LAYERS)), masked=int(masked), cosine=cosine, consistency=consistency,
                        bn_names=np.array([n for n, _ in bns]),
                        running=np.stack([torch.stack([b.running_mean, b.running_var]).numpy() for _, b in bns]),
                        num_batches_tracked=np.array([int(b.num_batches_tracked) for _, b in bns]))
    print(tag, "loss %.6f" % loss.item(), "->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


def main():
    # es_mc_s.yaml: context 16, table 16, masked, COSINE 2.0, CONSISTENCY_LOSS 0.05 (applied twice)
    gen_text_train_s0("text_train_s0_ctx16", 16, seed_w=121, seed_t=221, seed_p=321, masked=True, cosine=2.0, consistency=0.05)
    # the 77-entry table resized to 32 tokens, unmasked
    gen_text_train_s0("text_train_s0_ctx32", 32, seed_w=122, seed_t=222, seed_p=322, masked=False, cosine=1.0, consistency=0.0,
                      table=77)


if __name__ == "__main__":
    main()
