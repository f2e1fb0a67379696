"""Stage-1 text-student training step on one GPU: the native step (TextStudentEncoder train mode + text KD loss + backward +
clip + FlatAdamW) against the oracle's functional restatement (oracle/text.py) trained eagerly on the same GPU, once the way the
reference trains (fp16 autocast, torch.amp.GradScaler, torch.optim.AdamW) and once in fp32.  Prints one JSON line.

    python scripts/bench_text_train.py [--steps 20] [--warmup 5]

One timed iteration is the configured one of the text_{s1,l,s0}_ctx{16,32} configs (their es_mc_m / es_mc_l bases set
MASK_PAD_TOKENS True, COSINE 2.0, CONSISTENCY_LOSS 0.05): captions -> tokenise -> forward -> masked text MSE + 2.0 * cosine ->
the consistency block twice (permute_words, tokenise, a second and a third forward, mse of the L-means) -> backward through all
three forwards -> global-norm clip 5.0 -> AdamW.  Both arms tokenise on the host inside the timed region.  The median and the
10th / 90th percentiles of `--steps` per-iteration CUDA-event times after `--warmup` iterations are reported.  Captions are
seeded word sequences (3-14 words) over the words of the test strings, tokenised with the CLIP merge subset the tests rebuild
(tests/golden/text_bpe_subset.json); teacher embeddings are seeded random fp16 values upcast to fp32, as stored.
MobileCLIP-S0 runs with every BatchNorm frozen in .eval() (TRAIN.EVAL_BN_WHEN_TRAINING: running statistics, as the oracle's BN
in both eager arms).  Algorithmic FLOPs per step (train_flops): three forwards (oracle.text.flops_mobileclip) and three backwards, each GEMM's backward
2x its forward, the attention backward 10 B L^2 C per layer (S recomputed, dP, dV, dQ, dK) against the forward's 4 B L^2 C.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import statistics
import sys
from types import SimpleNamespace as NS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench_text import gpu_info  # noqa: E402

COSINE, CONSISTENCY = 2.0, 0.05


def captions(n, seed):
    import numpy as np
    words = sorted({w for s in np.load(os.path.join(ROOT, "tests", "golden", "text_tokens.npz"))["strings"] for w in str(s).split()
                    if w.isascii() and w.isalpha()})
    g = random.Random(seed)
    return [" ".join(g.choice(words) for _ in range(g.randint(3, 14))) for _ in range(n)]


def train_flops(cfg, B, L, out_dim):
    from oracle import text as OT
    fwd = OT.flops_mobileclip(cfg, B, L, out_dim)
    attn_fwd = cfg["n_transformer_layers"] * 4 * B * L * L * cfg["dim"]
    bwd = 2 * (fwd - attn_fwd) + cfg["n_transformer_layers"] * 10 * B * L * L * cfg["dim"]
    return 3 * (fwd + bwd)


def per_step_ms(fn, steps, warmup):
    """(median, p10, p90) of per-iteration CUDA-event times in ms."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    q = statistics.quantiles(times, n=10)
    return statistics.median(times), q[0], q[-1]


def eager_arm(sd_dev, tok, ctx, caps, teacher, cfg, amp, trainable=None):
    """The oracle graph trained as the reference's loop does (train_text_encoder_stage1.py:221-288), consistency block twice.
    trainable: the parameter names (default: every state_dict entry; BatchNorm buffers are not parameters)."""
    from efficientsam3_b200.stage1.losses import permute_words
    from oracle import text as OT
    params = {k: v.clone().requires_grad_(True) for k, v in sd_dev.items()
              if k != "encoder.projection_layer" and (trainable is None or k in trainable)}
    sd = dict(sd_dev, **params)
    opt = torch.optim.AdamW(list(params.values()), lr=1e-4, weight_decay=0.05)
    scaler = torch.amp.GradScaler("cuda", enabled=amp)
    dev = teacher.device

    def step():
        ids = tok(caps, context_length=ctx).to(dev, non_blocking=True)
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            preds = OT.text_student(sd, ids, cfg)[1].transpose(0, 1)
            valid = (ids != 0).float()
            sim = F.cosine_similarity(preds, teacher, dim=2)
            n = valid.sum(1).clamp(min=1.0)
            loss = (((preds - teacher) * valid.unsqueeze(-1)).square().sum(dim=(1, 2)) / (n * preds.size(2))).mean()
            loss = loss + COSINE * (((1.0 - sim) * valid).sum(1) / n).mean()
            for _ in range(2):
                pids = tok([permute_words(c) for c in caps], context_length=ctx).to(dev, non_blocking=True)
                q = OT.text_student(sd, pids, cfg)[1].transpose(0, 1)
                loss = loss + CONSISTENCY * F.mse_loss(preds.mean(dim=1), q.mean(dim=1))
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(list(params.values()), 5.0)
        scaler.step(opt)
        scaler.update()
        opt.zero_grad()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text_train.py measures on a CUDA device; none is available")
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import text_kd_train_step
    from efficientsam3_b200.stage1.model import build_text_student_model
    from efficientsam3_b200.stage1.optim import FlatAdamW
    from oracle.weights import fill_state_dict
    from test_text_cpu import BPE

    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = dict(metric="text_train_step_ms", steps=args.steps, warmup=args.warmup, **gpu_info(dev),
               timed_region="per-iteration CUDA events: captions -> tokenise -> 3 forwards (consistency twice) -> masked KD loss + "
                            "consistency -> backward -> clip -> AdamW; median and p10 / p90",
               loss=dict(mask_pad_tokens=True, cosine=COSINE, consistency=CONSISTENCY))
    for tag, backbone, B, L in (("mobileclip_s1_b64_ctx32", "MobileCLIP-S1", 64, 32), ("mobileclip_s1_b64_ctx16", "MobileCLIP-S1", 64, 16),
                                ("mobileclip2_l_b32_ctx32", "MobileCLIP2-L", 32, 32), ("mobileclip2_l_b32_ctx16", "MobileCLIP2-L", 32, 16),
                                ("mobileclip_b_b64_ctx32", "MobileCLIP-B", 64, 32),
                                ("mobileclip_s0_b64_ctx32", "MobileCLIP-S0", 64, 32), ("mobileclip_s0_b64_ctx16", "MobileCLIP-S0", 64, 16)):
        m = build_text_student_model(NS(MODEL=NS(BACKBONE=backbone, BPE_PATH=BPE), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=L)))
        sd = fill_state_dict(m.state_dict(), 1)
        m.load_state_dict(sd)
        m = m.to(dev).train()
        enc = m.encoder
        mct = enc.transformer[0].__class__.__name__ == "RepMixerBlock"
        if mct:       # S0 trains with frozen BatchNorm (TRAIN.EVAL_BN_WHEN_TRAINING); the oracle's BN uses running statistics too
            for mod in m.modules():
                if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
                    mod.eval()
        caps = captions(B, 0)
        teacher = (torch.randn(B, L, 256, generator=torch.Generator().manual_seed(2)) * 0.5).half().float().to(dev)
        opt = FlatAdamW(m, lr=1e-4, weight_decay=0.05, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
        cfg = dict(causal_masking=enc.causal_masking, model_name="mct" if mct else "base",
                   n_transformer_layers=len(enc.transformer) - (2 if mct else 0),
                   n_heads_per_layer=enc.transformer[1 if mct else 0].pre_norm_mha[1].num_heads, dim=enc.model_dim,
                   ffn_multiplier_per_layer=4.0)
        random.seed(0)

        def native():
            text_kd_train_step(m, opt, caps, teacher, cosine_weight=COSINE, mask_pad_tokens=True, consistency_weight=CONSISTENCY,
                               clip_grad=5.0, lr=1e-4)

        native()
        n0 = ops.launch_count
        native()
        launches = ops.launch_count - n0
        ms, ms_lo, ms_hi = per_step_ms(native, args.steps, args.warmup)
        sd_dev = {k: v.to(dev) for k, v in sd.items()}
        names = {n for n, _ in m.named_parameters()}
        ms16, ms16_lo, ms16_hi = per_step_ms(eager_arm(sd_dev, m.tokenizer, L, caps, teacher, cfg, True, names), args.steps,
                                             args.warmup)
        ms32, ms32_lo, ms32_hi = per_step_ms(eager_arm(sd_dev, m.tokenizer, L, caps, teacher, cfg, False, names), args.steps,
                                             args.warmup)
        flops = train_flops(cfg, B, L, 256)
        r3 = lambda *v: [round(x, 3) for x in v]  # noqa: E731
        res[tag] = dict(batch=B, ctx=L, **(dict(frozen_bn=True) if mct else {}), native_ms=round(ms, 3), native_p10_p90_ms=r3(ms_lo, ms_hi), launches_per_step=launches,
                        gflop_per_step=round(flops / 1e9, 1), native_tflops=round(flops / ms / 1e9, 2),
                        eager_fp16_autocast_ms=round(ms16, 3), eager_fp16_autocast_p10_p90_ms=r3(ms16_lo, ms16_hi),
                        eager_fp32_ms=round(ms32, 3), eager_fp32_p10_p90_ms=r3(ms32_lo, ms32_hi),
                        speedup_vs_fp16_autocast=round(ms16 / ms, 2), speedup_vs_fp32=round(ms32 / ms, 2))
        del m, opt, sd, sd_dev
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
