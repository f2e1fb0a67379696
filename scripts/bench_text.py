"""Text-encoder throughput on one GPU: native MobileCLIP-S0 / MobileCLIP-B students and the SAM3 text teacher against the CPU
oracle's functional restatement (oracle/text.py) run eagerly on the same GPU in fp32 and under fp16 autocast (how the
reference trains).  Prints one JSON line.

    python scripts/bench_text.py [--steps 20] [--warmup 5]

Batches are 64 sequences (the text configs' batch) of seeded token ids laid out as the tokenizer lays out captions (start token,
3-14 word ids, end token, zero padding): the timed region is the forward from token ids.
Weights are seeded random (oracle.weights.fill_state_dict); throughput does not depend on their values.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace as NS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SOT, EOT = 49406, 49407


def gpu_info(dev):
    name = torch.cuda.get_device_name(dev)
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
        pl, mx = [s.strip() for s in out.split(",")[:2]]
        return dict(gpu=name, power_limit_w=float(pl), sm_max_mhz=float(mx))
    except Exception as e:   # nvidia-smi missing: the numbers are still measured, the card's limit is then unknown
        return dict(gpu=name, power_limit_w=None, note=f"nvidia-smi: {e}")


def token_ids(n, L, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(n, L, dtype=torch.long)
    for i in range(n):
        k = min(int(torch.randint(3, 15, (1,), generator=g)), L - 2)
        ids[i, :k + 2] = torch.cat([torch.tensor([SOT]), torch.randint(1, SOT, (k,), generator=g), torch.tensor([EOT])])
    return ids


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text.py measures on a CUDA device; none is available")
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.model import SAM3TextTeacherEncoder, build_text_student_model
    from oracle import text as OT
    from oracle.weights import fill_state_dict

    dev = torch.device("cuda:0")
    B = args.batch
    res = dict(metric="text_encoder_sequences_per_s", batch=B, steps=args.steps, warmup=args.warmup, **gpu_info(dev),
               timed_region="forward from token ids, CUDA events")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    def record(tag, native, oracle, flops):
        n0 = ops.launch_count
        native()
        launches = ops.launch_count - n0
        ms = timed(native, args.steps, args.warmup)
        ms32 = timed(oracle, args.steps, args.warmup)
        with torch.autocast("cuda", dtype=torch.float16):
            ms16 = timed(oracle, args.steps, args.warmup)
        res[tag] = dict(native_ms=round(ms, 3), native_seq_per_s=round(B / ms * 1e3, 1), launches_per_forward=launches,
                        gflop_per_batch=round(flops / 1e9, 2), native_tflops=round(flops / ms / 1e9, 2),
                        eager_fp32_ms=round(ms32, 3), eager_fp32_seq_per_s=round(B / ms32 * 1e3, 1),
                        eager_fp16_autocast_ms=round(ms16, 3), eager_fp16_autocast_seq_per_s=round(B / ms16 * 1e3, 1),
                        speedup_vs_fp32=round(ms32 / ms, 2), speedup_vs_fp16_autocast=round(ms16 / ms, 2))

    with torch.no_grad():
        for tag, backbone in (("mobileclip_s0_ctx32", "MobileCLIP-S0"), ("mobileclip_b_ctx32", "MobileCLIP-B")):
            m = build_text_student_model(NS(MODEL=NS(BACKBONE=backbone), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=32)))
            sd = fill_state_dict(m.state_dict(), 1)
            m.load_state_dict(sd)
            m = m.to(dev).eval()
            ids = token_ids(B, 32, 0)
            cfg = dict(causal_masking=m.encoder.causal_masking, model_name="mct" if backbone == "MobileCLIP-S0" else "base",
                       n_transformer_layers=4 if backbone == "MobileCLIP-S0" else 12, n_heads_per_layer=8, dim=512,
                       ffn_multiplier_per_layer=4.0)
            sd_dev = {k: v.to(dev) for k, v in sd.items()}
            ids_dev = ids.to(dev)
            record(tag, lambda: m(ids), lambda: OT.text_student(sd_dev, ids_dev, cfg), OT.flops_mobileclip(cfg, B, 32, 256))
            del m, sd, sd_dev
        t = SAM3TextTeacherEncoder(context_length=32)
        ve = t.sam3.backbone.language_backbone
        sd = fill_state_dict(ve.state_dict(), 2)
        ve.load_state_dict(sd)
        t = t.to(dev)
        sd_dev = {k: v.to(dev) for k, v in sd.items()}
        for L in (16, 32):
            ids = token_ids(B, L, 0)
            ids_dev = ids.to(dev)
            record(f"sam3_text_teacher_ctx{L}", lambda: ve(ids), lambda: OT.ve_text_encoder(sd_dev, ids_dev, heads=16),
                   OT.flops_ve(1024, 24, B, L))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
