"""Text-encoder eval forward from CUDA graphs (enable_cuda_graphs) against the same forward launched kernel by kernel and against
the oracle's eager restatement (oracle/text.py) under fp16 autocast, on one GPU.  Prints one JSON line.

    python scripts/bench_text_graphs.py [--steps 50] [--warmup 10] [--rounds 3]

Models: MobileCLIP-S0, MobileCLIP-B, MobileCLIP-S1 (students built at the context length, as the ctx-16 / ctx-32 configs build
them) and the SAM3 text teacher (24 layers, its 32-entry table).  Shapes: context 16 and 32, batch 1 and 64, seeded token ids laid
out as bench_text.py lays them out; the timed call is the forward from host token ids (validation, copy in, kernels).
Per arm and shape: the median and p10-p90 of per-call device time (CUDA events around each call), the median host time until the
call returns (the enqueue; no synchronisation inside the window), and es3 launches per forward.  The arms run in turn, `--rounds`
times, so that a drift of the machine falls on all of them.  `graph_equals_uncaptured` checks the replayed output bit for bit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from types import SimpleNamespace as NS

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))

import torch  # noqa: E402

from bench_text import gpu_info, token_ids  # noqa: E402

STUDENTS = {"MobileCLIP-S0": ("mobileclip_s0", "mct", 4, False), "MobileCLIP-B": ("mobileclip_b", "base", 12, True),
            "MobileCLIP-S1": ("mobileclip_s1", "base", 12, False)}


def percentile(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, max(0, int(round(q / 100 * (len(xs) - 1)))))]


def sample(fn, steps, dev_ms, host_ms):
    """`steps` calls, each between two CUDA events and timed on the host until it returns."""
    evs = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        t0 = time.perf_counter()
        fn()
        host_ms.append((time.perf_counter() - t0) * 1e3)
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    dev_ms += [e0.elapsed_time(e1) for e0, e1 in evs]


def compare(arms, steps, warmup, rounds):
    """arms: name -> (callable, launches per forward | None) -> per-arm statistics."""
    for fn, _ in arms.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    dev = {k: [] for k in arms}
    host = {k: [] for k in arms}
    for r in range(rounds):
        names = list(arms) if r % 2 == 0 else list(reversed(arms))
        for k in names:
            sample(arms[k][0], steps, dev[k], host[k])
    out = {}
    for k, (_, launches) in arms.items():
        d = dev[k]
        out[k] = dict(median_ms=round(percentile(d, 50), 4), p10_ms=round(percentile(d, 10), 4), p90_ms=round(percentile(d, 90), 4),
                      host_enqueue_median_ms=round(percentile(host[k], 50), 4), launches_per_forward=launches, samples=len(d))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=str, default="1,64")
    ap.add_argument("--contexts", type=str, default="16,32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text_graphs.py measures on a CUDA device; none is available")
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.model import SAM3TextTeacherEncoder, build_text_student_model
    from oracle import text as OT
    from oracle.weights import fill_state_dict

    dev = torch.device("cuda:0")
    batches = [int(b) for b in args.batches.split(",")]
    contexts = [int(c) for c in args.contexts.split(",")]
    res = dict(metric="text_encoder_forward_ms", steps=args.steps, warmup=args.warmup, rounds=args.rounds, **gpu_info(dev),
               timed_region="forward from host token ids; per-call CUDA events; host time until the call returns")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    def launches(fn):
        n0 = ops.launch_count
        fn()
        return ops.launch_count - n0

    def run(tag, model, native, eager):
        model.enable_cuda_graphs(False)
        ref = [t.clone() for t in native()]
        n_uncaptured = launches(native)
        model.enable_cuda_graphs(True)
        got = native()
        same = all(torch.equal(a, b) for a, b in zip(got, ref))
        arms = {"graph_replay": (native, model.graph_launches_per_step),
                "uncaptured": (lambda: model.forward_uncaptured(*native.args), n_uncaptured)}

        def autocast():
            with torch.autocast("cuda", dtype=torch.float16):
                eager()
        arms["eager_fp16_autocast"] = (autocast, None)
        r = compare(arms, args.steps, args.warmup, args.rounds)
        r["graph_equals_uncaptured"] = same
        res[tag] = r
        print(tag, json.dumps(r), file=sys.stderr, flush=True)

    class Call:
        def __init__(self, fn, *a):
            self.fn, self.args = fn, a

        def __call__(self):
            out = self.fn(*self.args)
            return out if isinstance(out, tuple) else (out,)

    with torch.no_grad():
        for backbone, (name, variant, layers, causal) in STUDENTS.items():
            for L in contexts:
                m = build_text_student_model(NS(MODEL=NS(BACKBONE=backbone), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=L)))
                sd = fill_state_dict(m.state_dict(), 1)
                m.load_state_dict(sd)
                m = m.to(dev).eval()
                cfg = dict(causal_masking=causal, model_name=variant, n_transformer_layers=layers, n_heads_per_layer=8, dim=512,
                           ffn_multiplier_per_layer=4.0)
                sd_dev = {k: v.to(dev) for k, v in sd.items()}
                for B in batches:
                    ids = token_ids(B, L, 0)
                    ids_dev = ids.to(dev)
                    run(f"{name}_b{B}_ctx{L}", m, Call(m, ids), lambda: OT.text_student(sd_dev, ids_dev, cfg))
                del m, sd, sd_dev
        t = SAM3TextTeacherEncoder(context_length=32)
        ve = t.sam3.backbone.language_backbone
        sd = fill_state_dict(ve.state_dict(), 2)
        ve.load_state_dict(sd)
        t = t.to(dev)
        sd_dev = {k: v.to(dev) for k, v in sd.items()}
        for L in contexts:
            for B in batches:
                ids = token_ids(B, L, 0)
                ids_dev = ids.to(dev)
                run(f"sam3_text_teacher_b{B}_ctx{L}", ve, Call(ve, ids), lambda: OT.ve_text_encoder(sd_dev, ids_dev, heads=16))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
