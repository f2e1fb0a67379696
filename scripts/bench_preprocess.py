"""Cost of preparing stage-1 images on the device from decoded uint8 (es3_prepare_images_u8) against the alternatives.

    python scripts/bench_preprocess.py [--batch 32] [--h 1500] [--w 2250] [--img 1008] [--iters 20] [--rounds 5]

Inputs: a batch of seeded uint8 images at the SA-1B decoded size, in pinned host memory.  Prints one JSON line with
  * device preparation alone (CUDA events): ms per batch and achieved bytes/s over the algorithmic bytes (uint8 in, workspace
    written and read, fp32 out), against the H100 SXM data-sheet 3.35 TB/s;
  * pinned uint8 H2D + preparation, against the H2D of the same batch already prepared as pinned fp32;
  * the reference's CPU transform (ResizeLongestSide + norm + pad, oracle/preprocess.py) per image on one thread;
  * the EV-M student forward end to end from pinned uint8 originals against from pinned fp32 prepared images, arms alternated;
and the GPU name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from types import SimpleNamespace as NS

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def _time_ms(fn, iters):
    """Median over `iters` of CUDA-event time of fn() on the current stream."""
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--h", type=int, default=1500)
    ap.add_argument("--w", type=int, default=2250)
    ap.add_argument("--img", type=int, default=1008)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cpu-images", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_preprocess.py measures on a CUDA device; none found")
    from efficientsam3_b200 import _lib, ops
    from efficientsam3_b200.stage1.model import build_image_student_model
    from efficientsam3_b200.stage1.preprocess import get_preprocess_shape, pack_images, prepare_images
    from oracle import preprocess as O

    dev = torch.device("cuda:0")
    _lib.init(0)
    gpu = _gpu_info()
    B, S = args.batch, args.img
    g = torch.Generator().manual_seed(0)
    imgs = [torch.randint(0, 256, (args.h, args.w, 3), dtype=torch.uint8, generator=g) for _ in range(B)]
    packed = pack_images(imgs).pin_memory()
    table = packed.table()
    ho, wo = get_preprocess_shape(args.h, args.w, S)
    nws = ops.image_table_ws_floats(table, packed.data.numel(), S)
    bytes_alg = packed.data.numel() + 8 * nws + 4 * B * 3 * S * S
    src = packed.data.to(dev)
    out = torch.empty(B, 3, S, S, device=dev)
    x_f32, _ = prepare_images(packed, S, device=dev)
    host_f32 = x_f32.cpu().pin_memory()
    dev_f32 = torch.empty_like(x_f32)

    # device preparation alone
    ops.prepare_images_u8(src, table, S, O.MEAN, O.STD, out=out)
    torch.cuda.synchronize()
    prep_ms = _time_ms(lambda: ops.prepare_images_u8(src, table, S, O.MEAN, O.STD, out=out), args.iters)

    # pinned uint8 H2D + preparation vs the H2D of the prepared fp32 batch
    h2d_u8_prep_ms = _time_ms(lambda: prepare_images(packed, S, device=dev, out=out), args.iters)
    h2d_f32_ms = _time_ms(lambda: dev_f32.copy_(host_f32, non_blocking=True), args.iters)

    # the reference transform on the host CPU, one thread
    nthreads = torch.get_num_threads()
    torch.set_num_threads(1)
    O.prepare_image(imgs[0], S)
    t0 = time.perf_counter()
    for i in range(args.cpu_images):
        O.prepare_image(imgs[i % B], S)
    cpu_ms = (time.perf_counter() - t0) * 1e3 / args.cpu_images
    torch.set_num_threads(nthreads)

    # EV-M forward end to end: pinned uint8 originals vs pinned fp32 prepared images, arms alternated
    cfg = NS(MODEL=NS(BACKBONE="efficientvit_b1"), DATA=NS(IMG_SIZE=S), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=S // 14))
    torch.manual_seed(0)
    m = build_image_student_model(cfg).to(dev).eval()

    def from_u8():
        x, _ = prepare_images(packed, S, device=dev, out=out)
        return m(x)

    def from_f32():
        return m(host_f32.to(dev, non_blocking=True))

    with torch.no_grad():
        for fn in (from_u8, from_f32):
            fn()
        torch.cuda.synchronize()
        arms = {"uint8": [], "fp32": []}
        for _ in range(args.rounds):
            for name, fn in (("uint8", from_u8), ("fp32", from_f32)):
                arms[name].append(_time_ms(fn, max(2, args.iters // 4)))
    e2e = {k: statistics.median(v) for k, v in arms.items()}

    print(json.dumps({
        "gpu": gpu, "batch": B, "image": [args.h, args.w], "img_size": S, "resized": [ho, wo],
        "prepare_ms": round(prep_ms, 3),
        "prepare_bytes": bytes_alg,
        "prepare_TBps": round(bytes_alg / (prep_ms * 1e-3) / 1e12, 3),
        "prepare_share_of_3.35TBps": round(bytes_alg / (prep_ms * 1e-3) / HBM_BYTES_PER_S, 3),
        "h2d_uint8_plus_prepare_ms": round(h2d_u8_prep_ms, 3), "h2d_uint8_bytes": packed.data.numel(),
        "h2d_fp32_prepared_ms": round(h2d_f32_ms, 3), "h2d_fp32_bytes": host_f32.numel() * 4,
        "cpu_reference_ms_per_image_1_thread": round(cpu_ms, 1),
        "evm_forward_ms": {k: round(v, 3) for k, v in e2e.items()},
        "evm_forward_ms_rounds": {k: [round(t, 3) for t in v] for k, v in arms.items()},
    }))


if __name__ == "__main__":
    main()
