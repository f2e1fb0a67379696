"""Cost of synchronised BatchNorm on the EV-M stage-1 KD step: the same data-parallel step with per-rank BatchNorm2d and with
nn.SyncBatchNorm (convert_sync_batchnorm), alternated in one run, and the number of BN exchanges (all-gathers) per step.

    torchrun --nproc_per_node 8 scripts/bench_syncbn.py [--batch 32] [--img 1008] [--steps 20] [--warmup 5] [--rounds 3]

Needs at least two ranks (with one rank a SyncBatchNorm does not synchronise, so there is nothing to measure) and one GPU per rank
(NCCL).  Prints one JSON line from rank 0: per-arm median step time (CUDA events on each rank, max over ranks), the difference,
the exchanges per step, and the GPU name and power limit the numbers were taken on.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace as NS

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backbone", default="efficientvit_b1")
    ap.add_argument("--batch", type=int, default=32, help="images per GPU")
    ap.add_argument("--img", type=int, default=1008)
    ap.add_argument("--embed", type=int, default=72)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3, help="BN / SyncBN windows, alternated")
    a = ap.parse_args()

    dist.init_process_group("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    if world < 2:
        raise SystemExit("bench_syncbn: needs >= 2 ranks (torchrun --nproc_per_node N, N >= 2); with one rank SyncBatchNorm does not "
                         "synchronise")
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    from efficientsam3_b200 import sync_bn
    from efficientsam3_b200.stage1.losses import kd_train_step
    from efficientsam3_b200.stage1.model import build_image_student_model
    from efficientsam3_b200.stage1.optim import FlatAdamW

    cfg = NS(MODEL=NS(BACKBONE=a.backbone), DATA=NS(IMG_SIZE=a.img), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=a.embed))
    g = torch.Generator().manual_seed(1234 + rank)
    x = torch.randn(a.batch, 3, a.img, a.img, generator=g).to(dev)
    t = torch.randn(a.batch, 1024, a.embed, a.embed, generator=g).to(dev)
    sizes = [(3, a.img, a.img)] * a.batch
    arms = {}
    for arm in ("bn", "syncbn"):
        torch.manual_seed(0)
        m = build_image_student_model(cfg).to(dev)
        if arm == "syncbn":
            m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
        m.train()
        arms[arm] = (m, FlatAdamW(m, lr=1e-4))

    def window(arm, steps):
        m, opt = arms[arm]
        e0 = sync_bn.exchanges
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        start.record()
        for _ in range(steps):
            kd_train_step(m, opt, x, t, sizes, 1.0)
        end.record()
        torch.cuda.synchronize()
        ms = torch.tensor([start.elapsed_time(end) / steps], device=dev)
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return ms.item(), (sync_bn.exchanges - e0) / steps

    for arm in arms:
        window(arm, a.warmup)
    times = {arm: [] for arm in arms}
    exch = {}
    for _ in range(a.rounds):
        for arm in arms:
            ms, ex = window(arm, a.steps)
            times[arm].append(ms)
            exch[arm] = ex
    if rank == 0:
        med = {arm: statistics.median(v) for arm, v in times.items()}
        print(json.dumps({"metric": "syncbn_step_ms", "backbone": a.backbone, "world": world, "batch_per_gpu": a.batch, "img": a.img,
                          "bn_ms": med["bn"], "syncbn_ms": med["syncbn"], "delta_ms": med["syncbn"] - med["bn"],
                          "bn_ms_all": times["bn"], "syncbn_ms_all": times["syncbn"],
                          "exchanges_per_step": exch["syncbn"], "exchanges_per_step_bn": exch["bn"], "gpu": _gpu_info()}))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
