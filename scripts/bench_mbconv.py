"""Time the fused MBConv kernels (mbconv_tc, mbconv_tc_s2, dwproj_tc) one instantiation at a time, at the shapes the EV-M
student runs them at in bench.py (batch 32, 1024^2 input), and check each output against the op-by-op statement.

    python scripts/bench_mbconv.py [--lib PATH] [--batch 32] [--img 1024] [--seconds 1.0] [--json OUT] [--save-outputs DIR]

--lib loads another build of libes3.so (same C ABI), so that two builds can be timed alternately, one process each.  Prints one
JSON line: per instantiation the kernel time (CUDA events over enough launches to run for --seconds after warm-up), the
compulsory HBM bytes (each input read once, each output written once), the fraction of the 3.35 TB/s HBM3 bound that is, and
the max error / scale against the fp32 statement; plus the GPU name, power limit and SM clock the numbers were taken on.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BPS = 3.35e12    # H100 SXM data sheet


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def cases(img):
    """(name, kind, cin, mid, cout, stride, input side) of the EV-M blocks the three kernels run, in network order."""
    s = img // 2     # after the stem
    return [("mbconv_tc_s2<16,64,32>", "mbconv", 16, 64, 32, 2, s),
            ("mbconv_tc<32,128,32>", "mbconv", 32, 128, 32, 1, s // 2),
            ("mbconv_tc_s2<32,128,64>", "mbconv", 32, 128, 64, 2, s // 2),
            ("mbconv_tc<64,256,64>", "mbconv", 64, 256, 64, 1, s // 4),
            ("mbconv_tc_s2<64,256,128>", "mbconv", 64, 256, 128, 2, s // 4),
            ("mbconv_tc<128,512,128>", "mbconv", 128, 512, 128, 1, s // 8),
            ("mbconv_tc_s2<128,512,256>", "mbconv", 128, 512, 256, 2, s // 8),
            ("dwproj_tc<512,128>", "dwproj", 0, 512, 128, 1, s // 8),
            ("dwproj_tc<1024,256>", "dwproj", 0, 1024, 256, 1, s // 16)]


def _time(run, seconds):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        run()
    e1.record()
    torch.cuda.synchronize()
    n = max(10, math.ceil(seconds * 1e3 / (e0.elapsed_time(e1) / 5)))
    e0.record()
    for _ in range(n):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, n


def bench_case(ops, name, kind, cin, mid, cout, stride, side, B, seconds, dev, save_dir=None):
    g = torch.Generator().manual_seed(mid + side + stride)
    bf = lambda t: t.to(torch.bfloat16).to(dev)
    H = W = side
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    wdw = torch.randn(mid, 1, 3, 3, generator=g) / 3
    wdw9 = wdw.reshape(mid, 9).t().contiguous().to(dev)
    b2 = (torch.randn(mid, generator=g) * 0.2).to(dev)
    w3 = bf(torch.randn(cout, mid, generator=g) / math.sqrt(mid))
    s3 = (torch.rand(cout, generator=g) + 0.5).to(dev)
    b3 = (torch.randn(cout, generator=g) * 0.2).to(dev)
    if kind == "dwproj":
        m = bf(torch.randn(B, H, W, mid, generator=g))
        x = bf(torch.randn(B, H, W, cout, generator=g))
        run = lambda: ops.dwproj(m, wdw9, b2, w3, s3, b3, residual=x)
        nbytes = 2 * (m.numel() + 2 * x.numel())
        d = F.conv2d(m.float().permute(0, 3, 1, 2), wdw.to(dev).to(torch.bfloat16).float(), b2, padding=1, groups=mid)
        resid = x.float().permute(0, 3, 1, 2)
    else:
        x = bf(torch.randn(B, H, W, cin, generator=g))
        w1 = bf(torch.randn(mid, cin, generator=g) / math.sqrt(cin))
        s1 = (torch.rand(mid, generator=g) + 0.5).to(dev)
        b1 = (torch.randn(mid, generator=g) * 0.2).to(dev)
        res = stride == 1
        run = lambda: ops.mbconv_fused(x, w1, s1, b1, wdw9, b2, w3, s3, b3, stride, res, "hswish")
        nbytes = 2 * (x.numel() + B * Ho * Wo * cout)
        xn = x.float().permute(0, 3, 1, 2)
        e = F.hardswish(F.conv2d(xn, w1.float()[:, :, None, None]) * s1.view(1, -1, 1, 1) + b1.view(1, -1, 1, 1))
        d = F.conv2d(e.to(torch.bfloat16).float(), wdw.to(dev), b2, stride=stride, padding=1, groups=mid)
        del e
        resid = xn if res else None
    y = run()
    assert y is not None, f"{name}: not instantiated"
    if save_dir:
        # the kernel's bf16 output bits, so that two builds can be compared bit for bit (inputs are seeded per instantiation)
        tag = "".join(ch if ch.isalnum() else "_" for ch in name).strip("_")
        torch.save(y.view(torch.int16).cpu(), os.path.join(save_dir, f"{tag}.pt"))
    d = F.hardswish(d).to(torch.bfloat16).float()
    ref = F.conv2d(d, w3.float()[:, :, None, None]) * s3.view(1, -1, 1, 1) + b3.view(1, -1, 1, 1)
    del d
    if resid is not None:
        ref = ref + resid
    ref = ref.permute(0, 2, 3, 1)
    err = ((y.float() - ref).abs().max() / (ref.abs().max() + 1e-12)).item()
    del ref, resid
    torch.cuda.empty_cache()
    ms, n = _time(run, seconds)
    return {"name": name, "shape": [B, H, W, cin or mid, mid, cout, stride], "ms": round(ms, 4), "launches": n,
            "bytes": nbytes, "hbm_frac": round(nbytes / HBM_BPS * 1e3 / ms, 3), "max_err_over_scale": err, "ok": err <= 1e-2}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="libes3.so to load instead of the in-tree build")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--img", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=1.0, help="timed window per instantiation (after warm-up)")
    ap.add_argument("--only", default=None, help="substring of the instantiation names to run")
    ap.add_argument("--json", default=None, help="also write the result line to this file")
    ap.add_argument("--save-outputs", default=None, metavar="DIR",
                    help="write each instantiation's output (bf16 bits as int16, <name>.pt) under DIR")
    args = ap.parse_args()
    if args.save_outputs:
        os.makedirs(args.save_outputs, exist_ok=True)
    if not torch.cuda.is_available():
        sys.exit("bench_mbconv: no CUDA device")
    from efficientsam3_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = Path(args.lib).resolve()
    from efficientsam3_b200 import ops
    _lib.init(0)
    dev = torch.device("cuda", 0)
    rows = [bench_case(ops, *c, args.batch, args.seconds, dev, args.save_outputs) for c in cases(args.img)
            if not args.only or args.only in c[0]]
    out = {"gpu": _gpu_info(), "lib": str(_lib.LIB_PATH), "batch": args.batch, "img": args.img, "kernels": rows,
           "total_ms": round(sum(r["ms"] for r in rows), 4), "total_bytes": sum(r["bytes"] for r in rows),
           "all_ok": all(r["ok"] for r in rows)}
    line = json.dumps(out)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")
    if not out["all_ok"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
