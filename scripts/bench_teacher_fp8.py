"""The frozen SAM3 ViT teacher (32 blocks, 1008^2 -> 1024 x 72 x 72) in three modes on one GPU: bf16 (the default), block-scaled
FP8 linear layers (ViT.enable_fp8()), and FP8 linear layers + FP8 attention (ViT.enable_fp8(attention=True)).  Prints the card and
its power limit, then one JSON line:

    python scripts/bench_teacher_fp8.py [--batch 8] [--rounds 10] [--gemm-iters 20] [--attn-iters 50]

  * teacher img/s per mode: every mode warmed, then `rounds` forwards of each, the modes taking turns, each timed with CUDA events
    around one forward; median and p10 - p90 over the rounds
  * the four FP8 GEMMs at the teacher's shapes (M = batch * 5184 tokens) with their real epilogues, timed with CUDA events over
    `gemm-iters` launches, as achieved TFLOP/s (2 M N K / time) and as a share of the H100 SXM data sheet's dense FP8 rate
    (1,979 TFLOP/s at 700 W); the bf16 GEMM of the same layer beside it
  * the attention kernels alone at the teacher's two shapes (24-windows on 72 x 72, L = 576, and global, L = 5184; batch `batch`,
    16 heads): es3_attention_tc_bf16 against es3_attention_fp8 (its K / V pre-pass included), CUDA events over `attn-iters`
    launches, as achieved TFLOP/s (4 B HW L C / time) and as a share of the data sheet's dense rate of each kernel's MMA type (989 bf16, 1,979 e4m3)
  * each kernel family's share of the teacher forward per mode (ops.Profiler, one profiled forward after the timed rounds)
  * the embedding differences on the timed inputs: fp8 linears vs bf16, and fp8 attention vs bf16 and vs fp8 linears: rel-L2 and
    per-token cosine (mean, min)
Weights are the module's seeded random initialisation; neither time depends on their values.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

FP8_PEAK_TFLOPS = 1979.0          # H100 SXM data sheet, dense e4m3
BF16_PEAK_TFLOPS = 989.0


def gpu_info(dev):
    name = torch.cuda.get_device_name(dev)
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
        pl, mx = [s.strip() for s in out.split(",")[:2]]
        return dict(gpu=name, power_limit_w=float(pl), sm_max_mhz=float(mx))
    except Exception as e:   # nvidia-smi missing: the numbers are still measured, the card's limit is then unknown
        return dict(gpu=name, power_limit_w=None, note=f"nvidia-smi: {e}")


def _pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, max(0, round(q * (len(xs) - 1))))]


def _timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return out, e0.elapsed_time(e1)


def _gemm_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def gemm_legs(dev, batch, iters):
    from efficientsam3_b200 import ops
    H = W = 72
    C, Hd = 1024, 4736
    M = batch * H * W
    g = torch.Generator(device=dev).manual_seed(0)
    tab = torch.randn(24 * 24, 32, 2, device=dev, generator=g)
    x1 = torch.randn(M, C, device=dev, generator=g)
    xh = torch.randn(M, Hd, device=dev, generator=g).to(torch.bfloat16)
    res = torch.randn(M, C, device=dev, generator=g)
    rows = []
    for name, N, K in (("qkv", 3 * C, C), ("proj", C, C), ("fc1", Hd, C), ("fc2", C, Hd)):
        w = torch.randn(N, K, device=dev, generator=g) * 0.02
        b = torch.randn(N, device=dev, generator=g)
        qw, sw = ops.pack_weight_e4m3(w)
        a16 = (x1 if K == C else xh.float()).to(torch.bfloat16)
        qa, sa = ops.quantize_e4m3(a16)
        wb = w.to(torch.bfloat16)
        if name == "qkv":
            f8 = lambda: ops.gemm_fp8(qa, sa, qw, sw, b, rope=(tab, 2 * C, H, W, 24))
            f16 = lambda: ops.gemm(a16, wb, bias=b, rope=(tab, 2 * C, H, W, 24))
        elif name == "fc1":
            f8 = lambda: ops.gemm_fp8(qa, sa, qw, sw, b, act="gelu", out_dtype=ops.E4M3)
            f16 = lambda: ops.gemm(a16, wb, bias=b, act="gelu")
        else:
            f8 = lambda: ops.gemm_fp8(qa, sa, qw, sw, b, residual=res, out_dtype=torch.float32)
            f16 = lambda: ops.gemm(a16, wb, bias=b, residual=res, out_dtype=torch.float32)
        ms8, ms16 = _gemm_ms(f8, iters), _gemm_ms(f16, iters)
        fl = 2.0 * M * N * K
        rows.append(dict(layer=name, M=M, N=N, K=K, fp8_ms=round(ms8, 4), fp8_tflops=round(fl / ms8 / 1e9, 1),
                         fp8_share_of_1979=round(fl / ms8 / 1e9 / FP8_PEAK_TFLOPS, 3), bf16_ms=round(ms16, 4),
                         bf16_tflops=round(fl / ms16 / 1e9, 1)))
    return rows


def attention_legs(dev, batch, iters):
    from efficientsam3_b200 import ops
    H = W = 72
    heads, C = 16, 1024
    g = torch.Generator(device=dev).manual_seed(2)
    qkv = torch.randn(batch * H * W, 3 * C, device=dev, generator=g).to(torch.bfloat16)
    rows = []
    for win in (24, 0):
        L = win * win if win else H * W
        f16 = lambda: ops.attention(qkv, batch, H, W, C, heads, win, 0.125, impl="tc")
        f8 = lambda: ops.attention_fp8(qkv, batch, H, W, C, heads, win, 0.125)
        ms16, ms8 = _gemm_ms(f16, iters), _gemm_ms(f8, iters)
        ms16, ms8 = min(ms16, _gemm_ms(f16, iters)), min(ms8, _gemm_ms(f8, iters))    # two alternating windows each
        fl = 4.0 * batch * H * W * L * C
        rows.append(dict(win=win, L=L, bf16_ms=round(ms16, 4), bf16_tflops=round(fl / ms16 / 1e9, 1),
                         bf16_share_of_989=round(fl / ms16 / 1e9 / BF16_PEAK_TFLOPS, 3), fp8_ms=round(ms8, 4),
                         fp8_tflops=round(fl / ms8 / 1e9, 1), fp8_share_of_1979=round(fl / ms8 / 1e9 / FP8_PEAK_TFLOPS, 3),
                         fp8_speedup=round(ms16 / ms8, 3)))
    return rows


def _family(tag):
    return tag.split("[")[0]


def family_shares(model, x):
    """Each kernel family's share of one profiled forward (CUDA events around every launch)."""
    from efficientsam3_b200 import ops
    prof = ops.Profiler()
    ops.set_profiler(prof)
    try:
        model(x)
    finally:
        ops.set_profiler(None)
    agg = {}
    for tag, a in prof.summary().items():
        agg[_family(tag)] = agg.get(_family(tag), 0.0) + a["ms"]
    total = sum(agg.values())
    return {k: dict(ms=round(v, 3), share=round(v / total, 4)) for k, v in sorted(agg.items(), key=lambda kv: -kv[1])}


def _diff(y, ref):
    a = y.double().flatten(2).transpose(1, 2).reshape(-1, y.shape[1])
    b = ref.double().flatten(2).transpose(1, 2).reshape(-1, ref.shape[1])
    cos = (a * b).sum(1) / (a.norm(dim=1) * b.norm(dim=1))
    return dict(rel_l2=float((a - b).norm() / b.norm()), token_cos_mean=round(cos.mean().item(), 6), token_cos_min=round(cos.min().item(), 6))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--gemm-iters", type=int, default=20)
    ap.add_argument("--attn-iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_teacher_fp8: needs a CUDA device (nothing is timed on the CPU)")
    dev = torch.device("cuda:0")
    info = gpu_info(dev)
    print(f"# {info['gpu']}, power limit {info.get('power_limit_w')} W", flush=True)

    from efficientsam3_b200.stage1.model import SAM3ImageTeacherEncoder
    torch.manual_seed(0)
    t16 = SAM3ImageTeacherEncoder(embed_size=72).to(dev)
    t8 = SAM3ImageTeacherEncoder(embed_size=72).to(dev)
    t8.load_state_dict(t16.state_dict())
    t8.enable_fp8()
    ta = SAM3ImageTeacherEncoder(embed_size=72).to(dev)
    ta.load_state_dict(t16.state_dict())
    ta.enable_fp8(attention=True)
    modes = {"bf16": t16, "fp8": t8, "fp8_attn": ta}
    x = torch.randn(args.batch, 3, 1008, 1008, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    for _ in range(2):
        for m in modes.values():
            m(x)
    torch.cuda.synchronize()
    ms = {k: [] for k in modes}
    ys = {}
    for _ in range(args.rounds):
        for k, m in modes.items():
            ys[k], t = _timed(lambda: m(x))
            ms[k].append(t)
    teacher = {}
    for k, v in ms.items():
        ips = [args.batch / m * 1e3 for m in v]
        teacher[k] = dict(img_per_s_median=round(statistics.median(ips), 2), img_per_s_p10=round(_pct(ips, 0.1), 2),
                          img_per_s_p90=round(_pct(ips, 0.9), 2), ms_median=round(statistics.median(v), 2))
    teacher["fp8_over_bf16"] = round(teacher["fp8"]["img_per_s_median"] / teacher["bf16"]["img_per_s_median"], 3)
    teacher["fp8_attn_over_fp8"] = round(teacher["fp8_attn"]["img_per_s_median"] / teacher["fp8"]["img_per_s_median"], 3)
    teacher["fp8_attn_over_bf16"] = round(teacher["fp8_attn"]["img_per_s_median"] / teacher["bf16"]["img_per_s_median"], 3)

    diff = _diff(ys["fp8"], ys["bf16"])
    diff_attn = dict(vs_bf16=_diff(ys["fp8_attn"], ys["bf16"]), vs_fp8_linears=_diff(ys["fp8_attn"], ys["fp8"]))
    shares = {k: family_shares(m, x) for k, m in modes.items()}
    attn = attention_legs(dev, args.batch, args.attn_iters)
    for r in attn:
        print(f"# attention L={r['L']} B={args.batch}: bf16 tc {r['bf16_ms']:.3f} ms {r['bf16_tflops']} TFLOP/s "
              f"({100 * r['bf16_share_of_989']:.1f}% of 989)   fp8 {r['fp8_ms']:.3f} ms {r['fp8_tflops']} TFLOP/s "
              f"({100 * r['fp8_share_of_1979']:.1f}% of 1979)   speedup {r['fp8_speedup']}", flush=True)
    for k, sh in shares.items():
        print(f"# {k} forward shares: " + ", ".join(f"{n} {100 * v['share']:.1f}%" for n, v in list(sh.items())[:6]), flush=True)

    gemms = gemm_legs(dev, args.batch, args.gemm_iters)
    for r in gemms:
        print(f"# {r['layer']:5s} M={r['M']} N={r['N']} K={r['K']}: fp8 {r['fp8_ms']:.3f} ms {r['fp8_tflops']} TFLOP/s "
              f"({100 * r['fp8_share_of_1979']:.1f}% of 1979)   bf16 {r['bf16_ms']:.3f} ms {r['bf16_tflops']} TFLOP/s", flush=True)
    print(f"# teacher B={args.batch}: bf16 {teacher['bf16']['img_per_s_median']} img/s, fp8 {teacher['fp8']['img_per_s_median']} img/s, "
          f"fp8 + fp8 attention {teacher['fp8_attn']['img_per_s_median']} img/s; fp8 vs bf16 embedding rel-L2 {diff['rel_l2']:.3e}, "
          f"token cosine mean {diff['token_cos_mean']} min {diff['token_cos_min']}; fp8 attention vs bf16 rel-L2 "
          f"{diff_attn['vs_bf16']['rel_l2']:.3e} (cos min {diff_attn['vs_bf16']['token_cos_min']}), vs fp8 linears rel-L2 "
          f"{diff_attn['vs_fp8_linears']['rel_l2']:.3e} (cos min {diff_attn['vs_fp8_linears']['token_cos_min']})", flush=True)
    print(json.dumps(dict(**info, batch=args.batch, img=1008, rounds=args.rounds, teacher=teacher, fp8_vs_bf16_embedding=diff,
                          fp8_attention_embedding=diff_attn, attention=attn, forward_shares=shares, gemms=gemms)))


if __name__ == "__main__":
    main()
