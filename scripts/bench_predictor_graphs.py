"""Per-click latency of the interactive point-prompt predictor (SAM3InteractiveImagePredictor.predict) with its prompt side
replayed from CUDA graphs (enable_cuda_graphs), launched kernel by kernel (uncaptured()), and as the oracle's eager torch
restatement of the SAM heads (oracle/sam_heads.py) on the same GPU and the same image features.  Prints one JSON line.

    python scripts/bench_predictor_graphs.py [--steps 30] [--warmup 5] [--rounds 3] [--out results.json]

Models: the point segmenter over the SAM3 ViT trunk and over the EV-M student encoder (build_efficientsam3_point_segmenter
("efficientvit", "b1")), both at 1008^2 with their default initialisation (the timing does not depend on the weights).  One
set_image on a seeded 1500 x 2250 uint8 image, then predict with 1, 3, 8 and 12 points (6 output tokens, 12 points and the
padding point: 19 image-to-token keys, more than one 16-key tile), a box, a box plus a point and a point plus a mask_input, each with multimask_output True and False; the predictor's defaults otherwise (hole filling up to 256 px, binary
masks at the original size).  The oracle arm runs without hole filling: its fill_holes labels components with scipy on the CPU.
Per arm and call: the median and p10-p90 of the device time (CUDA events around the call) and of the host time until predict
returns (it returns host arrays, so both include the copy out).  The arms run in turn, `--rounds` times, so that a drift of the
machine falls on all of them.  `graph_equals_uncaptured` checks masks, ious and low-res logits bit for bit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_text import gpu_info  # noqa: E402


def percentile(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, max(0, int(round(q / 100 * (len(xs) - 1)))))]


def sample(fn, steps, dev_ms, host_ms):
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        t0 = time.perf_counter()
        fn()
        host_ms.append((time.perf_counter() - t0) * 1e3)
        e1.record()
        e1.synchronize()
        dev_ms.append(e0.elapsed_time(e1))


def stats(xs):
    return dict(median=round(percentile(xs, 50), 4), p10=round(percentile(xs, 10), 4), p90=round(percentile(xs, 90), 4))


def cases(low_prev):
    rng = np.random.default_rng(0)
    pts = rng.uniform([0, 0], [2250, 1500], size=(8, 2))
    lab = rng.integers(0, 2, size=8)
    box = np.array([300.0, 200.0, 1800.0, 1300.0])
    pts12 = np.concatenate([pts, rng.uniform([0, 0], [2250, 1500], size=(4, 2))])     # drawn after: the first 8 stay as they were
    lab12 = np.concatenate([lab, rng.integers(0, 2, size=4)])
    return {"1 point": dict(point_coords=pts[:1], point_labels=lab[:1]),
            "3 points": dict(point_coords=pts[:3], point_labels=lab[:3]),
            "8 points": dict(point_coords=pts, point_labels=lab),
            "12 points": dict(point_coords=pts12, point_labels=lab12),
            "box": dict(box=box),
            "box + point": dict(box=box, point_coords=pts[:1], point_labels=lab[:1]),
            "point + mask_input": dict(point_coords=pts[:1], point_labels=lab[:1], mask_input=low_prev)}


def oracle_call(pred, seg, kw, mm):
    """oracle/sam_heads.predict on the device, on the predictor's own image features; returns host arrays as predict does."""
    from oracle import sam_heads as OH
    f, S, hw = seg._features, seg.image_size, pred._orig_hw[0]
    sd = {k: v for k, v in seg.state_dict().items()}
    sd_md = {k[len("sam_mask_decoder."):]: v for k, v in sd.items() if k.startswith("sam_mask_decoder.")}
    sd_pe = {k[len("sam_prompt_encoder."):]: v for k, v in sd.items() if k.startswith("sam_prompt_encoder.")}
    emb = pred.get_image_embedding()
    hr = (f["feat_s0"].permute(0, 3, 1, 2).contiguous(), f["feat_s1"].permute(0, 3, 1, 2).contiguous())
    sc = torch.tensor([S / hw[1], S / hw[0]], device=emb.device)

    def call():
        dev = emb.device
        pc = pl = bx = mi = None
        if "point_coords" in kw:
            pc = (torch.as_tensor(kw["point_coords"], dtype=torch.float32, device=dev) * sc)[None]
            pl = torch.as_tensor(kw["point_labels"], dtype=torch.int32, device=dev)[None]
        if "box" in kw:
            bx = (torch.as_tensor(kw["box"], dtype=torch.float32, device=dev).reshape(-1, 2, 2) * sc).reshape(-1, 4)
        if "mask_input" in kw:
            mi = torch.as_tensor(kw["mask_input"], dtype=torch.float32, device=dev)[None]
        with torch.no_grad(), torch.device(dev):        # the oracle's own tensors (padding point, box labels) on the GPU too
            m, i, low = OH.predict(sd_pe, sd_md, emb, hr, pc, pl, bx, mi, S, hw, multimask_output=mm, return_logits=False,
                                   max_hole_area=0.0)
        return m[0].float().cpu().numpy(), i[0].float().cpu().numpy(), low[0].float().cpu().numpy()
    return call


def bench_model(name, seg, args, dev):
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor
    seg = seg.to(dev).eval()
    pred = SAM3InteractiveImagePredictor(seg).enable_cuda_graphs(max_graphs=16)
    image = np.random.default_rng(1).integers(0, 256, size=(1500, 2250, 3), dtype=np.uint8)
    pred.set_image(image)
    low_prev = pred.predict(point_coords=np.array([[1100.0, 700.0]]), point_labels=np.array([1]), multimask_output=False)[2]
    rows = []
    for case, kw in cases(low_prev).items():
        for mm in (True, False):
            graph = lambda: pred.predict(multimask_output=mm, **kw)

            def uncaptured():
                with seg.uncaptured():
                    return pred.predict(multimask_output=mm, **kw)
            arms = dict(graph=graph, uncaptured=uncaptured, oracle=oracle_call(pred, seg, kw, mm))
            g, u = graph(), uncaptured()
            equal = all(np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)) for a, b in zip(g, u))
            launches = pred.graph_launches_per_step
            for fn in arms.values():
                for _ in range(args.warmup):
                    fn()
            dev_ms = {k: [] for k in arms}
            host_ms = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, fn in arms.items():
                    sample(fn, args.steps, dev_ms[k], host_ms[k])
            r = dict(model=name, prompt=case, multimask_output=mm, graph_equals_uncaptured=equal, es3_launches=launches,
                     **{f"{k}_device_ms": stats(dev_ms[k]) for k in arms}, **{f"{k}_host_ms": stats(host_ms[k]) for k in arms})
            print(json.dumps(r), file=sys.stderr, flush=True)
            rows.append(r)
    pred.enable_cuda_graphs(False)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_predictor_graphs: needs a CUDA device")
    dev = torch.device("cuda:0")
    from efficientsam3_b200.model.sam1_task import Sam3PointPromptSegmenter
    from efficientsam3_b200.model_builder import build_efficientsam3_point_segmenter
    torch.manual_seed(0)
    res = dict(info=gpu_info(dev), steps=args.steps, rounds=args.rounds, rows=[])
    res["rows"] += bench_model("SAM3 ViT", Sam3PointPromptSegmenter(), args, dev)
    res["rows"] += bench_model("EV-M student", build_efficientsam3_point_segmenter("efficientvit", "b1"), args, dev)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
