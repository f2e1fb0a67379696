"""Automatic mask generation on native kernels (amg.cu) and SamAutomaticMaskGenerator end to end.

- es3_amg_mask_stats: counts, boxes, stability, filters and the arena are exactly what torch computes from ops.bilinear_nchw's
  output (which pins the shared bilinear expression); against an fp64 bilinear, the counts differ by at most the pixels whose
  fp64 value lies within the kernel's rounding bound of a threshold.
- es3_box_nms: equal to oracle.amg.nms_stable (ties, zero-area boxes, N from 1 to 12288) and, on distinct scores, to
  torchvision's batched_nms on the CPU.
- es3_amg_rle: equal to oracle.amg.mask_to_rle_pytorch of the uncropped ops.bilinear_nchw binarisation; its uint8 masks are the
  same masks.
- Every entry point: NaN-prefilled outputs keep their sentinel bits past the written region, two runs are bit-identical, and a
  declined shape writes nothing.
- The generator with the synthetic decoder reproduces the reference's committed records; on a seeded point segmenter it equals
  oracle.amg.generate fed the same decode_prompts outputs, in both precision modes and with CUDA graphs on and off.
- amg.cu compiles without spills or stack frames.
"""
import subprocess
import types

import numpy as np
import pytest
import torch

import ref_sam as R
from bounds import TAIL, _INT, _assert_untouched, _flat_out, _gen, _lib, _st
from oracle import amg as OA
from test_amg_cpu import assert_records_equal, case_kwargs, load_cases

gpu = pytest.mark.gpu


def _bits(t):
    return t.view(_INT[t.dtype]) if t.dtype in _INT else t


def _declined(lib, name, args, bufs):
    from efficientsam3_b200._lib import Es3Error
    before = [b.clone() for b in bufs]
    with pytest.raises(Es3Error):
        lib.call(name, *args)
    torch.cuda.synchronize()
    for b, b0 in zip(bufs, before):
        assert torch.equal(_bits(b), _bits(b0)), f"{name}: a declined call wrote"


# ----------------------------------------------------------------------------------------------------------- mask statistics
class _Arena:
    """A NaN-prefilled arena of `cap` slots with TAIL sentinel cells past each buffer (the int ones are views of fp32 storage)."""

    def __init__(self, cap, Hi, Wi, cuda):
        self.cap, self.Hi, self.Wi = cap, Hi, Wi
        self.bufs = {k: _flat_out(n, torch.float32, cuda)[0] for k, n in
                     (("low", cap * Hi * Wi), ("box", cap * 4), ("iou", cap), ("stab", cap), ("point", cap))}
        self.bufs["count"] = torch.zeros(1, dtype=torch.int32, device=cuda)

    def ptrs(self):
        b = self.bufs
        return [b["low"].data_ptr(), b["box"].data_ptr(), b["iou"].data_ptr(), b["stab"].data_ptr(), b["point"].data_ptr(),
                b["count"].data_ptr()]

    def clone(self):
        a = _Arena.__new__(_Arena)
        a.cap, a.Hi, a.Wi = self.cap, self.Hi, self.Wi
        a.bufs = {k: v.clone() for k, v in self.bufs.items()}
        return a

    def view(self, n):
        b = self.bufs
        return dict(low=b["low"][:n * self.Hi * self.Wi].view(n, self.Hi, self.Wi), box=b["box"].view(torch.int32)[:n * 4].view(n, 4),
                    iou=b["iou"][:n], stab=b["stab"][:n], point=b["point"].view(torch.int32)[:n])

    def untouched_past(self, n):
        sizes = dict(low=self.Hi * self.Wi, box=4, iou=1, stab=1, point=1)
        for k, per in sizes.items():
            buf = self.bufs[k]
            inside = torch.zeros(buf.numel(), dtype=torch.bool, device=buf.device)
            inside[:n * per] = True
            _assert_untouched(buf, inside, f"arena {k}")


def _stats_ref(low, iou, crop, orig_hw, thr, off, iou_t, stab_t, point_base):
    """What the kernel must produce, by torch on ops.bilinear_nchw's output: (survivor mask indices, boxes, stability)."""
    from efficientsam3_b200 import ops
    P, K, Hi, Wi = low.shape
    x0, y0, x1, y1 = crop
    high = ops.bilinear_nchw(low, y1 - y0, x1 - x0)[0].flatten(0, 1)
    io = iou.flatten()
    keep = torch.ones(P * K, dtype=torch.bool, device=low.device)
    if iou_t > 0:
        keep &= io > iou_t
    stab = OA.calculate_stability_score(high, thr, off)
    if stab_t > 0:
        keep &= stab >= stab_t
    boxes = OA.batched_mask_to_box(high > thr)
    keep &= ~OA.is_box_near_crop_edge(boxes, list(crop), [0, 0, orig_hw[1], orig_hw[0]])
    idx = keep.nonzero()[:, 0]
    return idx, boxes[idx].int(), stab[idx], high


def _logits(P, K, Hi, Wi, kind, g, cuda):
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, Hi, device=cuda), torch.linspace(-1, 1, Wi, device=cuda), indexing="ij")
    c = torch.rand(P, K, 2, 1, 1, device=cuda, generator=g) * 1.6 - 0.8
    r = torch.rand(P, K, 1, 1, device=cuda, generator=g) * 0.5 + 0.05
    amp = torch.rand(P, K, 1, 1, device=cuda, generator=g) * 30 + 2
    d2 = (yy - c[:, :, 1]) ** 2 + (xx - c[:, :, 0]) ** 2
    low = amp * (torch.exp(-d2 / (2 * r * r)) - 0.5) + torch.randn(P, K, Hi, Wi, device=cuda, generator=g)
    if kind == "empty":
        low = -low.abs() - 1.5
    return low.contiguous()


# (P, K, Hi, Wi, crop XYXY, orig (h, w), kind): upsampling, downsampling (a crop smaller than the low-res grid), non-square,
# M = P K not a multiple of the 256-thread tile, an all-empty batch, rows too wide to stage in shared memory
STATS = [
    (4, 3, 24, 24, (0, 0, 200, 150), (150, 200), "bumps"),
    (7, 3, 288, 288, (30, 20, 160, 120), (150, 200), "bumps"),
    (90, 3, 16, 20, (100, 50, 357, 212), (300, 400), "bumps"),
    (5, 3, 32, 32, (0, 0, 77, 41), (41, 77), "empty"),
    (2, 3, 6, 4200, (10, 0, 60, 30), (30, 70), "bumps"),
    (64, 3, 72, 72, (200, 100, 700, 450), (450, 700), "bumps"),
]


@gpu
@pytest.mark.parametrize("P,K,Hi,Wi,crop,orig,kind", STATS)
@pytest.mark.parametrize("filters", [(0.5, 0.6), (0.0, 0.0)])
def test_amg_mask_stats(cuda, P, K, Hi, Wi, crop, orig, kind, filters):
    lib = _lib(cuda)
    g = _gen(cuda, "stats", P, Hi, Wi, crop)
    low = _logits(P, K, Hi, Wi, kind, g, cuda)
    iou = torch.rand(P, K, device=cuda, generator=g)
    iou_t, stab_t = filters
    thr, off, base = 0.0, 1.0, 11
    M = P * K
    cap = M + 3
    arena = _Arena(cap, Hi, Wi, cuda)
    arena.bufs["count"].fill_(2)                 # appends after what the arena already holds
    ws = torch.empty(lib.size("es3_amg_mask_stats_ws_floats", M), dtype=torch.int32, device=cuda)
    args = lambda a: [low.data_ptr(), iou.data_ptr(), M, K, Hi, Wi, *crop, orig[1], orig[0], thr, off, iou_t, stab_t, base,
                      ws.data_ptr(), *a.ptrs(), cap, _st()]
    a1, a2 = arena.clone(), arena.clone()
    lib.call("es3_amg_mask_stats", *args(a1))
    lib.call("es3_amg_mask_stats", *args(a2))
    for k in a1.bufs:
        assert torch.equal(_bits(a1.bufs[k]), _bits(a2.bufs[k])), f"two runs differ in {k}"
    idx, boxes, stab, high = _stats_ref(low, iou, crop, orig, thr, off, iou_t, stab_t, base)
    n = int(a1.bufs["count"].item())
    assert n == 2 + idx.numel(), (n, idx.numel())
    got = a1.view(n)
    sl = slice(2, n)
    assert torch.equal(got["box"][sl], boxes), "boxes"
    assert torch.equal(_bits(got["iou"][sl]), _bits(iou.flatten()[idx])), "iou"
    assert torch.equal(got["stab"][sl].isnan(), stab.isnan()) and torch.equal(got["stab"][sl].nan_to_num(7.0), stab.nan_to_num(7.0))
    assert torch.equal(got["point"][sl], (base + idx // K).int()), "point index"
    assert torch.equal(_bits(got["low"][sl]), _bits(low.flatten(0, 1)[idx])), "arena logits"
    assert bool(got["iou"][:2].isnan().all()), "the slots before the count were written"
    a1.untouched_past(n)
    if kind == "empty":
        assert idx.numel() == 0 or filters == (0.0, 0.0)
    # against fp64: the kernel's counts move only by pixels within fp32 rounding of a threshold
    Ho, Wo = crop[3] - crop[1], crop[2] - crop[0]
    ref64, bound = R.bilinear(low.flatten(0, 1).double(), Ho, Wo)
    for t in (thr + off, thr - off):
        cnt32 = (high > t).sum((1, 2))
        cnt64 = (ref64 > t).sum((1, 2))
        band = ((ref64 - t).abs() <= bound).sum((1, 2))
        assert bool(((cnt32 - cnt64).abs() <= band).all()), f"counts at {t} move beyond the rounding band"
    # declined: M not a multiple of K, a crop outside the image; neither writes
    before = [a1.bufs[k] for k in a1.bufs] + [ws]
    bad = args(a1)
    bad[3] = M + 1
    _declined(lib, "es3_amg_mask_stats", bad, before)
    bad = args(a1)
    bad[8] = orig[1] + 1
    _declined(lib, "es3_amg_mask_stats", bad, before)


# ----------------------------------------------------------------------------------------------------------- box NMS
def _boxes(N, g, cuda, ties, zero_area):
    xy = torch.randint(0, 300, (N, 2), generator=g, device=cuda)
    wh = torch.randint(1, 80, (N, 2), generator=g, device=cuda)
    if zero_area:
        wh[::7, 0] = 0
    boxes = torch.cat([xy, xy + wh], 1).int()
    scores = (torch.randint(0, 6, (N,), generator=g, device=cuda).float() / 8 if ties
              else torch.randperm(N, generator=g, device=cuda).float() / N + 0.1)
    return boxes.contiguous(), scores.contiguous()


@gpu
@pytest.mark.parametrize("N", [0, 1, 63, 64, 65, 3072, 12288])
@pytest.mark.parametrize("ties", [False, True])
def test_box_nms(cuda, N, ties):
    lib = _lib(cuda)
    g = _gen(cuda, "nms", N, ties)
    boxes, scores = _boxes(N, g, cuda, ties, zero_area=True)
    thr = 0.5
    ws = torch.empty(lib.size("es3_box_nms_ws_floats", N) + 2, dtype=torch.float32, device=cuda)
    keep0, inside = _flat_out(N, torch.float32, cuda)
    count0 = torch.full((1,), -5, dtype=torch.int32, device=cuda)
    runs = []
    for _ in range(2):
        keep, count = keep0.clone(), count0.clone()
        lib.call("es3_box_nms", boxes.data_ptr(), scores.data_ptr(), N, thr, keep.data_ptr(), count.data_ptr(), ws.data_ptr(), _st())
        runs.append((keep, count))
    assert torch.equal(_bits(runs[0][0]), _bits(runs[1][0])) and torch.equal(runs[0][1], runs[1][1]), "two runs differ"
    keep, count = runs[0]
    n = int(count.item())
    got = keep.view(torch.int32)[:n].long().cpu()
    ref = OA.nms_stable(boxes.cpu(), scores.cpu(), thr)
    assert got.tolist() == ref.tolist()
    inside = torch.zeros_like(inside)
    inside[:n] = True
    _assert_untouched(keep, inside, "keep")
    if not ties:
        from torchvision.ops import batched_nms
        tv = batched_nms(boxes.cpu().float(), scores.cpu(), torch.zeros(N, dtype=torch.int64), thr)
        assert got.tolist() == tv.tolist()
    from efficientsam3_b200 import ops
    k2, c2 = ops.box_nms(boxes, scores, thr)
    assert torch.equal(k2[:n].cpu().long(), got) and int(c2.item()) == n
    _declined(lib, "es3_box_nms", [boxes.data_ptr(), scores.data_ptr(), 65537, thr, keep.data_ptr(), count.data_ptr(), ws.data_ptr(),
                                    _st()], [keep, count])


# ----------------------------------------------------------------------------------------------------------- RLE
# (K, Hi, Wi, crop XYXY, orig (h, w)): the whole image (first and last pixel of the column-major order set), an interior crop,
# a crop in the bottom-right corner, downsampling
RLE = [
    (5, 16, 16, (0, 0, 90, 70), (70, 90)),
    (9, 24, 20, (13, 7, 101, 66), (80, 120)),
    (4, 12, 12, (40, 30, 120, 80), (80, 120)),
    (3, 288, 288, (5, 5, 105, 65), (70, 110)),
]


@gpu
@pytest.mark.parametrize("K,Hi,Wi,crop,orig", RLE)
def test_amg_rle(cuda, K, Hi, Wi, crop, orig):
    from efficientsam3_b200 import ops
    lib = _lib(cuda)
    g = _gen(cuda, "rle", K, Hi, crop)
    low = _logits(1, K, Hi, Wi, "bumps", g, cuda)[0].contiguous()
    low[0] = 5.0                                 # all set: touches the first and the last pixel
    low[1, 0, 0] = 50.0
    low[1, -1, -1] = 50.0
    low[2] = -5.0                                # empty
    H, W = orig
    x0, y0, x1, y1 = crop
    high = ops.bilinear_nchw(low[None], y1 - y0, x1 - x0, binarize_thr=0.0, want_float=False)[1][0].bool()
    full = OA.uncrop_masks(high, list(crop), H, W)
    ref = OA.mask_to_rle_pytorch(full)
    cap = 4 * W + 64
    ws = torch.empty(lib.size("es3_amg_rle_ws_floats", K, W), dtype=torch.int32, device=cuda)
    pos0, _ = _flat_out(K * cap, torch.float32, cuda)
    bin0 = torch.full((K * H * W + TAIL,), 7, dtype=torch.uint8, device=cuda)
    runs = []
    for _ in range(2):
        pos, b = pos0.clone(), bin0.clone()
        nt = torch.full((K,), -1, dtype=torch.int32, device=cuda)
        area = torch.full((K,), -1, dtype=torch.int32, device=cuda)
        lib.call("es3_amg_rle", low.data_ptr(), K, Hi, Wi, *crop, W, H, 0.0, ws.data_ptr(), pos.data_ptr(), cap, nt.data_ptr(),
                 area.data_ptr(), b.data_ptr(), _st())
        runs.append((pos, b, nt, area))
    for x, y in zip(*runs):
        assert torch.equal(_bits(x), _bits(y)), "two runs differ"
    pos, b, nt, area = runs[0]
    posi = pos.view(torch.int32)
    inside = torch.zeros(pos.numel(), dtype=torch.bool, device=cuda)
    for k in range(K):
        n = int(nt[k])
        counts = np.diff(np.concatenate([[0], posi[k * cap:k * cap + n].cpu().numpy(), [H * W]])).tolist()
        assert {"size": [H, W], "counts": counts} == ref[k], f"mask {k}"
        assert int(area[k]) == OA.area_from_rle(ref[k]) == int(full[k].sum())
        inside[k * cap:k * cap + n] = True
    _assert_untouched(pos, inside, "rle positions")
    assert torch.equal(b[:K * H * W].view(K, H, W).bool(), full), "uint8 masks"
    assert bool((b[K * H * W:] == 7).all()), "uint8 tail written"
    assert ref[2]["counts"] == [H * W] and (ref[0]["counts"][0] == 0) == (crop[:2] == (0, 0))
    # a buffer too small for a mask: that mask writes no positions, its n_trans says how many it needs
    small = pos0.clone()
    nt2 = torch.empty(K, dtype=torch.int32, device=cuda)
    lib.call("es3_amg_rle", low.data_ptr(), K, Hi, Wi, *crop, W, H, 0.0, ws.data_ptr(), small.data_ptr(), 2, nt2.data_ptr(),
             area.data_ptr(), 0, _st())
    assert torch.equal(nt2, nt)
    for k in range(K):
        seg = small.view(torch.int32)[k * 2:k * 2 + 2]
        if int(nt[k]) > 2:
            assert bool(torch.isnan(small[k * 2:k * 2 + 2]).all())
        else:
            assert seg[:int(nt[k])].tolist() == posi[k * cap:k * cap + int(nt[k])].tolist()
    _declined(lib, "es3_amg_rle", [low.data_ptr(), K, Hi, Wi, x0, y0, W + 1, y1, W, H, 0.0, ws.data_ptr(), pos.data_ptr(), cap,
                                   nt.data_ptr(), area.data_ptr(), b.data_ptr(), _st()], [pos, b, nt, area])


# ----------------------------------------------------------------------------------------------------------- end to end
def _synthetic_generator(cuda, case, seed):
    from efficientsam3_b200.model.automatic_mask_generator import SamAutomaticMaskGenerator
    model = types.SimpleNamespace(no_mem_embed=torch.zeros(1, device=cuda), _features=None)
    gen = SamAutomaticMaskGenerator(model, **case_kwargs(case))

    def decode_crop(cropped_im, points):
        for b in range(0, len(points), gen.points_per_batch):
            low, iou = OA.synthetic_decoder(points[b:b + gen.points_per_batch], cropped_im.shape[:2], seed)
            yield low.to(cuda), iou.to(cuda)

    gen._decode_crop = decode_crop
    return gen


@gpu
@pytest.mark.parametrize("idx", range(6))
def test_generator_reproduces_reference_records(cuda, idx):
    seed, cases = load_cases()
    case = cases[idx]
    gen = _synthetic_generator(cuda, case, seed)
    got = gen.generate(np.zeros((*case["image_hw"], 3), dtype=np.uint8))
    assert_records_equal(got, case["records"], case["tag"])


def _segmenter(cuda):
    from efficientsam3_b200.model.sam1_task import Sam3PointPromptSegmenter
    from oracle.weights import fill_state_dict
    seg = Sam3PointPromptSegmenter(vit_overrides=dict(depth=1, global_att_blocks=()))
    sd = {k: v for k, v in fill_state_dict(seg.state_dict(), 43).items() if not v.is_complex()}
    seg.load_state_dict(sd, strict=False)
    return seg.to(cuda)


def _oracle_on_segmenter(gen, image, kw):
    """oracle.amg.generate fed the segmenter's own decode_prompts outputs (each crop encoded as the generator encodes it) and
    ops.bilinear_nchw as the upsampling."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model.sam1_task import host_transform_coords
    pred, seg = gen.predictor, gen.predictor.model
    current = {}

    def decode(crop_box, points, hw):
        if current.get("box") != crop_box:
            x0, y0, x1, y1 = crop_box
            pred.set_image(image[y0:y1, x0:x1, :])
            current["box"] = crop_box
        c = host_transform_coords(torch.as_tensor(points, dtype=torch.float), True, hw, seg.image_size).to(pred.device)
        lab = torch.ones((len(points), 1), dtype=torch.int32, device=pred.device)
        low, iou, _ = seg.decode_prompts(0, (c[:, None, :], lab), multimask_output=True, obj_gate=False)
        return low.clone(), iou.clone()

    up = lambda low, h, w: ops.bilinear_nchw(low, h, w)[0]
    return OA.generate(image.shape[:2], decode, gen.point_grids, points_per_batch=gen.points_per_batch, upsample=up, **kw)


@gpu
@pytest.mark.parametrize("strict", [False, True])
def test_generator_on_segmenter_vs_oracle(cuda, strict):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model.automatic_mask_generator import SamAutomaticMaskGenerator
    seg = _segmenter(cuda)
    rng = np.random.default_rng(3)
    image = rng.integers(0, 256, size=(120, 170, 3), dtype=np.uint8)
    kw = dict(pred_iou_thresh=0.05, stability_score_thresh=0.1, stability_score_offset=0.25, crop_n_layers=1, box_nms_thresh=0.95,
              crop_nms_thresh=0.95, output_mode="uncompressed_rle")
    with ops.strict_precision(strict):
        gen = SamAutomaticMaskGenerator(seg, points_per_side=5, points_per_batch=16, **kw)
        outs = {}
        for graphs in (False, True):
            seg.enable_cuda_graphs(graphs)
            got = gen.generate(image)
            ref = _oracle_on_segmenter(gen, image, kw)
            assert_records_equal(got, ref, f"strict={strict} graphs={graphs}", digest=False)
            outs[graphs] = got
        seg.enable_cuda_graphs(False)
    print(f"strict={strict}: {len(outs[False])} records")
    assert len(outs[False]) > 0
    assert_records_equal(outs[True], outs[False], "graphs on vs off", digest=False)


# ----------------------------------------------------------------------------------------------------------- registers
def test_amg_kernels_do_not_spill(tmp_path):
    from efficientsam3_b200 import build
    from test_kernel_registers import _entries, _nvcc
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "amg.cu"), "-o", str(tmp_path / "amg.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rows = _entries(r.stdout + r.stderr)
    names = {"amg_stats_kernel", "amg_finalize_kernel", "amg_compact_kernel", "nms_rank_kernel", "nms_mask_kernel", "nms_sweep_kernel",
             "amg_rle_count_kernel", "amg_rle_scan_kernel", "amg_rle_write_kernel"}
    assert all(any(n in r[0] for r in rows) for n in names), [r[0] for r in rows]
    bad = [r for r in rows if r[1] or r[2] or r[3]]
    assert not bad, f"(kernel, stack, spill stores, spill loads) = {bad}"
