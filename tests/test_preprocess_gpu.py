"""Stage-1 image preparation from decoded uint8 on the device (es3_prepare_images_u8 through stage1.preprocess.prepare_images).

* element by element against an fp64 application of torch's fp32 antialias weights (UpSample.h, _compute_indices_min_size_weights_aa,
  restated in numpy float32 below), with a per-element bound: gamma_n sum |w||x| for each pass, plus the normalisation's rounding,
  over std; outputs and workspace NaN-prefilled, the pad region exactly +0, an image alone bit-identical to itself inside a ragged
  batch, repeated calls bit-identical;
* the reference's own transform (tests/golden/preprocess_small.npz) and torch CPU F.interpolate(antialias=True) at SA-1B sizes;
* train_one_epoch / save_embeddings_one_epoch fed uint8 images against the same loops fed the prepared fp32 images."""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from bounds import U, _check, report_worst
from oracle import preprocess as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from gen_golden_preprocess import CASES, case_image  # noqa: E402

pytestmark = pytest.mark.gpu
_report = report_worst("stage-1 image preparation")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "preprocess_small.npz")
STD = torch.tensor(O.STD, dtype=torch.float64)
MEAN = torch.tensor(O.MEAN, dtype=torch.float64)


def _gamma(n):
    return n * U / (1 - n * U)


def aa_weights(n_in, n_out):
    """[n_out, n_in] float64 matrix of torch's fp32 antialiased bilinear weights, and the largest tap count."""
    f = np.float32
    scale = f(n_in) / f(n_out)
    support = scale if scale >= 1 else f(1)
    invscale = f(1) / scale if scale >= 1 else f(1)
    W = np.zeros((n_out, n_in), np.float64)
    taps = 0
    for i in range(n_out):
        center = scale * (f(i) + f(0.5))
        lo = max(int((center - support) + f(0.5)), 0)
        hi = min(int((center + support) + f(0.5)), n_in)
        ws = []
        for j in range(lo, hi):
            x = abs((f(j) - center + f(0.5)) * invscale)
            ws.append(f(1) - x if x < f(1) else f(0))
        total = f(0)
        for w in ws:
            total = f(total + w)
        W[i, lo:hi] = [float(w / total) if total != 0 else float(w) for w in ws]
        taps = max(taps, hi - lo)
    return W, taps


def _reference(img, S, cuda):
    """(fp64 output [3,S,S], per-element bound, (h', w')) of one HWC uint8 image."""
    from efficientsam3_b200.stage1.preprocess import get_preprocess_shape
    h, w = img.shape[:2]
    ho, wo = get_preprocess_shape(h, w, S)
    Wh, nh = aa_weights(w, wo)
    Wv, nv = aa_weights(h, ho)
    Wh, Wv = torch.from_numpy(Wh).to(cuda), torch.from_numpy(Wv).to(cuda)
    x = img.to(cuda).double().permute(2, 0, 1)                              # [3, h, w], exact
    t = x @ Wh.T                                                             # horizontal pass, [3, h, w']
    a = x @ Wh.abs().T                                                       # sum |w||x|
    bh = _gamma(nh + 1) * a                                                  # fp32 error of the stored horizontal result
    v = Wv @ t                                                               # [3, h', w']
    bv = _gamma(nv + 1) * (Wv.abs() @ (a + bh)) + Wv.abs() @ bh
    m, s = MEAN.to(cuda).view(3, 1, 1), STD.to(cuda).view(3, 1, 1)
    ref = (v - m) / s
    bound = bv / s + 2.01 * U * ((v - m).abs() + bv) / s + 1e-30
    R = torch.zeros(3, S, S, dtype=torch.float64, device=cuda)
    B = torch.ones(3, S, S, dtype=torch.float64, device=cuda)
    R[:, :ho, :wo], B[:, :ho, :wo] = ref, bound
    return R, B, (ho, wo)


@pytest.fixture
def nan_ws(monkeypatch):
    from efficientsam3_b200 import ops
    monkeypatch.setattr(ops, "_f32ws", lambda n, dev: torch.full((max(int(n), 1),), float("nan"), device=dev))


def _images(shapes, seed):
    return [case_image(h, w, seed * 1000 + i) for i, (h, w) in enumerate(shapes)]


RAGGED = [(300, 451), (451, 300), (37, 23), (256, 256), (1, 150), (257, 3), (131, 97)]


@pytest.mark.parametrize("S", [96, 256])
def test_ragged_batch_element_by_element(cuda, nan_ws, S):
    from efficientsam3_b200.stage1.preprocess import prepare_images
    imgs = _images(RAGGED, S)
    out = torch.full((len(imgs), 3, S, S), float("nan"), device=cuda)
    x, sizes = prepare_images(imgs, S, device=cuda, out=out)
    assert x.data_ptr() == out.data_ptr()
    torch.cuda.synchronize()
    for b, img in enumerate(imgs):
        ref, bound, (ho, wo) = _reference(img, S, cuda)
        assert sizes[b].tolist() == [3, ho, wo]
        _check("ragged batch", x[b], ref, bound, f"image {b} {tuple(img.shape)} at S={S}")
        pad = torch.ones(3, S, S, dtype=torch.bool, device=cuda)
        pad[:, :ho, :wo] = False
        assert (x[b][pad].view(torch.int32) == 0).all(), "pad region is not +0"      # +0 bit pattern, not -0
        alone, _ = prepare_images([img], S, device=cuda)
        assert torch.equal(alone[0].view(torch.int32), x[b].view(torch.int32)), f"image {b} alone != inside the batch"
    again, _ = prepare_images(imgs, S, device=cuda)
    assert torch.equal(again.view(torch.int32), x.view(torch.int32))


def test_sa1b_size_element_by_element(cuda, nan_ws):
    from efficientsam3_b200.stage1.preprocess import prepare_images
    img = _images([(1500, 2250)], 7)[0]
    x, _ = prepare_images([img], 1008, device=cuda)
    ref, bound, _ = _reference(img, 1008, cuda)
    _check("SA-1B size 1500x2250 -> 1008", x[0], ref, bound, "1500x2250")


def test_more_images_than_one_launch_takes(cuda, nan_ws):
    """Batches above ops.PREPARE_MAX_IMAGES run as several calls into one output."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.preprocess import pack_images, prepare_images
    g = torch.Generator().manual_seed(5)
    shapes = [tuple(int(v) for v in torch.randint(1, 40, (2,), generator=g)) for _ in range(ops.PREPARE_MAX_IMAGES + 9)]
    imgs = _images(shapes, 11)
    n0 = ops.launch_count
    x, sizes = prepare_images(pack_images(imgs).pin_memory(), 32, device=cuda)
    assert ops.launch_count - n0 == 4
    for b in (0, ops.PREPARE_MAX_IMAGES - 1, ops.PREPARE_MAX_IMAGES, len(imgs) - 1):
        ref, bound, (ho, wo) = _reference(imgs[b], 32, cuda)
        assert sizes[b].tolist() == [3, ho, wo]
        _check("ragged batch", x[b], ref, bound, f"image {b} of {len(imgs)}")


def test_reference_fixture(cuda):
    from efficientsam3_b200.stage1.preprocess import prepare_images
    g = np.load(GOLDEN)
    for (tag, h, w, S, seed), size in zip(CASES, g["sizes"]):
        x, sizes = prepare_images([case_image(h, w, seed)], S, device=cuda)
        want = torch.from_numpy(g[f"out_{tag}"]).double()
        assert sizes[0].tolist() == list(size), tag
        err = ((x[0].cpu().double() - want).abs() * STD.view(3, 1, 1)).max().item()
        assert err <= 1e-3, (tag, err)


@pytest.mark.parametrize("hw", [(1500, 2250), (2250, 1500), (600, 800)])
def test_matches_torch_cpu_interpolate(cuda, hw):
    """A tap window shifted by one would show here as an O(1) error in 0..255 units."""
    from efficientsam3_b200.stage1.preprocess import prepare_images
    img = _images([hw], 3)[0]
    x, sizes = prepare_images([img], 1008, device=cuda)
    want, size = O.prepare_image(img, 1008)
    assert tuple(sizes[0].tolist()) == size
    err = ((x[0].cpu().double() - want.double()).abs() * STD.view(3, 1, 1)).max().item()
    print(f"\n{hw} -> 1008: max |device - torch CPU| = {err:.3g} (0..255 units)", end="")
    assert err <= 1e-3, err


def _student(cuda):
    from efficientsam3_b200.stage1.model import build_image_student_model
    from oracle.weights import fill_state_dict
    cfg = NS(MODEL=NS(BACKBONE="efficientvit_b1"), DATA=NS(IMG_SIZE=160), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=12))
    m = build_image_student_model(cfg)
    m.load_state_dict(fill_state_dict(m.state_dict(), 3))
    return m.to(cuda)


def _u8_batches(n, B):
    shapes = [(120, 180), (181, 97), (160, 160), (33, 64), (200, 150), (90, 91)]
    return [_images([shapes[(i * B + j) % len(shapes)] for j in range(B)], 20 + i) for i in range(n)]


def test_train_one_epoch_from_uint8_matches_prepared_fp32(cuda):
    from efficientsam3_b200.stage1.optim import FlatAdamW
    from efficientsam3_b200.stage1.preprocess import pack_images, prepare_images
    from efficientsam3_b200.stage1.train import train_one_epoch
    cfg = NS(TRAIN=NS(EVAL_BN_WHEN_TRAINING=True, ACCUMULATION_STEPS=2, EPOCHS=2, WARMUP_EPOCHS=0, MIN_LR=1e-6, WARMUP_LR=1e-7,
                      CLIP_GRAD=5.0),
             DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=12, COSINE=1.0), DATA=NS(IMG_SIZE=160, MEAN=list(O.MEAN), STD=list(O.STD)))
    batches = _u8_batches(4, 2)
    saved = [([np.random.RandomState(10 * i + j).randn(1024 * 144).astype(np.float16) for j in range(2)], [i, i]) for i in range(4)]
    runs = []
    for feed in ("list", "packed", "fp32"):
        m = _student(cuda)
        opt = FlatAdamW(m, lr=1e-4, weight_decay=0.01)
        if feed == "fp32":
            loader = []
            for imgs, s in zip(batches, saved):
                x, sizes = prepare_images(imgs, 160, device=cuda)
                loader.append(((list(x), {"img_size_before_pad": [tuple(r) for r in sizes.tolist()]}), s))
        else:
            loader = [((imgs if feed == "list" else pack_images(imgs), None), s) for imgs, s in zip(batches, saved)]
        runs.append(torch.stack(train_one_epoch(cfg, m, loader, opt, epoch=0)).cpu())
    assert torch.isfinite(runs[2]).all()
    assert torch.equal(runs[0], runs[2]) and torch.equal(runs[1], runs[2]), runs


def test_save_embeddings_from_uint8_matches_prepared_fp32(cuda, tmp_path):
    from efficientsam3_b200.stage1 import embeddings as E
    from efficientsam3_b200.stage1.preprocess import prepare_images
    m = _student(cuda).eval()
    batches = _u8_batches(3, 2)
    keys = [[f"img_{b}_{i}" for i in range(2)] for b in range(3)]
    seeds = [np.array([10 * b + i for i in range(2)], dtype=np.int32) for b in range(3)]
    u8 = [((imgs, None), (k, s)) for imgs, k, s in zip(batches, keys, seeds)]
    f32 = [((list(prepare_images(imgs, 160, device=cuda)[0]), None), (k, s)) for imgs, k, s in zip(batches, keys, seeds)]
    assert E.save_embeddings_one_epoch(m, u8, str(tmp_path / "u8"), rank=0) == 6
    assert E.save_embeddings_one_epoch(m, f32, str(tmp_path / "f32"), rank=0) == 6
    for name in ("rank0-keys.txt", "rank0-values.bin"):
        with open(tmp_path / "u8" / name, "rb") as a, open(tmp_path / "f32" / name, "rb") as b:
            assert a.read() == b.read(), name
