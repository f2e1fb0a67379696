"""Automatic mask generation on the CPU: oracle/amg.py reproduces the reference generator's committed records
(tests/golden/amg_small.json, made by tests/golden/gen_golden_amg.py from the unmodified reference), the native generator's host
geometry equals the oracle's bit for bit, its constructor validates as the reference's does, and the stable-tie NMS is
torchvision's batched_nms wherever scores are distinct."""
import importlib.util
import json
import os
import types

import numpy as np
import pytest
import torch

from oracle import amg as OA

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("gen_golden_amg", os.path.join(HERE, "golden", "gen_golden_amg.py"))
GG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(GG)


def load_cases():
    with open(os.path.join(HERE, "golden", "amg_small.json")) as f:
        g = json.load(f)
    return g["seed"], g["cases"]


def case_kwargs(case):
    return GG.case_kwargs(case["kwargs"])


def assert_records_equal(got, ref, what, digest=True):
    """Count, order and every field of each record (gen_golden_amg.record_row): `ref` holds rows (the fixture, digest=True) or
    records; a binary mask is compared as its RLE."""
    got = [GG.record_row(r, digest) for r in got]
    ref = [r if isinstance(r, list) else GG.record_row(r, digest) for r in ref]
    assert len(got) == len(ref), f"{what}: {len(got)} records, reference {len(ref)}"
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g == r, f"{what} record {i}: {g} != {r}"


def oracle_generate(case, seed):
    kw = case_kwargs(case)
    grids = kw.pop("point_grids", None)
    pps, down = kw.pop("points_per_side", None), kw.pop("crop_n_points_downscale_factor", 1)
    if pps is not None:
        grids = OA.build_all_layer_point_grids(pps, kw.get("crop_n_layers", 0), down)
    return OA.generate(case["image_hw"], lambda crop_box, points, hw: OA.synthetic_decoder(points, hw, seed), grids, **kw)


@pytest.mark.parametrize("idx", range(len(GG.CASES)))
def test_oracle_reproduces_reference_records(idx):
    seed, cases = load_cases()
    with torch.no_grad():
        got = oracle_generate(cases[idx], seed)
    assert_records_equal(got, cases[idx]["records"], cases[idx]["tag"])


def test_fixture_reaches_every_branch():
    """The committed cases keep masks with NaN stability and empty masks (filters off), masks of several crops, both outputs."""
    _, cases = load_cases()
    recs = [r for c in cases for r in c["records"]]
    assert any(r[5] == "nan" for r in recs) and any(r[1] == 0 for r in recs)
    assert len({tuple(r[6]) for r in recs}) > 3
    assert {c["kwargs"]["output_mode"] for c in cases} == {"binary_mask", "uncompressed_rle"}


def test_host_geometry_equals_oracle():
    from efficientsam3_b200.model import automatic_mask_generator as G
    from efficientsam3_b200.model.sam1_task import host_transform_coords
    for n in (1, 6, 7, 32, 64):
        assert np.array_equal(G.build_point_grid(n), OA.build_point_grid(n))
    for args in ((32, 2, 2), (16, 1, 1), (7, 2, 2)):
        a, b = G.build_all_layer_point_grids(*args), OA.build_all_layer_point_grids(*args)
        assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))
    for hw in ((1500, 2250), (150, 200), (151, 203), (97, 131), (2250, 1500)):
        for layers in range(4):
            for ratio in (512 / 1500, 0.25):
                assert G.generate_crop_boxes(hw, layers, ratio) == OA.generate_crop_boxes(hw, layers, ratio)
    # grid points in crop pixels -> model input, as SAM3InteractiveImagePredictor._transform_coords(normalize=True) scales them
    pts = OA.build_point_grid(32) * np.array([2250, 1500])[None]
    got = host_transform_coords(torch.as_tensor(pts, dtype=torch.float), True, (1500, 2250), 1008)
    one = torch.ones((), dtype=torch.float32)
    ref = torch.as_tensor(pts, dtype=torch.float).clone()
    ref[:, 0] = ref[:, 0] * (one / 2250)
    ref[:, 1] = ref[:, 1] * (one / 1500)
    assert torch.equal(got, ref * 1008)


def _gen(**kw):
    from efficientsam3_b200.model.automatic_mask_generator import SamAutomaticMaskGenerator
    return SamAutomaticMaskGenerator(types.SimpleNamespace(), **kw)


def test_constructor_validation():
    g = _gen()
    assert len(g.point_grids) == 1 and g.point_grids[0].shape == (1024, 2)
    assert g.predictor.max_hole_area == 0 and g.predictor.max_sprinkle_area == 0
    assert [p.shape[0] for p in _gen(points_per_side=8, crop_n_layers=2, crop_n_points_downscale_factor=2).point_grids] == [64, 16, 4]
    grids = [np.zeros((3, 2))]
    assert _gen(points_per_side=None, point_grids=grids).point_grids is grids
    with pytest.raises(AssertionError, match="Exactly one"):
        _gen(points_per_side=None)
    with pytest.raises(AssertionError, match="Exactly one"):
        _gen(points_per_side=8, point_grids=grids)
    with pytest.raises(AssertionError, match="Unknown output_mode"):
        _gen(output_mode="polygons")


def test_unsupported_options_raise():
    with pytest.raises(NotImplementedError, match="min_mask_region_area"):
        _gen(min_mask_region_area=100)
    try:
        import pycocotools  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError):
            _gen(output_mode="coco_rle")
    else:
        _gen(output_mode="coco_rle")


@pytest.mark.parametrize("n,thr", [(1, 0.7), (40, 0.5), (300, 0.7), (2000, 0.3)])
def test_stable_nms_equals_torchvision_on_distinct_scores(n, thr):
    from torchvision.ops import batched_nms
    g = torch.Generator().manual_seed(n)
    xy = torch.randint(0, 200, (n, 2), generator=g)
    wh = torch.randint(0, 60, (n, 2), generator=g)
    boxes = torch.cat([xy, xy + wh], 1).float()
    scores = torch.randperm(n, generator=g).float() / n + 0.25
    ref = batched_nms(boxes, scores, torch.zeros(n, dtype=torch.int64), thr)
    assert OA.nms_stable(boxes, scores, thr).tolist() == ref.tolist()


def test_stable_nms_tie_order():
    boxes = torch.tensor([[0, 0, 10, 10], [1, 1, 11, 11], [50, 50, 60, 60], [0, 0, 10, 10], [5, 5, 5, 5]], dtype=torch.float)
    scores = torch.tensor([0.5, 0.5, 0.5, 0.9, 0.5])
    # 3 first (highest), suppresses 0 and 1 (IoU > 0.5); then 2 and the zero-area 4 (NaN IoU suppresses nothing), in index order
    assert OA.nms_stable(boxes, scores, 0.5).tolist() == [3, 2, 4]
