"""CPU: the CUDA-graph switch of the point-prompt predictor and segmenter (enable_cuda_graphs) is off by default, the host-side
prompt preparation of the graphed path equals the device path's arithmetic bit for bit, and CPU modules still raise with
graphs on, with nothing captured."""
import numpy as np
import pytest
import torch

from efficientsam3_b200.model.sam1_task import (SAM3InteractiveImagePredictor, Sam3PointPromptSegmenter, host_prompts,
                                                host_transform_coords)


@pytest.fixture(scope="module")
def seg():
    return Sam3PointPromptSegmenter(image_size=112, vit_overrides=dict(img_size=112, depth=1, global_att_blocks=()))


def test_switch_is_off_by_default_and_returns_the_predictor(seg):
    pred = SAM3InteractiveImagePredictor(seg)
    assert seg._graphs is None and pred.graph_launches_per_step == 0
    assert pred.enable_cuda_graphs() is pred and seg._graphs == {} and seg._graph_max == 8
    assert pred.enable_cuda_graphs(False) is pred and seg._graphs is None
    assert seg.enable_cuda_graphs(max_graphs=2) is seg and seg._graph_max == 2
    seg.enable_cuda_graphs(False)
    for m in (pred, seg):
        with pytest.raises(ValueError, match="max_graphs"):
            m.enable_cuda_graphs(max_graphs=0)


def _device_transform(coords, normalize, hw, S):
    """What `_transform_coords` computes on a CUDA fp32 tensor: a division by a Python number is a multiplication by its
    fp32 reciprocal there, then the multiplication by S; every step rounds to fp32 (numpy float32 arithmetic is IEEE)."""
    c = coords.numpy().astype(np.float32).copy()
    if normalize:
        h, w = hw
        c[..., 0] = c[..., 0] * (np.float32(1.0) / np.float32(w))
        c[..., 1] = c[..., 1] * (np.float32(1.0) / np.float32(h))
    return c * np.float32(S)


@pytest.mark.parametrize("normalize", [True, False])
def test_host_transform_matches_the_device_arithmetic(normalize):
    g = torch.Generator().manual_seed(3)
    for _ in range(50):
        h, w = (int(v) for v in torch.randint(1, 5000, (2,), generator=g))
        S = int(torch.randint(64, 2048, (1,), generator=g))
        coords = torch.rand(3, 7, 2, generator=g) * torch.tensor([w, h]) * 1.1 - 0.05 * torch.tensor([w, h])
        if not normalize:
            coords = coords / torch.tensor([w, h])
        got = host_transform_coords(coords.clone(), normalize, (h, w), S)
        assert got.dtype == torch.float32
        np.testing.assert_array_equal(got.numpy().view(np.int32), _device_transform(coords, normalize, (h, w), S).view(np.int32))


def test_host_prompts_merge_box_corners_in_front():
    hw, S = (300, 420), 1008
    pc, pl = np.array([[210.0, 150.0], [30.0, 40.0]]), np.array([1, 0])
    box = np.array([10.0, 20.0, 200.0, 250.0])
    mask = np.random.default_rng(0).standard_normal((1, 288, 288)).astype(np.float32)
    coords, labels, mi = host_prompts(pc, pl, box, mask, True, hw, S)
    assert coords.shape == (1, 4, 2) and labels.dtype == torch.int32 and labels.tolist() == [[2, 3, 1, 0]]
    np.testing.assert_array_equal(coords[0, :2].numpy(), _device_transform(torch.tensor(box, dtype=torch.float32).reshape(2, 2), True, hw, S))
    np.testing.assert_array_equal(coords[0, 2:].numpy(), _device_transform(torch.tensor(pc, dtype=torch.float32), True, hw, S))
    assert mi.shape == (1, 1, 288, 288) and mi.dtype == torch.float32 and torch.equal(mi[0], torch.from_numpy(mask))
    coords, labels, mi = host_prompts(None, None, box, None, False, hw, S)
    assert coords.shape == (1, 2, 2) and labels.tolist() == [[2, 3]] and mi is None
    assert torch.equal(coords, torch.tensor(box, dtype=torch.float32).reshape(1, 2, 2) * S)
    assert host_prompts(None, None, None, None, True, hw, S) == (None, None, None)


def test_cpu_modules_still_raise_with_graphs_on(seg):
    pred = SAM3InteractiveImagePredictor(seg).enable_cuda_graphs()
    img = np.zeros((40, 60, 3), dtype=np.uint8)
    with pytest.raises(RuntimeError, match="set_image"):
        pred.predict(point_coords=np.array([[5.0, 5.0]]), point_labels=np.array([1]))
    with pytest.raises(ValueError, match="no CPU fallback"):
        pred.set_image(img)
    with pytest.raises(ValueError, match="no CPU fallback"):
        seg.set_image_batch(torch.zeros(1, 3, 112, 112))
    assert seg._graphs == {} and seg._feature_sets == {} and seg._features is None
    seg.enable_cuda_graphs(False)
