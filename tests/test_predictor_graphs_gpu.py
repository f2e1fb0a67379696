"""GPU: CUDA-graph replay of the point-prompt predictor and segmenter (enable_cuda_graphs) against the same calls launched kernel
by kernel (uncaptured()), bit for bit, on the SAM3 ViT trunk (one block) and the EV-M student encoder: every prompt kind, both
output modes, hole filling on and off, the batched entry points; the static image features across images, re-capture after
a weight change, eviction, the strict mode and the raise before set_image."""
import numpy as np
import pytest
import torch

from es3_recorder import point_segmenter as _seg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["vit", "student"])
def seg(request, cuda):
    return _seg(request.param, cuda)


def _img(seed, hw=(300, 420)):
    return np.random.default_rng(seed).integers(0, 256, size=(*hw, 3), dtype=np.uint8)


class _Captures:
    """Counts the segmenter's graph captures."""

    def __init__(self, seg):
        self.n, self.seg, inner = 0, seg, seg._capture

        def counted(*a):
            self.n += 1
            return inner(*a)
        seg._capture = counted

    def close(self):
        del self.seg._capture


def _same(a, b, what):
    for x, y, name in zip(a, b, ("masks", "iou", "low")):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape and x.dtype == y.dtype, (what, name, x.shape, y.shape)
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (what, name)


def _uncaptured(seg, call):
    from efficientsam3_b200 import ops
    with seg.uncaptured():
        n0 = ops.launch_count
        out = call()
        return out, ops.launch_count - n0


def _prompt_cases(low_prev):
    pts = np.array([[210.0, 150.0], [30.0, 40.0], [400.0, 10.0], [5.0, 290.0], [100.0, 100.0]])
    lab = np.array([1, 0, 1, 1, 0])
    box = np.array([40.0, 30.0, 380.0, 260.0])
    rng = np.random.default_rng(12)
    many = np.stack([rng.uniform(0, 420, 12), rng.uniform(0, 300, 12)], 1)
    many_lab = rng.integers(0, 2, 12)
    return {
        "N=1": dict(point_coords=pts[:1], point_labels=lab[:1]),
        "N=2": dict(point_coords=pts[:2], point_labels=lab[:2]),
        "N=5": dict(point_coords=pts, point_labels=lab),
        "N=12": dict(point_coords=many, point_labels=many_lab),
        "box+N=8": dict(box=box, point_coords=many[:8], point_labels=many_lab[:8]),
        "box": dict(box=box),
        "box+points": dict(box=box, point_coords=pts[:2], point_labels=lab[:2]),
        "point+mask": dict(point_coords=pts[:1], point_labels=lab[:1], mask_input=low_prev),
        "mask(cuda)": dict(mask_input=torch.from_numpy(low_prev).cuda()),
    }


@pytest.mark.parametrize("holes", [True, False])
def test_predict_replay_equals_uncaptured(seg, holes):
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor
    pred = SAM3InteractiveImagePredictor(seg, max_hole_area=64.0 if holes else 0.0, max_sprinkle_area=16.0 if holes else 0.0)
    pred.enable_cuda_graphs(max_graphs=4)
    pred.set_image(_img(0))
    low_prev = pred.predict(point_coords=np.array([[210.0, 150.0]]), point_labels=np.array([1]), multimask_output=False)[2]
    for name, kw in _prompt_cases(low_prev).items():
        for mm in (True, False):
            for logits in (True, False):
                what = f"{name} multimask={mm} logits={logits} holes={holes}"
                call = lambda: pred.predict(multimask_output=mm, return_logits=logits, **kw)
                first, again = call(), call()           # the capture's replay, then a replay with freshly staged prompts
                ref, launches = _uncaptured(seg, call)
                _same(first, ref, what)
                _same(again, ref, what)
                assert pred.graph_launches_per_step == launches, what
    pred.enable_cuda_graphs(False)


def test_predict_batch_replay_equals_uncaptured(seg):
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor
    pred = SAM3InteractiveImagePredictor(seg, max_hole_area=64.0, max_sprinkle_area=16.0).enable_cuda_graphs()
    pred.set_image_batch([_img(1), _img(2, (512, 384))])
    kw = dict(point_coords_batch=[np.array([[210.0, 150.0], [30.0, 40.0]]), np.array([[100.0, 400.0]])],
              point_labels_batch=[np.array([1, 0]), np.array([1])], box_batch=[None, np.array([10.0, 20.0, 300.0, 480.0])])
    for mm in (True, False):
        got = pred.predict_batch(multimask_output=mm, **kw)
        ref, _ = _uncaptured(seg, lambda: pred.predict_batch(multimask_output=mm, **kw))
        for i in range(2):
            _same([t[i] for t in got], [t[i] for t in ref], f"image {i} multimask={mm}")
    pred.enable_cuda_graphs(False)


def test_segmenter_entry_points_replay_equal_uncaptured(seg, cuda):
    seg.enable_cuda_graphs()
    S = seg.image_size
    g = torch.Generator().manual_seed(7)
    seg.set_image_batch(torch.randn(2, 3, S, S, generator=g).to(cuda))
    h = seg._features["h"]
    coords, labels = torch.rand(2, 3, 2, generator=g) * S, torch.tensor([[1, 0, 1], [1, 1, 0]], dtype=torch.int32)
    boxes = torch.tensor([[10.0, 20.0, 300.0, 400.0], [50.0, 60.0, 200.0, 100.0]])
    mask = torch.randn(2, 1, 4 * h, 4 * h, generator=g)
    for mm in (True, False):
        for logits in (True, False):
            call = lambda: seg.predict_batch(coords.to(cuda), labels.to(cuda), multimask_output=mm, return_logits=logits)
            got = {k: v.clone() for k, v in call().items()}
            ref, launches = _uncaptured(seg, call)
            assert got.keys() == ref.keys() and seg.graph_launches_per_step == launches
            for k in got:
                assert torch.equal(got[k], ref[k]), (k, mm, logits)
        for name, kw in {"points": dict(points=(coords, labels)), "boxes": dict(boxes=boxes),
                         "boxes+points+mask": dict(points=(coords, labels), boxes=boxes, mask_input=mask)}.items():
            kw = {k: tuple(t.to(cuda) for t in v) if isinstance(v, tuple) else v.to(cuda) for k, v in kw.items()}
            call = lambda: seg.decode_prompts(1, multimask_output=mm, obj_gate=True, **kw)
            got = [t.clone() for t in call()]
            ref, launches = _uncaptured(seg, call)
            assert seg.graph_launches_per_step == launches
            for x, y in zip(got, ref):
                assert torch.equal(x, y), (name, mm)
    n = len(seg._graphs)
    with pytest.raises(RuntimeError, match="CUDA tensor"):         # CPU prompts raise, graphs on or off
        seg.decode_prompts(0, points=(coords, labels))
    assert len(seg._graphs) == n
    seg.enable_cuda_graphs(False)


def test_static_features_serve_later_images_without_capture(seg):
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor
    pred = SAM3InteractiveImagePredictor(seg).enable_cuda_graphs()
    kw = dict(point_coords=np.array([[210.0, 150.0], [30.0, 40.0]]), point_labels=np.array([1, 0]))
    caps = _Captures(seg)
    try:
        pred.set_image(_img(3))
        out_a = pred.predict(**kw)
        buf = seg._features["keys_f32"].data_ptr()
        assert caps.n == 1 and len(seg._graphs) == 1
        pred.set_image(_img(4))
        assert seg._features["keys_f32"].data_ptr() == buf
        out_b = pred.predict(**kw)
        assert caps.n == 1 and len(seg._graphs) == 1
        ref_b, _ = _uncaptured(seg, lambda: pred.predict(**kw))
        _same(out_b, ref_b, "image B")
        assert not np.array_equal(out_a[2], out_b[2])
    finally:
        caps.close()
        pred.enable_cuda_graphs(False)


def test_recapture_after_load_state_dict_and_eviction(seg):
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor
    pred = SAM3InteractiveImagePredictor(seg).enable_cuda_graphs(max_graphs=2)
    pts = np.array([[210.0, 150.0], [30.0, 40.0], [400.0, 10.0]])
    lab = np.array([1, 0, 1])
    one = lambda n: pred.predict(point_coords=pts[:n], point_labels=lab[:n])
    sd0 = {k: v.clone() for k, v in seg.state_dict().items()}
    caps = _Captures(seg)
    try:
        pred.set_image(_img(5))
        before = one(1)
        sd = {k: v.clone() for k, v in sd0.items()}
        for k in ("sam_mask_decoder.output_hypernetworks_mlps.0.layers.2.weight", "sam_mask_decoder.iou_prediction_head.layers.2.bias",
                  "sam_prompt_encoder.point_embeddings.1.weight"):
            sd[k] = sd[k] * 1.5 + 0.1
        seg.load_state_dict(sd)
        after = one(1)
        assert caps.n == 2 and len(seg._graphs) == 1
        ref, _ = _uncaptured(seg, lambda: one(1))
        _same(after, ref, "after load_state_dict")
        assert not np.array_equal(before[1], after[1])
        one(2)
        first = list(seg._graphs)
        one(3)                                   # a third key: the oldest (N=1) goes
        assert caps.n == 4 and len(seg._graphs) == 2 and list(seg._graphs)[0] == first[1] and first[0] not in seg._graphs
        one(1)
        assert caps.n == 5
    finally:
        caps.close()
        seg.load_state_dict(sd0)
        pred.enable_cuda_graphs(False)


def test_strict_mode_is_never_replayed(cuda):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor
    seg = _seg("student", cuda)
    pred = SAM3InteractiveImagePredictor(seg)
    kw = dict(point_coords=np.array([[210.0, 150.0]]), point_labels=np.array([1]), box=np.array([40.0, 30.0, 380.0, 260.0]))
    with ops.strict_precision():
        pred.set_image(_img(6))
        off = pred.predict(**kw)
        pred.enable_cuda_graphs()
        pred.set_image(_img(6))
        on = pred.predict(**kw)
    _same(on, off, "strict")
    assert seg._graphs == {} and seg._feature_sets == {}


def test_predict_before_set_image_raises_before_any_launch(seg):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor
    pred = SAM3InteractiveImagePredictor(seg).enable_cuda_graphs()
    n0 = ops.launch_count
    with pytest.raises(RuntimeError, match="set_image"):
        pred.predict(point_coords=np.array([[5.0, 5.0]]), point_labels=np.array([1]))
    assert ops.launch_count == n0 and seg._graphs == {}
    pred.enable_cuda_graphs(False)


@pytest.mark.parametrize("normalize", [True, False])
def test_host_transform_equals_the_device_transform(seg, cuda, normalize):
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor, host_transform_coords
    pred = SAM3InteractiveImagePredictor(seg)
    g = torch.Generator().manual_seed(11)
    for _ in range(50):
        h, w = (int(v) for v in torch.randint(1, 5000, (2,), generator=g))
        coords = torch.rand(4, 5, 2, generator=g) * torch.tensor([w, h]) * (1.0 if normalize else 1.0 / max(h, w))
        dev = pred._transform_coords(coords.to(cuda), normalize, (h, w)).cpu()
        host = host_transform_coords(coords, normalize, (h, w), seg.image_size)
        assert torch.equal(dev.view(torch.int32), host.view(torch.int32)), (h, w)
