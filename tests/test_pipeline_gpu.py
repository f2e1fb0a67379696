"""GPU: FPN neck vs the reference fixture, and the batched point-prompt pipeline (ViT trunk -> SAM2-branch FPN ->
SAM heads, BASELINE config 3 geometry at reduced ViT depth) against the composition of the CPU oracles."""
import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden, max_err_over_scale, rel_l2, sd_from_keys

pytestmark = pytest.mark.gpu


class _Trunk(torch.nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.channel_list = [dim]

    def forward(self, x):
        return [x]


def test_neck_matches_reference_fixture(cuda):
    from efficientsam3_b200.model.necks import Sam3DualViTDetNeck
    g = load_golden("neck_small")
    dim, d_model, hw, B = int(g["dim"]), int(g["d_model"]), int(g["hw"]), int(g["B"])
    m = Sam3DualViTDetNeck(trunk=_Trunk(dim), position_encoding=None, d_model=d_model, scale_factors=[4.0, 2.0, 1.0, 0.5],
                           add_sam2_neck=True)
    sig = [f"{k}|{','.join(map(str, v.shape))}|{str(v.dtype).replace('torch.', '')}" for k, v in m.state_dict().items()]
    assert sig == [str(k) for k in g["keys"]]
    m.load_state_dict(sd_from_keys(g["keys"], int(g["seed_w"])))
    m = m.to(cuda).eval()
    x = torch.randn(B, dim, hw, hw, generator=torch.Generator().manual_seed(int(g["seed_x"]))).to(cuda)
    s3, _, s2, _ = m(x)
    for name, outs in (("sam3", s3), ("sam2", s2)):
        for i, t in enumerate(outs):
            ref = g[f"{name}_{i}"]
            assert t.shape == tuple(ref.shape)
            e = rel_l2(t.cpu(), ref)
            print(f"neck {name} level {i}: rel_l2={e:.3e}")
            assert e <= 1e-2


def test_point_prompt_pipeline_vs_oracles(cuda):
    from efficientsam3_b200.model.sam1_task import Sam3PointPromptSegmenter
    from oracle import necks as ON, sam_heads as OH, vitdet as OV
    from oracle.weights import fill_state_dict
    vit_cfg = dict(depth=2, global_att_blocks=(1,))
    seg = Sam3PointPromptSegmenter(vit_overrides=vit_cfg)
    sd = {k: v for k, v in fill_state_dict(seg.state_dict(), 41).items() if not v.is_complex()}
    seg.load_state_dict(sd, strict=False)
    B, S = 2, 1008
    g = torch.Generator().manual_seed(5)
    img = torch.randn(B, 3, S, S, generator=g)
    coords = torch.rand(B, 1, 2, generator=g) * S
    labels = torch.ones(B, 1, dtype=torch.int32)
    # ---- oracle composition on CPU
    with torch.no_grad():
        cfg = dict(OV.SAM3_VIT, **vit_cfg)
        trunk = OV.vit_trunk(sd, "backbone.vision_backbone.trunk.", img, cfg)
        l288, l144, l72 = ON.neck({k[len("backbone.vision_backbone."):]: v for k, v in sd.items() if k.startswith("backbone.vision_backbone.")},
                                  trunk, prefix="sam2_convs.")[:3]
        sd_md = {k[len("sam_mask_decoder."):]: v for k, v in sd.items() if k.startswith("sam_mask_decoder.")}
        sd_pe = {k[len("sam_prompt_encoder."):]: v for k, v in sd.items() if k.startswith("sam_prompt_encoder.")}
        hr = OH.high_res_from_fpn(sd_md, "", l288, l144)
        feat = l72 + sd["no_mem_embed"].reshape(1, -1, 1, 1)
        ref = OH.forward_sam_heads(sd_pe, sd_md, feat, hr, coords, labels, S, multimask_output=True)
    # ---- native
    seg = seg.to(cuda)
    out = seg.set_image_batch(img.to(cuda)).predict_batch(coords.to(cuda), labels.to(cuda), multimask_output=True, return_logits=True)
    low, high = out["low_res_multimasks"].cpu(), out["high_res"].cpu()
    e_low, e_obj = rel_l2(low, ref["low_res_multimasks"]), (out["object_score_logits"].cpu() - ref["object_score_logits"]).abs().max().item()
    print(f"pipeline low-res logits rel_l2={e_low:.3e}, obj abs err={e_obj:.3e}, ious err={(out['ious'].cpu() - ref['ious']).abs().max().item():.3e}")
    assert torch.equal(out["object_score_logits"].cpu() > 0, ref["object_score_logits"] > 0)
    assert e_low <= 2e-2 and e_obj <= 5e-2
    assert torch.equal(out["best"].cpu(), ref["best"])
    err = (high.double() - ref["high_res_multimasks"].double()).abs().max().item()
    safe = ref["high_res_multimasks"].abs() > err
    assert torch.equal((high > 0)[safe], (ref["high_res_multimasks"] > 0)[safe])
    agree = ((high > 0) == (ref["high_res_multimasks"] > 0)).float().mean().item()
    print(f"binary mask agreement {agree:.5f}, rounding band {(~safe).float().mean().item():.4%}")
    assert agree >= 0.99
    bm = seg.predict_batch(coords.to(cuda), labels.to(cuda), multimask_output=True)["high_res"]
    assert bm.dtype == torch.bool and torch.equal(bm.cpu(), high > 0)


def test_interactive_predictor_api_vs_oracle(cuda):
    """SAM3InteractiveImagePredictor drop-in (set_image / set_image_batch / predict / predict_batch): uint8 HWC images of
    arbitrary size, point / box / mask prompts, several prompts on one image, hole filling, resize to the original size.
    The decoder path is checked against oracle.sam_heads.predict fed with the NATIVE image features, so this test isolates
    prompt encoding + decoding + post-processing (the encoder has its own parity tests)."""
    import numpy as np
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor, Sam3PointPromptSegmenter
    from oracle import sam_heads as OH
    from oracle.weights import fill_state_dict
    seg = Sam3PointPromptSegmenter(vit_overrides=dict(depth=1, global_att_blocks=()))
    sd = {k: v for k, v in fill_state_dict(seg.state_dict(), 43).items() if not v.is_complex()}
    seg.load_state_dict(sd, strict=False)
    seg = seg.to(cuda)
    pred = SAM3InteractiveImagePredictor(seg, mask_threshold=0.0, max_hole_area=64.0, max_sprinkle_area=16.0)
    with pytest.raises(RuntimeError):
        pred.predict(point_coords=np.array([[5.0, 5.0]]), point_labels=np.array([1]))
    rng = np.random.default_rng(0)
    imgs = [rng.integers(0, 256, size=(300, 420, 3), dtype=np.uint8), rng.integers(0, 256, size=(512, 384, 3), dtype=np.uint8)]
    sd_md = {k[len("sam_mask_decoder."):]: v for k, v in sd.items() if k.startswith("sam_mask_decoder.")}
    sd_pe = {k[len("sam_prompt_encoder."):]: v for k, v in sd.items() if k.startswith("sam_prompt_encoder.")}
    S = 1008

    def oracle_for(idx, coords, labels, box, mask_in, mm, hw):
        f = seg._features
        emb = pred.get_image_embedding()[idx:idx + 1].float().cpu()
        hr = (f["feat_s0"][idx:idx + 1].permute(0, 3, 1, 2).float().cpu(), f["feat_s1"][idx:idx + 1].permute(0, 3, 1, 2).float().cpu())
        sc = torch.tensor([S / hw[1], S / hw[0]])
        pc = torch.as_tensor(coords, dtype=torch.float32) * sc if coords is not None else None
        pl = torch.as_tensor(labels, dtype=torch.int32) if labels is not None else None
        if pc is not None and pc.dim() == 2:
            pc, pl = pc[None], pl[None]
        bx = (torch.as_tensor(box, dtype=torch.float32).reshape(-1, 2, 2) * sc).reshape(-1, 4) if box is not None else None
        mi = torch.as_tensor(mask_in, dtype=torch.float32) if mask_in is not None else None
        if mi is not None and mi.dim() == 3:
            mi = mi[None]
        with torch.no_grad():
            return OH.predict(sd_pe, sd_md, emb, hr, pc, pl, bx, mi, S, hw, multimask_output=mm, return_logits=True,
                              mask_threshold=0.0, max_hole_area=64.0, max_sprinkle_area=16.0)

    def compare(got, ref, what):
        masks, iou, low = (torch.from_numpy(np.asarray(t)) for t in got)
        rm, ri, rl = ref
        rm, ri, rl = rm[0], ri[0], rl[0]
        assert masks.shape == rm.shape and low.shape == rl.shape, (masks.shape, rm.shape)
        e = rel_l2(low, rl)
        print(f"{what}: low-res rel_l2={e:.3e} iou err={(iou - ri).abs().max().item():.3e}")
        assert e <= 2e-2 and (iou - ri).abs().max().item() <= 3e-2
        agree = ((masks > 0) == (rm > 0)).float().mean().item()
        assert agree >= 0.99, (what, agree)

    # --- single image: point, box + point, then the returned low-res logits fed back as a mask prompt
    pred.set_image(imgs[0])
    hw = (300, 420)
    pc, pl = np.array([[210.0, 150.0], [30.0, 40.0]]), np.array([1, 0])
    out = pred.predict(point_coords=pc, point_labels=pl, multimask_output=True, return_logits=True)
    assert out[0].shape == (3, 300, 420) and out[1].shape == (3,) and out[2].shape == (3, 288, 288)
    compare(out, oracle_for(0, pc, pl, None, None, True, hw), "points")
    box = np.array([60.0, 50.0, 300.0, 220.0])
    out_b = pred.predict(point_coords=pc[:1], point_labels=pl[:1], box=box, multimask_output=False, return_logits=True)
    assert out_b[0].shape == (1, 300, 420)
    compare(out_b, oracle_for(0, pc[:1], pl[:1], box, None, False, hw), "box + point")
    out_m = pred.predict(point_coords=pc[:1], point_labels=pl[:1], mask_input=out_b[2], multimask_output=True, return_logits=True)
    compare(out_m, oracle_for(0, pc[:1], pl[:1], None, out_b[2], True, hw), "point + mask")
    # --- long prompts (repeated clicks): 6 output tokens + the points + the padding point pass 16 image-to-token keys
    many = np.stack([rng.uniform(0, 420, 20), rng.uniform(0, 300, 20)], 1)
    many_lab = rng.integers(0, 2, 20)
    for n, bx in ((10, None), (12, None), (20, None), (8, box)):
        out_n = pred.predict(point_coords=many[:n], point_labels=many_lab[:n], box=bx, multimask_output=bx is None, return_logits=True)
        compare(out_n, oracle_for(0, many[:n], many_lab[:n], bx, None, bx is None, hw), f"{'box + ' if bx is not None else ''}{n} points")
    bm = pred.predict(point_coords=pc, point_labels=pl, multimask_output=True)[0]
    # like the reference (`masks.squeeze(0).float()...numpy()`, :290) the thresholded masks come back as float32 0/1
    assert bm.dtype == np.float32 and set(np.unique(bm)) <= {0.0, 1.0} and np.array_equal(bm > 0.5, out[0] > 0)
    assert np.abs(out[2]).max() <= 32.0
    # --- batch of two images with per-image prompt lists; the second image gets two prompts (repeat_image path)
    pred.set_image_batch(imgs)
    pcs = [np.array([[100.0, 100.0]]), np.array([[[100.0, 200.0]], [[300.0, 50.0]]])]
    pls = [np.array([1]), np.array([[1], [1]])]
    masks, ious, lows = pred.predict_batch(pcs, pls, multimask_output=True, return_logits=True)
    assert masks[0].shape == (3, 300, 420) and masks[1].shape == (2, 3, 512, 384) and ious[1].shape == (2, 3)
    ref1 = oracle_for(1, pcs[1], pls[1], None, None, True, (512, 384))
    for j in range(2):
        compare((masks[1][j], ious[1][j], lows[1][j]), tuple(t[j:j + 1] for t in ref1), f"batch image 1 prompt {j}")
