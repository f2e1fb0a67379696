"""GPU parity of the SAM heads (PromptEncoder + TwoWayTransformer + MaskDecoder) through the reference-shaped
module API (-> C ABI).

Tolerances (stated; north-star: mask logits rtol 1e-3, argmax masks bit-exact): the image stream runs bf16 GEMM
operands with fp32 accumulation/residuals, the token stream and the hypernetwork tail are fp32.  Asserted: mask
logits rel-L2 <= 1e-2 and max|err| <= 2e-2 * max|logit|; IoU / object logits abs err <= 2e-2; the best-mask index
equals the reference's; binary masks (logit > 0) agree on every pixel whose reference |logit| exceeds the measured
max error (bit-exact outside the rounding band) and on >= 99.5 % of all pixels.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from es3_recorder import sam_heads as _build
from helpers import cosine, load_golden, max_err_over_scale, rel_l2, sd_from_keys

pytestmark = pytest.mark.gpu


def _inputs(B, E, S, seed):
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(B, 256, E, E, generator=g)
    f288 = torch.randn(B, 256, 4 * E, 4 * E, generator=g)
    f144 = torch.randn(B, 256, 2 * E, 2 * E, generator=g)
    coords = torch.rand(B, 1, 2, generator=g) * S
    labels = torch.ones(B, 1, dtype=torch.int32)
    return feat, f288, f144, coords, labels


def _mask_checks(got, ref, what):
    l2, mx = rel_l2(got, ref), max_err_over_scale(got, ref)
    err = (got.double() - ref.double()).abs().max().item()
    agree = ((got > 0) == (ref > 0)).float().mean().item()
    safe = ref.abs() > err
    print(f"{what}: rel_l2={l2:.3e} max/scale={mx:.3e} abs_err={err:.3e} binary agreement={agree:.5f} "
          f"({(~safe).float().mean().item():.4%} of pixels inside the rounding band)")
    assert l2 <= 1e-2 and mx <= 2e-2, (what, l2, mx)
    assert torch.equal((got > 0)[safe], (ref > 0)[safe])
    assert agree >= 0.995


def test_key_order_matches_reference_record():
    g = load_golden("sam_heads_16")
    from efficientsam3_b200.sam import MaskDecoder, PromptEncoder, TwoWayTransformer  # noqa: F401
    pe, md = _build(16, 224, sd_from_keys(g["keys_pe"], 5), sd_from_keys(g["keys_md"], 6), "cpu")
    sig = lambda sd: [f"{k}|{','.join(map(str, v.shape))}|{str(v.dtype).replace('torch.', '')}" for k, v in sd.items()]
    assert sig(pe.state_dict()) == [str(k) for k in g["keys_pe"]]
    assert sig(md.state_dict()) == [str(k) for k in g["keys_md"]]


def test_heads_match_reference_fixture(cuda):
    g = load_golden("sam_heads_16")
    E, S, B = int(g["E"]), int(g["S"]), int(g["B"])
    pe, md = _build(E, S, sd_from_keys(g["keys_pe"], int(g["seed_pe"])), sd_from_keys(g["keys_md"], int(g["seed_md"])), cuda)
    feat, f288, f144, coords, labels = [t.to(cuda) for t in _inputs(B, E, S, int(g["seed_x"]))]
    sp, de = pe(points=(coords, labels), boxes=None, masks=None)
    assert max_err_over_scale(sp.cpu(), g["sparse"]) < 1e-5
    dpe = pe.get_dense_pe()
    assert max_err_over_scale(dpe.cpu()[:, :, ::4, ::4], g["dense_pe"]) < 1e-5
    hr = [F.conv2d(f288, md.conv_s0.weight, md.conv_s0.bias), F.conv2d(f144, md.conv_s1.weight, md.conv_s1.bias)]  # test-side prep
    for mm, sfx in ((True, "mm"), (False, "single")):
        m, iou, tok, obj = md(image_embeddings=feat, image_pe=dpe, sparse_prompt_embeddings=sp, dense_prompt_embeddings=de,
                              multimask_output=mm, repeat_image=False, high_res_features=hr)
        _mask_checks(m.cpu(), torch.from_numpy(g[f"masks_{sfx}"]), f"fixture masks {sfx}")
        assert (iou.cpu() - torch.from_numpy(g[f"iou_{sfx}"])).abs().max() <= 2e-2
        assert (obj.cpu() - torch.from_numpy(g[f"obj_{sfx}"])).abs().max() <= 2e-2
        assert rel_l2(tok.cpu(), g[f"tok_{sfx}"]) <= 1e-2
        assert torch.equal(iou.cpu().argmax(-1), torch.from_numpy(g[f"iou_{sfx}"]).argmax(-1))
    q, k = md.transformer(feat, dpe.expand(B, -1, -1, -1), torch.cat([sp, sp], dim=1))
    assert rel_l2(q.cpu(), g["twoway_q"]) <= 1e-2


def test_heads_full_size_vs_oracle(cuda):
    """Config-3 geometry: 72x72 embeddings, 1008 px, 288x288 low-res masks, batch 4, against the CPU oracle,
    plus the upsample + threshold tail (sam3_tracker_base.py:344-360)."""
    from oracle import sam_heads as O
    from efficientsam3_b200 import ops
    g = load_golden("sam_heads_16")
    E, S, B = 72, 1008, 4
    sd_pe, sd_md = sd_from_keys(g["keys_pe"], 15), sd_from_keys(g["keys_md"], 16)
    feat, f288, f144, coords, labels = _inputs(B, E, S, 3)
    with torch.no_grad():
        hr = O.high_res_from_fpn(sd_md, "", f288, f144)
        ref = O.forward_sam_heads(sd_pe, sd_md, feat, hr, coords, labels, S, multimask_output=True)
    pe, md = _build(E, S, sd_pe, sd_md, cuda)
    sp, de = pe(points=(coords.to(cuda), labels.to(cuda)), boxes=None, masks=None)
    m, iou, tok, obj = md(image_embeddings=feat.to(cuda), image_pe=pe.get_dense_pe(), sparse_prompt_embeddings=sp,
                          dense_prompt_embeddings=de, multimask_output=True, repeat_image=False,
                          high_res_features=[h.to(cuda) for h in hr])
    _mask_checks(m.cpu(), ref["low_res_ungated"], "full-size low-res masks (ungated)")
    assert (obj.cpu() - ref["object_score_logits"]).abs().max() <= 2e-2
    assert torch.equal(obj.cpu() > 0, ref["object_score_logits"] > 0)
    gated = torch.where((obj > 0)[:, None, None], m, torch.full_like(m, -1024.0))
    _mask_checks(gated.cpu(), ref["low_res_multimasks"], "full-size low-res masks (object-gated)")
    hi_u, _ = ops.bilinear_nchw(m, S, S)
    _mask_checks(hi_u.cpu(), ref["high_res_ungated"], "full-size high-res masks (ungated)")
    assert torch.equal(iou.cpu().argmax(-1), ref["best"])
    assert (iou.cpu() - ref["ious"]).abs().max() <= 2e-2
    high, binm = ops.bilinear_nchw(gated, S, S, binarize_thr=0.0)
    _mask_checks(high.cpu(), ref["high_res_multimasks"], "full-size high-res masks")
    assert torch.equal(binm.bool().cpu(), high.cpu() > 0)


@pytest.mark.parametrize("Tk,hd,kv32", [(8, 32, True), (5184, 16, False), (100, 16, False), (33, 32, True)])
def test_attn_few_queries(cuda, Tk, hd, kv32):
    from efficientsam3_b200 import ops
    B, Tq, H = 2, 8, 8
    g = torch.Generator().manual_seed(Tk)
    q = torch.randn(B, Tq, H * hd, generator=g).to(cuda)
    k = torch.randn(B, Tk, H * hd, generator=g).to(cuda)
    v = torch.randn(B, Tk, H * hd, generator=g).to(cuda)
    if not kv32:
        k, v = k.bfloat16(), v.bfloat16()
    out = ops.attn_few_queries(q, k, v, H, hd ** -0.5)
    sep = lambda t: t.float().view(B, -1, H, hd).transpose(1, 2)
    ref = F.scaled_dot_product_attention(sep(q), sep(k), sep(v)).transpose(1, 2).reshape(B, Tq, H * hd)
    assert max_err_over_scale(out.cpu(), ref.cpu()) < 1e-4


def test_attn_few_keys_and_convt(cuda):
    from efficientsam3_b200 import ops
    B, Nq, Tk, H, hd = 2, 777, 8, 8, 16
    g = torch.Generator().manual_seed(0)
    q = torch.randn(B * Nq, H * hd, generator=g).bfloat16().to(cuda)
    k = torch.randn(B, Tk, H * hd, generator=g).to(cuda)
    v = torch.randn(B, Tk, H * hd, generator=g).to(cuda)
    out = ops.attn_few_keys(q, k, v, B, H, 0.25)
    sep = lambda t, n: t.float().view(B, n, H, hd).transpose(1, 2)
    ref = F.scaled_dot_product_attention(sep(q, Nq), sep(k, Tk), sep(v, Tk)).transpose(1, 2).reshape(B * Nq, H * hd)
    assert max_err_over_scale(out.cpu(), ref.cpu()) < 1e-2
    # ConvTranspose2d(k=2,s=2) + bias + fp32 residual, gelu after the residual
    x = torch.randn(2, 9, 7, 64, generator=g).bfloat16().to(cuda)
    w = (torch.randn(64, 32, 2, 2, generator=g) / 8).to(cuda)
    b = torch.randn(32, generator=g).to(cuda)
    r = torch.randn(2, 18, 14, 32, generator=g).to(cuda)
    y = ops.convt2x2(x, ops.convt2x2_weight(w), bias4=b.repeat(4).contiguous(), act="gelu", residual=r,
                     out_dtype=torch.float32, act_after_res=True)
    ref = F.gelu(F.conv_transpose2d(x.float().permute(0, 3, 1, 2), w.bfloat16().float(), b, stride=2) + r.permute(0, 3, 1, 2))
    assert max_err_over_scale(y.cpu(), ref.permute(0, 2, 3, 1).cpu()) < 2e-3


# ---- box / mask prompts, several prompts per image, hole filling (sam1_task_predictor.py:329-430) --------------------
def _prompt_inputs(g):
    E, S, P = int(g["E"]), int(g["S"]), int(g["P"])
    gen = torch.Generator().manual_seed(int(g["seed_x"]))
    feat = torch.randn(1, 256, E, E, generator=gen)
    f288 = torch.randn(1, 256, 4 * E, 4 * E, generator=gen)
    f144 = torch.randn(1, 256, 2 * E, 2 * E, generator=gen)
    coords = torch.rand(P, 2, 2, generator=gen) * S
    labels = torch.tensor([[1, 0], [1, 1], [0, 1]], dtype=torch.int32)
    xy0 = torch.rand(P, 2, generator=gen) * S * 0.5
    boxes = torch.cat([xy0, xy0 + 8 + torch.rand(P, 2, generator=gen) * S * 0.4], dim=1)
    mask_in = torch.randn(P, 1, 4 * E, 4 * E, generator=gen) * 4
    return E, S, P, feat, f288, f144, coords, labels, boxes, mask_in


def test_box_and_mask_prompts_match_reference_fixture(cuda):
    g = load_golden("sam_prompts_12")
    E, S, P, feat, f288, f144, coords, labels, boxes, mask_in = _prompt_inputs(g)
    pe, md = _build(E, S, sd_from_keys(g["keys_pe"], int(g["seed_pe"])), sd_from_keys(g["keys_md"], int(g["seed_md"])), cuda)
    c = lambda t: t.to(cuda)
    sp, de = pe(points=(c(coords), c(labels)), boxes=c(boxes), masks=c(mask_in))
    assert sp.shape == (P, 4, 256) and de.shape == (P, 256, E, E)
    assert (sp.cpu() - torch.from_numpy(g["sparse_pts_boxes"])).abs().max().item() <= 2e-5
    ref0 = torch.from_numpy(g["dense_mask0"])
    assert (de[:1].cpu() - ref0).abs().max().item() <= 1e-4 * ref0.abs().max().item()
    for i in range(P):
        d = de[i].double()
        got = torch.tensor([d.mean().item(), d.abs().mean().item(), d.std().item()], dtype=torch.float64)
        assert torch.allclose(got, torch.from_numpy(g["dense_mask_stats"][i]).double(), rtol=1e-3, atol=1e-5)
    # predictor-style merge (boxes in front as label-2/3 points, padding point appended) + repeat_image decoding
    cc = torch.cat([boxes.reshape(-1, 2, 2), coords], dim=1)
    cl = torch.cat([torch.tensor([[2, 3]], dtype=torch.int32).repeat(P, 1), labels], dim=1)
    sp2, de2 = pe(points=(c(cc), c(cl)), boxes=None, masks=c(mask_in))
    assert (sp2.cpu() - torch.from_numpy(g["sparse_merged"])).abs().max().item() <= 2e-5
    hr = [F.conv2d(c(f288), md.conv_s0.weight, md.conv_s0.bias), F.conv2d(c(f144), md.conv_s1.weight, md.conv_s1.bias)]
    for mm, sfx in ((True, "mm"), (False, "single")):
        masks, iou, tok, obj = md(image_embeddings=c(feat), image_pe=pe.get_dense_pe(), sparse_prompt_embeddings=sp2,
                                  dense_prompt_embeddings=de2, multimask_output=mm, repeat_image=True, high_res_features=hr)
        _mask_checks(masks.cpu(), torch.from_numpy(g[f"masks_{sfx}"]), f"repeat_image masks ({sfx})")
        assert (iou.cpu() - torch.from_numpy(g[f"iou_{sfx}"])).abs().max().item() <= 2e-2
        assert (obj.cpu() - torch.from_numpy(g[f"obj_{sfx}"])).abs().max().item() <= 2e-2


@pytest.mark.parametrize("case", ["fixture", "speckle288", "empty", "full", "checker"])
def test_fill_small_components_is_exact(cuda, case):
    """Integer / index work: the filled masks must equal the oracle's bit for bit (same float inputs, same 8-connectivity)."""
    from efficientsam3_b200 import ops
    from oracle import sam_heads as O
    if case == "fixture":
        g = load_golden("sam_prompts_12")
        x = torch.from_numpy(g["post_in"])
        hole, spr = 12.0, 5.0
        ref_resized = torch.from_numpy(g["post_out"])
    else:
        gen = torch.Generator().manual_seed(3)
        if case == "speckle288":
            x = F.avg_pool2d(torch.randn(2, 3, 288, 288, generator=gen), 5, 1, 2) * 3 + torch.randn(2, 3, 288, 288, generator=gen) * 0.3
        elif case == "empty":
            x = -torch.rand(1, 2, 40, 56, generator=gen) - 0.1
        elif case == "full":
            x = torch.rand(1, 2, 40, 56, generator=gen) + 0.1
        else:  # diagonal-only connections: one component under 8-connectivity, singletons under 4-connectivity
            yy, xx = torch.meshgrid(torch.arange(33), torch.arange(47), indexing="ij")
            x = (((yy + xx) % 2).float() * 2 - 1)[None, None].repeat(1, 2, 1, 1)
            x[0, 1] = -x[0, 1]
        hole, spr = 256.0, 9.0
        ref_resized = None
    got = ops.fill_small_components(x.to(cuda), 0.0, hole, spr).cpu()
    ref = O.fill_holes(x, 0.0, hole, spr)
    assert torch.equal(got, ref), f"{case}: {(got != ref).sum().item()} pixels differ"
    if case == "speckle288":
        assert (got != x).sum().item() > 1000          # the case really exercises the filling
    if ref_resized is not None:
        up, _ = ops.bilinear_nchw(got.to(cuda), 50, 70)
        assert (up.cpu() - ref_resized).abs().max().item() <= 1e-5 * ref_resized.abs().max().item()
    # only holes / only sprinkles
    assert torch.equal(ops.fill_small_components(x.to(cuda), 0.0, hole, 0.0).cpu(), O.fill_holes(x, 0.0, hole, 0.0))
    assert torch.equal(ops.fill_small_components(x.to(cuda), 0.0, 0.0, spr).cpu(), O.fill_holes(x, 0.0, 0.0, spr))
