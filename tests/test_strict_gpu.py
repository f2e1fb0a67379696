"""GPU: the strict (fp32-class) precision mode against the reference fixtures and the CPU oracle at north_star's tolerances:

    embeddings   rtol 1e-4   asserted as rel-L2 <= 1e-4 AND max|err| <= 1e-4 * max|ref|
    mask logits  rtol 1e-3   asserted as max|err| <= 1e-3 * max|logit| (measured ~1e-5)
    binary masks bit-exact   (logit > 0) identical on EVERY pixel of the fixtures

and the strict compositions conv2d_f32 (im2col + SGEMM), convt2x2_f32 and the SAM heads' fp32 twins against their torch statements in
tests/emu_strict.py.  The strict kernels themselves are held element by element to fp64 bounds: the ViT trunk's (sgemm_f32,
im2col_f32, ln_rows_f32, rope_f32, attention_f32) in tests/test_vit_kernels_gpu.py, the students' (dwconv_f32, litemla_attn_f32,
bilinear_nhwc_f32_to_nchw, bias_act_res_f32, scale_channels_f32) in tests/test_strict_kernels_gpu.py."""
from types import SimpleNamespace as NS

import pytest
import torch

import emu_strict as E
from helpers import load_golden, max_err_over_scale, rel_l2, sd_from_keys

pytestmark = pytest.mark.gpu

EMB_TOL = 1e-4          # north_star: embeddings rtol 1e-4
LOGIT_TOL = 1e-3        # north_star: mask logits rtol 1e-3


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close(got, ref, tol, what):
    err = max_err_over_scale(got.detach().cpu(), ref.detach().cpu())
    assert err <= tol, f"{what}: max err / scale = {err:.3e} > {tol}"


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("B,H,W,C,N,ks,stride,nchw", [(2, 9, 11, 16, 24, 3, 1, False), (1, 16, 16, 3, 16, 3, 2, True), (2, 7, 5, 32, 8, 1, 1, False),
                                                     (1, 10, 10, 64, 64, 3, 2, False), (1, 33, 31, 3, 8, 3, 2, True)])
def test_conv2d_f32(cuda, B, H, W, C, N, ks, stride, nchw):
    from efficientsam3_b200 import ops
    g = _g(B + H + C + N)
    x = torch.randn(B, C, H, W, generator=g) if nchw else torch.randn(B, H, W, C, generator=g)
    w = torch.randn(N, C, ks, ks, generator=g) / (C * ks * ks) ** 0.5
    sc, bi = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g)
    got = ops.conv2d_f32(x.to(cuda), w.to(cuda), stride, ks // 2, scale=sc.to(cuda), bias=bi.to(cuda), act="hswish", nchw=nchw)
    ref = E.conv2d_f32(x.double(), w.double(), stride, ks // 2, scale=sc.double(), bias=bi.double(), act="hswish", nchw=nchw)
    _close(got, ref.float(), 3e-6, "conv2d_f32")
    if not nchw and stride == 1:
        res = torch.randn_like(ref.float())
        got = ops.conv2d_f32(x.to(cuda), w.to(cuda), 1, ks // 2, bias=bi.to(cuda), residual=res.to(cuda))
        _close(got, E.conv2d_f32(x.double(), w.double(), 1, ks // 2, bias=bi.double(), residual=res.double()).float(), 3e-6, "conv2d_f32 + res")


def test_decoder_twins_f32(cuda):
    from efficientsam3_b200 import ops
    g = _g(4)
    B, Nq, Tk, H, hd = 2, 333, 8, 8, 16
    q, k, v = torch.randn(B * Nq, H * hd, generator=g), torch.randn(B, Tk, H * hd, generator=g), torch.randn(B, Tk, H * hd, generator=g)
    got = ops.attn_few_keys_f32(q.to(cuda), k.to(cuda), v.to(cuda), B, H, 0.25)
    _close(got, E.attn_few_keys_f32(q.double(), k.double(), v.double(), B, H, 0.25).float(), 2e-6, "attn_few_keys_f32")
    x, w, b = torch.randn(500, 64, generator=g) * 3, torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g)
    _close(ops.ln_rows_gelu_f32(x.to(cuda), w.to(cuda), b.to(cuda), 1e-6), E.ln_rows_gelu_f32(x.double(), w.double(), b.double(), 1e-6).float(),
           2e-6, "ln_rows_gelu_f32")
    xt, wt, bt = torch.randn(2, 9, 7, 64, generator=g), torch.randn(64, 32, 2, 2, generator=g) / 8, torch.randn(32, generator=g)
    r = torch.randn(2, 18, 14, 32, generator=g)
    got = ops.convt2x2_f32(xt.to(cuda), wt.to(cuda), bt.to(cuda), act="gelu", residual=r.to(cuda), act_after_res=True)
    _close(got, E.convt2x2_f32(xt.double(), wt.double(), bt.double(), act="gelu", residual=r.double(), act_after_res=True).float(), 3e-6, "convt2x2_f32")


# ------------------------------------------------------------------------------------------------ student encoders
def _student(name, img, embed, sd, dev):
    from efficientsam3_b200.stage1.model import build_image_student_model
    cfg = NS(MODEL=NS(BACKBONE=name), DATA=NS(IMG_SIZE=img), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=embed))
    m = build_image_student_model(cfg)
    m.load_state_dict(sd)
    return m.to(dev).eval()


STUDENTS = [("evm_160", "efficientvit_b1"), ("ev_b0_160", "efficientvit_b0"), ("ev_b2_192", "efficientvit_b2"), ("rvm_160", "repvit_m1_1"),
            ("rv_m0_9_128", "repvit_m0_9"), ("rv_m2_3_128", "repvit_m2_3"), ("tvm_160", "tiny_vit_11m"), ("tv_5m_160", "tiny_vit_5m"),
            ("tv_21m_160", "tiny_vit_21m")]


@pytest.mark.parametrize("fixture,name", STUDENTS)
def test_strict_student_matches_reference_fixture(cuda, fixture, name):
    from efficientsam3_b200 import ops
    g = load_golden(fixture)
    sd = sd_from_keys(g["keys"], int(g["seed_w"]))
    img, embed = int(g["img"]), int(g["embed"])
    m = _student(name, img, embed, sd, cuda)
    x = torch.randn(int(g["batch"]), 3, img, img, generator=_g(int(g["seed_x"]))).to(cuda)
    with ops.strict_precision():
        out = m(x)
        again = m(x)
    ref = torch.as_tensor(g["out"])
    l2, mx = rel_l2(out.cpu(), ref), max_err_over_scale(out.cpu(), ref)
    fast = m(x)                                              # bf16-operand mode on the same module, for the record
    print(f"{fixture}: strict rel-L2 {l2:.3e} max/scale {mx:.3e}   (bf16 mode rel-L2 {rel_l2(fast.cpu(), ref):.3e})")
    assert out.shape == ref.shape and l2 <= EMB_TOL and mx <= EMB_TOL, (l2, mx)
    assert torch.equal(out, again)                           # bit-reproducible
    assert rel_l2(fast.cpu(), ref) > 10 * l2                 # and the mode switch really switched


def test_strict_vit_trunk_matches_reference_fixture(cuda):
    """The SAM3 ViT trunk (the teacher) in the strict mode: RoPE, windowed + global attention, abs-pos tiling, all fp32."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model.vitdet import create_sam3_vit_backbone
    g = load_golden("vit_small_112")
    cfg = eval(str(g["cfg"]))
    m = create_sam3_vit_backbone(**cfg)
    m.load_state_dict(sd_from_keys(g["keys"], int(g["seed_w"])), strict=False)
    m = m.to(cuda).eval()
    x = torch.randn(int(g["batch"]), 3, cfg["img_size"], cfg["img_size"], generator=_g(int(g["seed_x"]))).to(cuda)
    with ops.strict_precision():
        out = m(x)[-1]
        again = m(x)[-1]
    fast = m(x)[-1]
    ref = torch.as_tensor(g["out"])
    l2, mx = rel_l2(out.cpu(), ref), max_err_over_scale(out.cpu(), ref)
    print(f"vit_small_112: strict rel-L2 {l2:.3e} max/scale {mx:.3e}   (bf16 mode rel-L2 {rel_l2(fast.cpu(), ref):.3e})")
    assert out.shape == ref.shape and l2 <= EMB_TOL and mx <= EMB_TOL, (l2, mx)
    assert torch.equal(out, again) and rel_l2(fast.cpu(), ref) > 10 * l2


def test_strict_teacher_geometry_vs_oracle(cuda):
    """Full-width teacher geometry (1008 px, 72 x 72 tokens, 24-windows, dim 1024, 16 heads; depth 3 so the CPU oracle takes seconds)
    through SAM3ImageTeacherEncoder in the strict mode."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.model import SAM3ImageTeacherEncoder
    from oracle import vitdet as O
    from oracle.weights import fill_state_dict
    over = dict(depth=3, global_att_blocks=(2,))
    t = SAM3ImageTeacherEncoder(embed_size=72, vit_overrides=over)
    vit = t.sam3.backbone.vision_backbone.trunk
    sd = {k: v for k, v in fill_state_dict(vit.state_dict(), 35).items() if not v.is_complex()}
    vit.load_state_dict(sd, strict=False)
    x = torch.randn(1, 3, 1008, 1008, generator=_g(10))
    from efficientsam3_b200.model.vitdet import SAM3_VIT_KWARGS
    with torch.no_grad():
        ref = O.vit_trunk(sd, "", x, dict(SAM3_VIT_KWARGS, **over))
    with ops.strict_precision():
        out = t.to(cuda)(x.to(cuda)).cpu()
    l2, mx = rel_l2(out, ref), max_err_over_scale(out, ref)
    print(f"teacher geometry (depth 3): strict rel-L2 {l2:.3e} max/scale {mx:.3e}")
    assert out.shape == ref.shape and l2 <= EMB_TOL and mx <= EMB_TOL, (l2, mx)


def test_strict_evm_at_the_headline_shape_vs_oracle(cuda):
    """EV-M at 1024^2 -> 64 x 64 (BASELINE shape), batch 2, against the fp32 CPU oracle of the reference modules."""
    from efficientsam3_b200 import ops
    from oracle import efficientvit as O
    g = load_golden("evm_160")
    sd = sd_from_keys(g["keys"], 21)
    m = _student("efficientvit_b1", 1024, 64, sd, cuda)
    x = torch.randn(2, 3, 1024, 1024, generator=_g(22))
    with torch.no_grad():
        ref = O.image_student_encoder(sd, x, 64, "b1")
    with ops.strict_precision():
        out = m(x.to(cuda)).cpu()
    fast = m(x.to(cuda)).cpu()
    l2, mx = rel_l2(out, ref), max_err_over_scale(out, ref)
    print(f"EV-M 1024^2 B=2: strict rel-L2 {l2:.3e} max/scale {mx:.3e}; bf16 mode rel-L2 {rel_l2(fast, ref):.3e}")
    assert l2 <= EMB_TOL and mx <= EMB_TOL, (l2, mx)
    assert rel_l2(fast, ref) <= 2e-2                         # the fast mode at the headline shape, its own (stated) tolerance


# ------------------------------------------------------------------------------------------------ SAM heads
def _heads(E_, S, sd_pe, sd_md, dev):
    from efficientsam3_b200.sam import MaskDecoder, PromptEncoder, TwoWayTransformer
    pe = PromptEncoder(embed_dim=256, image_embedding_size=(E_, E_), input_image_size=(S, S), mask_in_chans=16)
    md = MaskDecoder(num_multimask_outputs=3, transformer=TwoWayTransformer(depth=2, embedding_dim=256, mlp_dim=2048, num_heads=8),
                     transformer_dim=256, iou_head_depth=3, iou_head_hidden_dim=256, use_high_res_features=True,
                     iou_prediction_use_sigmoid=True, pred_obj_scores=True, pred_obj_scores_mlp=True, use_multimask_token_for_obj_ptr=True)
    pe.load_state_dict(sd_pe)
    md.load_state_dict(sd_md)
    return pe.to(dev).eval(), md.to(dev).eval()


def _strict_mask_checks(got, ref, what):
    err = (got.double() - ref.double()).abs().max().item()
    scale = ref.abs().max().item()
    flips = ((got > 0) != (ref > 0)).sum().item()
    print(f"{what}: max|err| {err:.3e} = {err / scale:.3e} of max|logit|; binary masks differ on {flips} of {ref.numel()} pixels")
    assert err <= LOGIT_TOL * scale, (what, err, scale)
    assert flips == 0, f"{what}: binary masks must be bit-exact in the strict mode ({flips} pixels differ)"


def test_strict_heads_masks_are_bit_exact_on_the_reference_fixture(cuda):
    from efficientsam3_b200 import ops
    g = load_golden("sam_heads_16")
    E_, S, B = int(g["E"]), int(g["S"]), int(g["B"])
    pe, md = _heads(E_, S, sd_from_keys(g["keys_pe"], int(g["seed_pe"])), sd_from_keys(g["keys_md"], int(g["seed_md"])), cuda)
    gen = _g(int(g["seed_x"]))
    feat = torch.randn(B, 256, E_, E_, generator=gen).to(cuda)
    f288 = torch.randn(B, 256, 4 * E_, 4 * E_, generator=gen).to(cuda)
    f144 = torch.randn(B, 256, 2 * E_, 2 * E_, generator=gen).to(cuda)
    coords = (torch.rand(B, 1, 2, generator=gen) * S).to(cuda)
    labels = torch.ones(B, 1, dtype=torch.int32, device=cuda)
    with ops.strict_precision():
        sp, de = pe(points=(coords, labels), boxes=None, masks=None)
        dpe = pe.get_dense_pe()
        hr = [t.permute(0, 3, 1, 2).contiguous() for t in md.project_high_res(f288.permute(0, 2, 3, 1).contiguous(), f144.permute(0, 2, 3, 1).contiguous())]
        for mm, sfx in ((True, "mm"), (False, "single")):
            m, iou, tok, obj = md(image_embeddings=feat, image_pe=dpe, sparse_prompt_embeddings=sp, dense_prompt_embeddings=de,
                                  multimask_output=mm, repeat_image=False, high_res_features=hr)
            _strict_mask_checks(m.cpu(), torch.from_numpy(g[f"masks_{sfx}"]), f"strict fixture masks {sfx}")
            assert (iou.cpu() - torch.from_numpy(g[f"iou_{sfx}"])).abs().max() <= 1e-4
            assert (obj.cpu() - torch.from_numpy(g[f"obj_{sfx}"])).abs().max() <= 1e-3
            assert rel_l2(tok.cpu(), g[f"tok_{sfx}"]) <= 1e-4
            assert torch.equal(iou.cpu().argmax(-1), torch.from_numpy(g[f"iou_{sfx}"]).argmax(-1))
        q, k = md.transformer(feat, dpe.expand(B, -1, -1, -1), torch.cat([sp, sp], dim=1))
        assert rel_l2(q.cpu(), g["twoway_q"]) <= 1e-4


def test_strict_box_and_mask_prompts_are_bit_exact_on_the_reference_fixture(cuda):
    from efficientsam3_b200 import ops
    g = load_golden("sam_prompts_12")
    E_, S, P = int(g["E"]), int(g["S"]), int(g["P"])
    gen = _g(int(g["seed_x"]))
    feat = torch.randn(1, 256, E_, E_, generator=gen)
    f288 = torch.randn(1, 256, 4 * E_, 4 * E_, generator=gen)
    f144 = torch.randn(1, 256, 2 * E_, 2 * E_, generator=gen)
    coords = torch.rand(P, 2, 2, generator=gen) * S
    labels = torch.tensor([[1, 0], [1, 1], [0, 1]], dtype=torch.int32)
    xy0 = torch.rand(P, 2, generator=gen) * S * 0.5
    boxes = torch.cat([xy0, xy0 + 8 + torch.rand(P, 2, generator=gen) * S * 0.4], dim=1)
    mask_in = torch.randn(P, 1, 4 * E_, 4 * E_, generator=gen) * 4
    pe, md = _heads(E_, S, sd_from_keys(g["keys_pe"], int(g["seed_pe"])), sd_from_keys(g["keys_md"], int(g["seed_md"])), cuda)
    c = lambda t: t.to(cuda)
    cc = torch.cat([boxes.reshape(-1, 2, 2), coords], dim=1)
    cl = torch.cat([torch.tensor([[2, 3]], dtype=torch.int32).repeat(P, 1), labels], dim=1)
    with ops.strict_precision():
        sp2, de2 = pe(points=(c(cc), c(cl)), boxes=None, masks=c(mask_in))
        # conv_s0 / conv_s1 through the strict SGEMM (F.conv2d on the GPU would run cuDNN's TF32 path: 1e-3 off fp32)
        hr = [t.permute(0, 3, 1, 2).contiguous() for t in md.project_high_res(c(f288).permute(0, 2, 3, 1).contiguous(),
                                                                               c(f144).permute(0, 2, 3, 1).contiguous())]
        for mm, sfx in ((True, "mm"), (False, "single")):
            masks, iou, tok, obj = md(image_embeddings=c(feat), image_pe=pe.get_dense_pe(), sparse_prompt_embeddings=sp2,
                                      dense_prompt_embeddings=de2, multimask_output=mm, repeat_image=True, high_res_features=hr)
            _strict_mask_checks(masks.cpu(), torch.from_numpy(g[f"masks_{sfx}"]), f"strict repeat_image masks ({sfx})")
            assert (iou.cpu() - torch.from_numpy(g[f"iou_{sfx}"])).abs().max().item() <= 1e-4


def test_strict_efficientsam3_segmenter_vs_oracles(cuda):
    """EfficientSAM3 (EV-M student encoder -> FPN -> SAM heads -> 1008^2 masks) end to end in the strict mode against the oracle
    composition: low-res logits at rtol 1e-3, binary masks bit-exact outside a 1e-4 band (and the number of pixels inside it)."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model_builder import build_efficientsam3_point_segmenter
    from oracle import efficientvit as EV, necks as ON, sam_heads as OH
    from oracle.weights import fill_state_dict
    S, B = 448, 2
    seg = build_efficientsam3_point_segmenter("efficientvit", "b1", image_size=S)
    # weight seed 51: the oracle's object score is negative for image 0 (masks gated to -1024) and positive for image 1
    sd = {k: v for k, v in fill_state_dict(seg.state_dict(), 51).items() if not v.is_complex()}
    seg.load_state_dict(sd, strict=False)
    seg = seg.to(cuda)
    g = _g(6)
    img = torch.randn(B, 3, S, S, generator=g)
    coords = torch.rand(B, 1, 2, generator=g) * S
    labels = torch.ones(B, 1, dtype=torch.int32)
    with ops.strict_precision():
        res = seg.set_image_batch(img.to(cuda)).predict_batch(coords.to(cuda), labels.to(cuda), multimask_output=True, return_logits=True)
    with torch.no_grad():
        vb = {k[len("backbone.vision_backbone."):]: v for k, v in sd.items() if k.startswith("backbone.vision_backbone.")}
        feats = EV.image_student_encoder({k[len("trunk.model."):]: v for k, v in vb.items() if k.startswith("trunk.model.")}, img, S // 14, "b1")
        l288, l144, l72 = ON.neck(vb, feats, prefix="sam2_convs.")[:3]
        sd_md = {k[len("sam_mask_decoder."):]: v for k, v in sd.items() if k.startswith("sam_mask_decoder.")}
        sd_pe = {k[len("sam_prompt_encoder."):]: v for k, v in sd.items() if k.startswith("sam_prompt_encoder.")}
        hr = OH.high_res_from_fpn(sd_md, "", l288, l144)
        ref = OH.forward_sam_heads(sd_pe, sd_md, l72 + sd["no_mem_embed"].reshape(1, -1, 1, 1), hr, coords, labels, S, multimask_output=True)
    low, refl = res["low_res_multimasks"].cpu(), ref["low_res_multimasks"]
    assert torch.equal(res["object_score_logits"].cpu() > 0, ref["object_score_logits"] > 0)      # same images gated
    assert (refl > -1000).any() and (refl < -1000).any()
    err = (low.double() - refl.double()).abs().max().item()
    scale = refl[refl > -1000].abs().max().item()
    print(f"strict EfficientSAM3 pipeline: low-res max|err| {err:.3e} = {err / scale:.3e} of max|logit|")
    assert err <= LOGIT_TOL * scale
    hi, refh = res["high_res"].cpu(), ref["high_res_multimasks"]
    band = refh.abs() <= 1e-4 * scale
    flips = ((hi > 0) != (refh > 0))
    print(f"high-res binary masks: {flips.sum().item()} of {hi.numel()} pixels differ; {band.sum().item()} pixels inside the 1e-4 band")
    assert (flips & ~band).sum().item() == 0
    assert torch.equal(res["best"].cpu(), ref["best"])
