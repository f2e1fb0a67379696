"""Records the es3_* calls a piece of native work makes (tests/test_route_closure_gpu.py): every _lib.call, and every _lib.call_rc
that ran (rc == 0; a declined shape returns -1); and builds the model paths recorded there -- the image students' eval forward and
training step (the eval forward in both precision modes), whole stage-1 image and text iterations (train_one_epoch and
train_text_one_epoch with the optimiser update), the text students' training steps and the SAM3 text teacher, the interactive predictor and the SAM heads' module
API, the SAM3 image teacher (bf16, strict and FP8), ViT backbones and the point segmenter's set_image."""
import numpy as np
import torch

STUDENTS = ["efficientvit_b0", "efficientvit_b1", "efficientvit_b2", "repvit_m0_9", "repvit_m1_1", "repvit_m2_3", "tiny_vit_5m",
            "tiny_vit_11m", "tiny_vit_21m"]


def record_calls(monkeypatch, run):
    """Run `run()` with the es3 entry points recorded; returns [(name, args)] in call order."""
    from efficientsam3_b200 import _lib as L
    calls = []
    real_call, real_rc = L.call, L.call_rc

    def rc_rec(n, *a):
        rc = real_rc(n, *a)
        if rc == 0:
            calls.append((n, a))
        return rc
    monkeypatch.setattr(L, "call", lambda n, *a: (calls.append((n, a)), real_call(n, *a))[1])
    monkeypatch.setattr(L, "call_rc", rc_rec)
    try:
        run()
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    return calls


def student(cuda, name, img, embed):
    """The stage-1 image student `name` with deterministic weights, on `cuda`."""
    from types import SimpleNamespace as NS
    from efficientsam3_b200.stage1.model import build_image_student_model
    from oracle.weights import fill_state_dict
    cfg = NS(MODEL=NS(BACKBONE=name), DATA=NS(IMG_SIZE=img), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=embed))
    m = build_image_student_model(cfg)
    m.load_state_dict(fill_state_dict(m.state_dict(), 3))
    return m.to(cuda)


def training_step_calls(cuda, monkeypatch, name, frozen_bn, img=1024, embed=64, B=1):
    """The es3_* calls of one native KD training step (forward, loss, backward) of `name`."""
    from efficientsam3_b200.stage1.optim import KDLossFunction
    m = student(cuda, name, img, embed).train()
    if frozen_bn:
        for mod in m.modules():
            if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
                mod.eval()
    g = torch.Generator(device=cuda).manual_seed(0)
    x = torch.randn(B, 3, img, img, device=cuda, generator=g)
    teacher = torch.randn(B, 1024, embed, embed, device=cuda, generator=g)
    sz = torch.tensor([[img, img]] * B, dtype=torch.int32, device=cuda)
    return record_calls(monkeypatch, lambda: KDLossFunction.apply(m(x), teacher, sz, img, 1.0).backward())


def _stage1_cfg(**distill):
    from types import SimpleNamespace as NS
    return NS(TRAIN=NS(ACCUMULATION_STEPS=2, EPOCHS=3, WARMUP_EPOCHS=1, MIN_LR=1e-5, WARMUP_LR=1e-6, CLIP_GRAD=5.0,
                       EVAL_BN_WHEN_TRAINING=False), DISTILL=NS(COSINE=1.0, **distill))


def image_epoch_calls(cuda, monkeypatch, name, img=1024, embed=64):
    """The es3_* calls of stage1.train.train_one_epoch over `name` with batch-statistics BatchNorm and FlatAdamW with a dynamic loss
    scale: a two-iteration loader, ACCUMULATION_STEPS 2 (one update, clipped at 5), each batch two decoded uint8 images of different
    sizes (prepared on the device, so the masks pad) and the stored fp16 embeddings."""
    from types import SimpleNamespace as NS
    from efficientsam3_b200.stage1.optim import FlatAdamW
    from efficientsam3_b200.stage1.train import train_one_epoch
    m = student(cuda, name, img, embed)
    cfg = _stage1_cfg(EMBED_DIM=1024, EMBED_SIZE=embed)
    cfg.DATA = NS(IMG_SIZE=img)
    opt = FlatAdamW(m, lr=1e-4, weight_decay=0.05, loss_scale=65536.0, dynamic_loss_scale=True)
    g = torch.Generator().manual_seed(7)
    rng = np.random.default_rng(7)

    def batch(i):
        imgs = [torch.randint(0, 256, hw + (3,), dtype=torch.uint8, generator=g) for hw in ((480, 640), (700, 500))]
        embs = [(rng.standard_normal(1024 * embed * embed) * 0.5).astype(np.float16) for _ in imgs]
        return (imgs, None), (embs, [i, i])
    loader = [batch(i) for i in range(2)]
    return record_calls(monkeypatch, lambda: train_one_epoch(cfg, m, loader, opt, epoch=0))


def text_epoch_calls(cuda, monkeypatch, backbone, layers=2, ctx=32):
    """The es3_* calls of stage1.train.train_text_one_epoch over a depth-`layers` text student (`backbone`), FlatAdamW without its
    unused projection, masked loss with consistency, ACCUMULATION_STEPS 2 over a two-iteration loader of stored fp16 embeddings.
    MobileCLIP-S0 trains with batch-statistics BatchNorm (enable_batch_stat_bn, TRAIN.EVAL_BN_WHEN_TRAINING False)."""
    import random
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.model import text_student_cfg
    from efficientsam3_b200.stage1.optim import FlatAdamW
    from efficientsam3_b200.stage1.train import train_text_one_epoch
    from oracle.weights import fill_state_dict
    from test_text_cpu import BPE
    cfg = text_student_cfg(backbone)
    cfg["n_transformer_layers"] = layers
    cfg["context_length"] = ctx
    m = TextStudentEncoder(cfg=cfg, context_length=ctx, output_dim=256, bpe_path=BPE)
    m.load_state_dict(fill_state_dict(m.state_dict(), 21))
    m = m.to(cuda)
    if backbone == "MobileCLIP-S0":
        m.enable_batch_stat_bn()
    opt = FlatAdamW(m, lr=1e-3, weight_decay=0.05, loss_scale=65536.0, dynamic_loss_scale=True,
                    exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    tcfg = _stage1_cfg(NUM_EMBED=ctx, EMBED_DIM=256, MASK_PAD_TOKENS=True, CONSISTENCY_LOSS=0.5)
    caps = _captions(6)
    rng = np.random.default_rng(8)
    loader = [[list(caps), [[(rng.standard_normal(ctx * 256) * 0.5).astype(np.float16) for _ in caps], list(range(6))]]
              for _ in range(2)]
    random.seed(5)
    return record_calls(monkeypatch, lambda: train_text_one_epoch(tcfg, m, loader, opt, epoch=0))


def eval_forward_calls(cuda, monkeypatch, name, img=1024, embed=64, B=2, strict=False):
    """The es3_* calls of one eval forward of `name`, in the strict precision mode or not."""
    from efficientsam3_b200 import ops
    m = student(cuda, name, img, embed).eval()
    x = torch.randn(B, 3, img, img, device=cuda, generator=torch.Generator(device=cuda).manual_seed(0))

    def run():
        with torch.no_grad():
            if strict:
                with ops.strict_precision():
                    m(x)
            else:
                m(x)
    return record_calls(monkeypatch, run)


# (label, backbone, context, positional-table length (None: the context), masked loss, consistency weight, captions): one native
# text training step each -- S0 with frozen BN, S1, B (causal) and MobileCLIP2-S3 (width 768) at contexts 32 and 77, the 77-entry
# table at 32 and at 128 (the longest sequence the text kernels take: B's causal attention on 128-row tiles), masked and plain
# loss, with consistency; and 512 captions x 77 tokens, whose LayerNorm backward runs over more rows than 592 blocks of 64.
TEXT_ROUTES = [("S0 frozen BN", "MobileCLIP-S0", 32, None, True, 0.5, 6), ("S1", "MobileCLIP-S1", 32, None, True, 0.5, 6),
               ("B ctx 77", "MobileCLIP-B", 77, None, False, 0.0, 6), ("B ctx 128", "MobileCLIP-B", 128, 77, True, 0.5, 6),
               ("S3 table 77 at 32", "MobileCLIP2-S3", 32, 77, True, 0.5, 6), ("S3 batch 512", "MobileCLIP2-S3", 77, None, False, 0.5, 512)]


def _captions(n):
    from helpers import load_golden
    caps = [str(s) for s in load_golden("text_tokens")["strings"][:6]]
    return [caps[i % len(caps)] + (f" number {i}" if i >= len(caps) else "") for i in range(n)]


def text_step_calls(cuda, monkeypatch, backbone, ctx, table, masked, w_con, ncap, layers=2):
    """The es3_* calls of one native text training step (forward, KD loss with consistency over two word permutations, backward) of
    a depth-`layers` text student with deterministic weights, BatchNorm frozen (S0's RepMixerBlocks)."""
    import random
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import TextKDLossFunction, permute_words
    from efficientsam3_b200.stage1.model import text_student_cfg
    from oracle.weights import fill_state_dict
    from test_text_cpu import BPE
    cfg = text_student_cfg(backbone)
    cfg["n_transformer_layers"] = layers
    cfg["context_length"] = table or ctx
    m = TextStudentEncoder(cfg=cfg, context_length=ctx, output_dim=256, bpe_path=BPE)
    m.load_state_dict(fill_state_dict(m.state_dict(), 21))
    m = m.to(cuda).train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
            mod.eval()
    caps = _captions(ncap)
    random.seed(5)
    perms = [[permute_words(s) for s in caps] for _ in range(2)] if w_con > 0 else []
    teacher = torch.randn(ncap, ctx, 256, device=cuda, generator=torch.Generator(device=cuda).manual_seed(0))

    def step():
        pad, mem, _ = m(caps)
        qs = [m(pc)[1].transpose(0, 1) for pc in perms]
        loss, _, _, _ = TextKDLossFunction.apply(mem.transpose(0, 1), teacher, pad if masked else None, 1.0, w_con, *qs)
        loss.backward()
    return record_calls(monkeypatch, step)


def text_teacher_calls(cuda, monkeypatch):
    """The es3_* calls of the eval forward of the SAM3 text encoder as model_builder.create_text_encoder builds it (width 1024,
    16 heads, 24 layers, causal), deterministic weights."""
    from efficientsam3_b200.model_builder import create_text_encoder
    from oracle.weights import fill_state_dict
    from test_text_cpu import BPE
    t = create_text_encoder(BPE)
    t.load_state_dict(fill_state_dict(t.state_dict(), 106))
    t = t.to(cuda).eval()
    caps = _captions(6)

    def run():
        with torch.no_grad():
            t(caps, device=cuda)
    return record_calls(monkeypatch, run)


def point_segmenter(kind, cuda):
    """Sam3PointPromptSegmenter with deterministic weights: the ViT override with one windowed block ("vit") or EV-B1 at 448 px."""
    from efficientsam3_b200.model.sam1_task import Sam3PointPromptSegmenter
    from efficientsam3_b200.model_builder import build_efficientsam3_point_segmenter
    from oracle.weights import fill_state_dict
    if kind == "vit":
        seg = Sam3PointPromptSegmenter(vit_overrides=dict(depth=1, global_att_blocks=()))
    else:
        seg = build_efficientsam3_point_segmenter("efficientvit", "b1", image_size=448)
    seg.load_state_dict({k: v for k, v in fill_state_dict(seg.state_dict(), 43).items() if not v.is_complex()}, strict=False)
    return seg.to(cuda)


def predictor_calls(seg, monkeypatch):
    """The es3_* calls of SAM3InteractiveImagePredictor over `seg` (points, box, box + points, point + mask, mask only, 12 points;
    multimask and return_logits on and off) and of seg.predict_batch (object-gated, 11 points), after set_image."""
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor
    pred = SAM3InteractiveImagePredictor(seg, max_hole_area=64.0, max_sprinkle_area=16.0)
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, size=(300, 420, 3), dtype=np.uint8)
    pred.set_image(img)
    pts = np.stack([rng.uniform(0, 420, 12), rng.uniform(0, 300, 12)], 1)
    lab = rng.integers(0, 2, 12)
    box = np.array([40.0, 30.0, 380.0, 260.0])
    low = pred.predict(point_coords=pts[:1], point_labels=lab[:1], multimask_output=False)[2]
    prompts = [dict(point_coords=pts[:3], point_labels=lab[:3]), dict(box=box), dict(box=box, point_coords=pts[:2], point_labels=lab[:2]),
               dict(point_coords=pts[:1], point_labels=lab[:1], mask_input=low), dict(mask_input=low),
               dict(point_coords=pts, point_labels=lab)]

    def run():
        for kw in prompts:
            for mm in (True, False):
                for logits in (True, False):
                    pred.predict(multimask_output=mm, return_logits=logits, **kw)
        S = seg.image_size
        dev = next(seg.parameters()).device
        seg.set_image_batch(torch.randn(2, 3, S, S, generator=torch.Generator().manual_seed(1)).to(dev))
        c = torch.rand(2, 11, 2, generator=torch.Generator().manual_seed(2)) * S
        lb = torch.ones(2, 11, dtype=torch.int32)
        for mm in (True, False):
            for logits in (True, False):
                seg.predict_batch(c.to(dev), lb.to(dev), multimask_output=mm, return_logits=logits)
    return record_calls(monkeypatch, run)


def sam_heads(E, S, sd_pe, sd_md, dev):
    """PromptEncoder and MaskDecoder (two-way transformer, high-res features, object scores) with state dicts sd_pe / sd_md, eval."""
    from efficientsam3_b200.sam import MaskDecoder, PromptEncoder, TwoWayTransformer
    pe = PromptEncoder(embed_dim=256, image_embedding_size=(E, E), input_image_size=(S, S), mask_in_chans=16)
    md = MaskDecoder(num_multimask_outputs=3, transformer=TwoWayTransformer(depth=2, embedding_dim=256, mlp_dim=2048, num_heads=8),
                     transformer_dim=256, iou_head_depth=3, iou_head_hidden_dim=256, use_high_res_features=True,
                     iou_prediction_use_sigmoid=True, pred_obj_scores=True, pred_obj_scores_mlp=True,
                     use_multimask_token_for_obj_ptr=True)
    pe.load_state_dict(sd_pe)
    md.load_state_dict(sd_md)
    return pe.to(dev).eval(), md.to(dev).eval()


def module_api_calls(cuda, monkeypatch):
    """The es3_* calls of the SAM heads' module API (sam_heads on the sam_heads_16 fixture's keys): points, boxes and a mask prompt,
    multimask on and off."""
    from helpers import load_golden, sd_from_keys
    g = load_golden("sam_heads_16")
    E, S, B = 16, 224, 2
    pe, md = sam_heads(E, S, sd_from_keys(g["keys_pe"], 5), sd_from_keys(g["keys_md"], 6), cuda)
    gen = torch.Generator().manual_seed(4)
    feat = torch.randn(B, 256, E, E, generator=gen).to(cuda)
    hr = [torch.randn(B, 32, 4 * E, 4 * E, generator=gen).to(cuda), torch.randn(B, 64, 2 * E, 2 * E, generator=gen).to(cuda)]
    coords = (torch.rand(B, 3, 2, generator=gen) * S).to(cuda)
    labels = torch.ones(B, 3, dtype=torch.int32, device=cuda)
    boxes = torch.tensor([[10.0, 20.0, 100.0, 200.0]] * B, device=cuda)
    masks = torch.randn(B, 1, 4 * E, 4 * E, generator=gen).to(cuda)

    def run():
        for kw in (dict(points=(coords, labels), boxes=None, masks=None), dict(points=None, boxes=boxes, masks=masks),
                   dict(points=(coords, labels), boxes=boxes, masks=None)):
            sp, de = pe(**kw)
            for mm in (True, False):
                md(image_embeddings=feat, image_pe=pe.get_dense_pe(), sparse_prompt_embeddings=sp, dense_prompt_embeddings=de,
                   multimask_output=mm, repeat_image=False, high_res_features=hr)
    return record_calls(monkeypatch, run)


def teacher_calls(cuda, monkeypatch, strict, fp8=None):
    """The es3_* calls of SAM3ImageTeacherEncoder at 1008 px (one windowed and one global block, B = 2), in the strict mode or not;
    fp8 = "linear" or "attention": with enable_fp8(True, attention=fp8 == "attention"), the weights packed inside the recorded
    forward."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.model import SAM3ImageTeacherEncoder
    t = SAM3ImageTeacherEncoder(embed_size=72, vit_overrides=dict(depth=2, global_att_blocks=(1,))).to(cuda)
    if fp8 is not None:
        t.enable_fp8(True, attention=fp8 == "attention")
    x = torch.randn(2, 3, 1008, 1008, device=cuda, generator=torch.Generator(device=cuda).manual_seed(0))

    def run():
        with torch.no_grad():
            if strict:
                with ops.strict_precision():
                    t(x)
            else:
                t(x)
    return record_calls(monkeypatch, run)


def backbone_calls(cuda, monkeypatch, which):
    """The es3_* calls of create_sam3_vit_backbone's eval forward (B = 2) with tests/test_vit_gpu.py's 336 configuration or the
    vit_small_112 fixture's."""
    from efficientsam3_b200.model.vitdet import create_sam3_vit_backbone
    from helpers import load_golden
    cfg = (dict(img_size=336, pretrain_img_size=112, patch_size=14, embed_dim=256, depth=4, num_heads=4, mlp_ratio=4.625,
                window_size=8, global_att_blocks=(1, 3)) if which == "336" else eval(str(load_golden("vit_small_112")["cfg"])))
    m = create_sam3_vit_backbone(**cfg).to(cuda).eval()
    x = torch.randn(2, 3, cfg["img_size"], cfg["img_size"], device=cuda, generator=torch.Generator(device=cuda).manual_seed(1))

    def run():
        with torch.no_grad():
            m(x)
    return record_calls(monkeypatch, run)


def segmenter_set_image_calls(cuda, monkeypatch):
    """The es3_* calls of the interactive predictor's set_image over Sam3PointPromptSegmenter (one windowed block), 600 x 800."""
    from efficientsam3_b200.model.sam1_task import SAM3InteractiveImagePredictor, Sam3PointPromptSegmenter
    seg = Sam3PointPromptSegmenter(vit_overrides=dict(depth=1, global_att_blocks=())).to(cuda).eval()
    pred = SAM3InteractiveImagePredictor(seg)
    img = np.random.default_rng(4).integers(0, 256, (600, 800, 3), dtype=np.uint8)
    return record_calls(monkeypatch, lambda: pred.set_image(img))
