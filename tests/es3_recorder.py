"""Records the es3_* calls a piece of native work makes (the route-closure tests of tests/test_train_bwd_gpu.py,
tests/test_fwd_kernels_gpu.py and tests/test_text_kernels_gpu.py): every _lib.call, and every _lib.call_rc that ran (rc == 0; a
declined shape returns -1)."""
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


def eval_forward_calls(cuda, monkeypatch, name, img=1024, embed=64, B=2):
    """The es3_* calls of one eval forward of `name`."""
    m = student(cuda, name, img, embed).eval()
    x = torch.randn(B, 3, img, img, device=cuda, generator=torch.Generator(device=cuda).manual_seed(0))

    def run():
        with torch.no_grad():
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
