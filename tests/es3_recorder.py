"""Records the es3_* calls a piece of native work makes (the route-closure tests of tests/test_train_bwd_gpu.py and
tests/test_fwd_kernels_gpu.py): every _lib.call, and every _lib.call_rc that ran (rc == 0; a declined shape returns -1)."""
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
