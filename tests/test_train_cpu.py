"""CPU: the host side of the student backward.  The training graph of efficientsam3_b200 (what each unit saves, how
gradients are chained through residual joins, every weight re-layout and stride) runs with the libes3 ops swapped for
their torch statements (tests/emu_ops.py) and is compared with torch.autograd of the train-mode oracle.  The CUDA kernels
themselves are compared with the same statements in tests/test_train_gpu.py."""
from types import SimpleNamespace as NS

import pytest
import torch

import emu_ops
from oracle import efficientvit as O
from oracle.kd_loss import kd_loss as oracle_kd_loss
from oracle.weights import fill_state_dict


def _student(name="efficientvit_b1", img=160, embed=12, seed=3):
    from efficientsam3_b200.stage1.model import build_image_student_model
    cfg = NS(MODEL=NS(BACKBONE=name), DATA=NS(IMG_SIZE=img), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=embed))
    m = build_image_student_model(cfg)
    m.load_state_dict(fill_state_dict(m.state_dict(), seed))
    return m


def _oracle_step(sd0, x, teacher, img, sizes, variant, embed, bn_train=True):
    sd = {k: (v.clone().requires_grad_(True) if (v.is_floating_point() and "running" not in k) else v.clone()) for k, v in sd0.items()}
    if bn_train:
        with O.bn_batch_stats():
            out = O.image_student_encoder(sd, x, embed, variant)
    else:
        out = O.image_student_encoder(sd, x, embed, variant)
    loss, _, _ = oracle_kd_loss(out, teacher, img, sizes, 1.0)
    loss.backward()
    return out.detach(), loss.detach(), sd


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def _round_like_product(sd, dw5_fp32=False):
    """The weights the product packs to bf16 (every dense contraction operand: 1x1 / dense 3x3 convs and the LiteMLA
    aggregation taps); depthwise 3x3 taps, the stem conv, biases and BN vectors stay fp32.  dw5_fp32: the dim-32 LiteMLA route
    (efficientvit_b2) keeps the 5x5 aggregation taps in fp32 (es3_dwconv), only the grouped 1x1 is a bf16 GEMM operand."""
    out = {}
    for k, v in sd.items():
        dense = v.dim() == 4 and k.endswith(".weight") and (v.shape[1] > 1 or ".aggreg." in k) and "input_stem.op_list.0." not in k
        if dw5_fp32 and ".aggreg.0.0." in k:
            dense = False
        out[k] = v.to(torch.bfloat16).float() if dense else v.clone()
    return out


# exact=True : the emulation computes and stores in fp64 and the oracle runs in fp64 at the same bf16-rounded weights ->
#              only the fp32 parameter-gradient accumulators are left, so ANY mistake in the graph logic (saved tensors,
#              chaining, layouts, strides, BN algebra) shows.  (fp64 because the fp32 oracle itself is 2.5e-3 away from
#              the fp64 one on this configuration.)
# exact=False: activations / activation gradients rounded to bf16 wherever the kernels store them -> the error the real
#              path carries.  Random-weight batch-statistics BN at this size is ill-conditioned (rounding only the oracle's
#              weights to bf16 already moves its stage-4 output by 13 %), so the batch-BN case is held to loose bounds and
#              the frozen-BN case (well conditioned) to tight ones.
@pytest.mark.parametrize("bn_train,exact", [(True, True), (False, True), (True, False), (False, False)])
def test_train_graph_matches_oracle_autograd(monkeypatch, bn_train, exact):
    emu_ops.install(monkeypatch)
    if exact:
        from efficientsam3_b200 import ops
        monkeypatch.setattr(emu_ops, "BF", torch.float64)
        monkeypatch.setattr(emu_ops, "CD", torch.float64)
        monkeypatch.setattr(ops, "ACT_DTYPE", torch.float64)
    torch.manual_seed(0)
    img, embed, B = 160, 12, 2
    m = _student(img=img, embed=embed)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    sd_ref = _round_like_product(sd0) if exact else sd0
    tol_out, tol_each, tol_all, tol_run = ((1e-5, 1e-4, 1e-5, 1e-5) if exact else
                                           ((0.5, 1e9, 1e9, 0.2) if bn_train else (2e-2, 0.12, 3e-2, 1e-6)))
    x = torch.randn(B, 3, img, img, generator=torch.Generator().manual_seed(1))
    teacher = torch.randn(B, 1024, embed, embed, generator=torch.Generator().manual_seed(2))
    sizes = [(3, img, img * 3 // 4), (3, img * 2 // 3, img)]
    m.train()
    if not bn_train:   # set_bn_state(EVAL_BN_WHEN_TRAINING): BN modules in eval inside a training model
        for mod in m.modules():
            if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
                mod.eval()
    out = m(x)
    assert out.requires_grad and out.shape == (B, 1024, embed, embed) and out.dtype == (torch.float64 if exact else torch.float32)
    loss, _, _ = oracle_kd_loss(out, teacher.to(out.dtype), img, sizes, 1.0)
    loss.backward()

    if exact:
        sd_ref = {k: (v.double() if v.is_floating_point() else v) for k, v in sd_ref.items()}
        ref_out, ref_loss, sd = _oracle_step(sd_ref, x.double(), teacher.double(), img, sizes, "b1", embed, bn_train)
    else:
        ref_out, ref_loss, sd = _oracle_step(sd_ref, x, teacher, img, sizes, "b1", embed, bn_train)
    gscale = max(v.grad.norm().item() for k, v in sd.items() if v.is_floating_point() and v.grad is not None)
    assert _rel(out.detach(), ref_out) < tol_out, _rel(out.detach(), ref_out)
    assert abs(loss.item() - ref_loss.item()) < tol_out * abs(ref_loss.item())
    worst, missing = 0.0, []
    tot_num = tot_den = 0.0
    for name, p in m.named_parameters():
        g_ref = sd[name].grad
        if p.grad is None:
            missing.append(name)
            continue
        assert p.grad.shape == p.shape and p.grad.dtype == torch.float32
        tot_num += (p.grad.double() - g_ref.double()).pow(2).sum().item()
        tot_den += g_ref.double().pow(2).sum().item()
        # gradients that are analytically zero (a bias in front of a batch-statistics BN) are held to an absolute bound
        err = (p.grad.double() - g_ref.double()).norm().item()
        r = err / max(g_ref.double().norm().item(), 1e-3 * gscale)
        assert r < tol_each, (name, r)
        worst = max(worst, r)
    assert not missing, missing
    assert (tot_num / tot_den) ** 0.5 < tol_all, (tot_num / tot_den) ** 0.5
    print(f"bn_train={bn_train} exact={exact}: out {_rel(out.detach(), ref_out):.2e}, worst grad {worst:.2e}, "
          f"all grads {(tot_num / tot_den) ** 0.5:.2e}")
    # running statistics: updated in train mode exactly as nn.BatchNorm2d does, untouched when frozen
    for k, v in m.state_dict().items():
        if "running_" in k:
            assert _rel(v, sd[k]) < tol_run, (k, _rel(v, sd[k]))
            if not bn_train:
                assert torch.equal(v, sd0[k]), k
        if "num_batches_tracked" in k:
            assert int(v) == int(sd0[k]) + (1 if bn_train else 0), k


def test_eval_plan_is_rebuilt_after_a_train_forward(monkeypatch):
    """Parameters / running stats move through raw pointers during training: the cached eval-mode packing must not survive."""
    emu_ops.install(monkeypatch)
    m = _student(img=160, embed=12)
    m.eval()
    m._plan_key = ("stale",)
    m.backbone.model._plan_key = ("stale",)
    m.train()
    m(torch.randn(1, 3, 160, 160))
    assert m._plan_key is None and m.backbone.model._plan_key is None


def test_train_mode_has_no_cpu_fallback():
    """All nine students have a training graph now; without the device ops (CPU tensors) train mode raises like eval mode does."""
    from efficientsam3_b200 import _lib
    from efficientsam3_b200.stage1.model import build_image_student_model
    for name in ("efficientvit_b1", "repvit_m1_1", "tiny_vit_11m"):
        cfg = NS(MODEL=NS(BACKBONE=name), DATA=NS(IMG_SIZE=160), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=12))
        m = build_image_student_model(cfg).train()
        with pytest.raises(_lib.Es3Error):
            m(torch.randn(1, 3, 160, 160))


@pytest.mark.parametrize("B,H,W,N,C", [(2, 5, 7, 32, 16), (1, 8, 8, 64, 24), (3, 4, 14, 16, 8)])
def test_conv3x3_wgrad_composition(monkeypatch, B, H, W, N, C):
    """ops.conv3x3_wgrad = zero-framed transposes + nine GEMMs over the pixel index + strided accumulation: the composition
    (frame geometry, tap offsets, strides) against autograd, with the three primitives emulated."""
    from efficientsam3_b200 import ops
    emu_ops.install(monkeypatch)
    g = torch.Generator().manual_seed(B + H + N)
    dy = torch.randn(B, H, W, N, generator=g).to(torch.bfloat16)
    a = torch.randn(B, H, W, C, generator=g).to(torch.bfloat16)
    ref = torch.full((N, C, 3, 3), 0.5)
    emu_ops.conv3x3_wgrad(dy, a, ref)
    got = torch.full((N, C, 3, 3), 0.5)
    ops.conv3x3_wgrad(dy, a, got)
    assert (got - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()


# ------------------------------------------------------------------------------------------------- RepViT (config 4)
def _round_like_product_repvit(sd):
    """bf16 in the product: every 1x1 Conv2d_BN weight, the second patch-embed conv, the head convs.  fp32: the stem conv,
    depthwise taps (3x3 and the RepVGGDW 1x1), SqueezeExcite (es3_gemm_simt on fp32), BN vectors."""
    out = {}
    for k, v in sd.items():
        dense = (v.dim() == 4 and v.shape[1] > 1 and (k.endswith(".c.weight") or k in ("head.0.weight", "head.3.weight"))
                 and not k.endswith("features.0.0.c.weight"))
        out[k] = v.to(torch.bfloat16).float() if dense else v.clone()
    return out


def _oracle_step_repvit(sd0, x, teacher, img, sizes, embed, bn_train, variant="repvit_m1_1"):
    from oracle import repvit as R
    sd = {k: (v.clone().requires_grad_(True) if (v.is_floating_point() and "running" not in k) else v.clone()) for k, v in sd0.items()}
    if bn_train:
        with O.bn_batch_stats():
            out = R.image_student_encoder(sd, x, embed, variant)
    else:
        out = R.image_student_encoder(sd, x, embed, variant)
    loss, _, _ = oracle_kd_loss(out, teacher, img, sizes, 1.0)
    loss.backward()
    return out.detach(), loss.detach(), sd


@pytest.mark.parametrize("name", ["repvit_m0_9", "repvit_m2_3"])
def test_repvit_padded_patch_embed_exact(monkeypatch, name):
    """repvit_m0_9: the 24-channel first conv is zero-padded to the 32 channels the stride-2 kernel is instantiated for; repvit_m2_3: the
    40-channel first conv + BN run zero-padded to 48 end to end (PaddedStemUnit).  The padding must not leak into any gradient or
    running statistic (fp64 emulation vs oracle autograd)."""
    from efficientsam3_b200 import ops
    emu_ops.install(monkeypatch)
    monkeypatch.setattr(emu_ops, "BF", torch.float64)
    monkeypatch.setattr(emu_ops, "CD", torch.float64)
    monkeypatch.setattr(ops, "ACT_DTYPE", torch.float64)
    img, embed, B = 128, 8, 2
    m = _student(name, img=img, embed=embed, seed=13)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(B, 3, img, img, generator=torch.Generator().manual_seed(1))
    teacher = torch.randn(B, 1024, embed, embed, generator=torch.Generator().manual_seed(2)).double()
    sizes = [(3, img, img)] * B
    m.train()
    out = m(x)
    loss, _, _ = oracle_kd_loss(out, teacher, img, sizes, 1.0)
    loss.backward()
    sd_ref = {k: (v.double() if v.is_floating_point() else v) for k, v in _round_like_product_repvit(sd0).items()}
    ref_out, _, sd = _oracle_step_repvit(sd_ref, x.double(), teacher, img, sizes, embed, True, name)
    assert _rel(out.detach(), ref_out) < 1e-5
    for k, v in m.state_dict().items():
        if "running_" in k:
            assert v.shape == sd[k].shape and _rel(v, sd[k]) < 1e-5, k
    num = den = 0.0
    for k, p in m.named_parameters():
        g = sd[k].grad.double()
        assert p.grad.shape == p.shape
        num += (p.grad.double() - g).pow(2).sum().item()
        den += g.pow(2).sum().item()
    assert (num / den) ** 0.5 < 2e-5, (num / den) ** 0.5


@pytest.mark.parametrize("bn_train,exact", [(True, True), (False, True), (False, False)])
def test_repvit_train_graph_matches_oracle_autograd(monkeypatch, bn_train, exact):
    """RepViT-M1.1 training graph (un-fused RepVGGDW with batch-statistics BN, SqueezeExcite, stride-2 patch-embed conv through
    the 2x2 phase decomposition) vs autograd of the oracle; exact = fp64 emulation (logic check), else bf16 storage (frozen BN)."""
    from efficientsam3_b200 import ops
    emu_ops.install(monkeypatch)
    if exact:
        monkeypatch.setattr(emu_ops, "BF", torch.float64)
        monkeypatch.setattr(emu_ops, "CD", torch.float64)
        monkeypatch.setattr(ops, "ACT_DTYPE", torch.float64)
    img, embed, B = 128, 8, 2
    m = _student("repvit_m1_1", img=img, embed=embed, seed=11)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(B, 3, img, img, generator=torch.Generator().manual_seed(1))
    teacher = torch.randn(B, 1024, embed, embed, generator=torch.Generator().manual_seed(2))
    sizes = [(3, img, img * 3 // 4), (3, img * 2 // 3, img)]
    m.train()
    if not bn_train:
        for mod in m.modules():
            if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
                mod.eval()
    out = m(x)
    loss, _, _ = oracle_kd_loss(out, teacher.to(out.dtype), img, sizes, 1.0)
    loss.backward()
    if exact:
        sd_ref = {k: (v.double() if v.is_floating_point() else v) for k, v in _round_like_product_repvit(sd0).items()}
        ref_out, ref_loss, sd = _oracle_step_repvit(sd_ref, x.double(), teacher.double(), img, sizes, embed, bn_train)
        tol_out, tol_each, tol_all = 1e-5, 2e-4, 2e-5
    else:
        ref_out, ref_loss, sd = _oracle_step_repvit(sd0, x, teacher, img, sizes, embed, bn_train)
        tol_out, tol_each, tol_all = 3e-2, 0.3, 6e-2
    assert _rel(out.detach(), ref_out) < tol_out, _rel(out.detach(), ref_out)
    gscale = max(v.grad.norm().item() for v in sd.values() if v.is_floating_point() and v.grad is not None)
    num = den = worst = 0.0
    for name, p in m.named_parameters():
        assert p.grad is not None, name
        g_ref = sd[name].grad.double()
        err = (p.grad.double() - g_ref).norm().item()
        num += err ** 2
        den += g_ref.pow(2).sum().item()
        r = err / max(g_ref.norm().item(), 1e-3 * gscale)
        assert r < tol_each, (name, r)
        worst = max(worst, r)
    print(f"repvit bn_train={bn_train} exact={exact}: out {_rel(out.detach(), ref_out):.2e}, worst grad {worst:.2e}, all grads {(num / den) ** 0.5:.2e}")
    assert (num / den) ** 0.5 < tol_all
    for k, v in m.state_dict().items():
        if "num_batches_tracked" in k:
            assert int(v) == int(sd0[k]) + (1 if bn_train else 0), k


def test_train_one_epoch_follows_the_reference_loop(monkeypatch):
    """stage1.train.train_one_epoch with the reference's loader contract: gradient accumulation (loss / ACCUMULATION_STEPS, update
    and zero_grad every ACCUMULATION_STEPS iterations), per-update LR from the cosine schedule, frozen BN through set_bn_state.
    The device ops are emulated; the optimiser update (a CUDA kernel) is replaced by a recorder that applies plain SGD."""
    import numpy as np
    from efficientsam3_b200.stage1 import optim as OPT
    from efficientsam3_b200.stage1.train import train_one_epoch
    emu_ops.install(monkeypatch)
    img, embed, B, iters, accum = 160, 12, 1, 4, 2

    # KD loss ops on CPU: the oracle's loss through autograd stands in for es3_kd_loss_fwd / _bwd
    from efficientsam3_b200 import ops

    def kd_fwd(preds, teacher, sizes, img_size, w):
        szl = [(3, int(a), int(b)) for a, b in sizes.tolist()]
        loss, mse, cos = oracle_kd_loss(preds.float(), teacher, img_size, szl, w)
        return torch.stack([loss, mse, cos]).detach(), None

    def kd_bwd(preds, teacher, sizes, per, img_size, w, grad_scale=1.0, scale_dev=None):
        szl = [(3, int(a), int(b)) for a, b in sizes.tolist()]
        p = preds.detach().float().requires_grad_(True)
        with torch.enable_grad():
            loss, _, _ = oracle_kd_loss(p, teacher, img_size, szl, w)
            (g,) = torch.autograd.grad(loss, p)
        return g * grad_scale * (scale_dev[0] if scale_dev is not None else 1.0)

    monkeypatch.setattr(ops, "kd_loss_fwd", kd_fwd)
    monkeypatch.setattr(ops, "kd_loss_bwd", kd_bwd)
    calls = []

    def fake_step(self, lr=None, max_norm=5.0, world_size=1):
        if lr is not None:
            self.lr = lr                       # the real step() bookkeeping: the schedule must not be built from this value
        calls.append((lr, max_norm, world_size, float(self.flat_grad.norm())))
        self.flat_param -= 1e-6 * self.flat_grad

    monkeypatch.setattr(OPT.FlatAdamW, "step", fake_step)
    cfg = NS(TRAIN=NS(EVAL_BN_WHEN_TRAINING=True, ACCUMULATION_STEPS=accum, EPOCHS=3, WARMUP_EPOCHS=1, MIN_LR=1e-6, WARMUP_LR=1e-7,
                      CLIP_GRAD=5.0),
             DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=embed, COSINE=1.0), DATA=NS(IMG_SIZE=img))
    m = _student("efficientvit_b0", img=img, embed=embed)
    opt = OPT.FlatAdamW(m, lr=1e-3, weight_decay=0.01)
    g = torch.Generator().manual_seed(3)
    loader = [(([torch.randn(3, img, img, generator=g) for _ in range(B)], {"img_size_before_pad": [(3, img, img)] * B}),
               ([np.random.RandomState(i).randn(1024 * embed * embed).astype(np.float16) for _ in range(B)], [i] * B)) for i in range(iters)]
    losses = train_one_epoch(cfg, m, loader, opt, epoch=0) + train_one_epoch(cfg, m, loader, opt, epoch=1)
    assert len(losses) == 2 * iters and all(torch.isfinite(v) for v in losses)
    assert len(calls) == 2 * iters // accum                              # one update per ACCUMULATION_STEPS iterations
    n_iter = iters // accum
    # the reference's order (train_image_encoder_stage1.py:216-229): optimizer.step() with the LR currently in the optimiser, THEN
    # lr_scheduler.step_update(arg); the scheduler's constructor leaves lr_at(0) (= WARMUP_LR when there is a warm-up) behind
    sched = lambda t: OPT.cosine_lr(t, 1e-3, 3 * n_iter, 1e-6, 1 * n_iter, 1e-7)
    cur, expect = sched(0), []
    for epoch in (0, 1):
        for idx in range(iters):
            if (idx + 1) % accum == 0:
                expect.append(cur)
                cur = sched((epoch * iters + idx) // accum)
    assert [c[0] for c in calls] == expect and all(c[1] == 5.0 and c[2] == 1 for c in calls)
    assert opt.base_lr == 1e-3 and opt.lr == expect[-1]
    assert opt.flat_grad.abs().sum().item() == 0                         # cleared right after the last update
    assert all(not mod.training for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d)) and m.training
    assert all(c[3] > 0 for c in calls)


def test_smoke_training_half_runs_under_emulation(monkeypatch, capsys):
    """__graft_entry__.smoke()'s training half (wiring, thresholds) with the device ops emulated on CPU."""
    import sys
    import os
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import __graft_entry__ as G
    from efficientsam3_b200 import ops
    emu_ops.install(monkeypatch)

    def kd_fwd(preds, teacher, sizes, img_size, w):
        szl = [(3, int(a), int(b)) for a, b in sizes.tolist()]
        loss, mse, cos = oracle_kd_loss(preds.float(), teacher, img_size, szl, w)
        return torch.stack([loss, mse, cos]).detach(), None

    def kd_bwd(preds, teacher, sizes, per, img_size, w, grad_scale=1.0, scale_dev=None):
        szl = [(3, int(a), int(b)) for a, b in sizes.tolist()]
        p = preds.detach().float().requires_grad_(True)
        with torch.enable_grad():
            loss, _, _ = oracle_kd_loss(p, teacher, img_size, szl, w)
            (g,) = torch.autograd.grad(loss, p)
        return g * grad_scale * (scale_dev[0] if scale_dev is not None else 1.0)

    monkeypatch.setattr(ops, "kd_loss_fwd", kd_fwd)
    monkeypatch.setattr(ops, "kd_loss_bwd", kd_bwd)
    img, embed = 192, 9
    m = _student("efficientvit_b1", img=img, embed=embed, seed=3)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(2, 3, img, img, generator=torch.Generator().manual_seed(0))
    G._smoke_train_step(torch.device("cpu"), m, sd, x, img, embed)
    assert "training step" in capsys.readouterr().out and not m.training


@pytest.mark.parametrize("name,variant,img,embed", [("efficientvit_b0", "b0", 160, 12), ("efficientvit_b1", "b1", 224, 9),
                                                    ("efficientvit_b2", "b2", 192, 9)])
def test_other_sizes_exact(monkeypatch, name, variant, img, embed):
    """The fp64 logic check on the second EfficientViT name with a training graph (b0: 8-channel stem, 2-block stages) and on an
    odd-sized map chain (224 -> 112 / 56 / 28 / 14 / 7: stride-2 layers over odd extents, head resize 7 -> 9)."""
    from efficientsam3_b200 import ops
    emu_ops.install(monkeypatch)
    monkeypatch.setattr(emu_ops, "BF", torch.float64)
    monkeypatch.setattr(emu_ops, "CD", torch.float64)
    monkeypatch.setattr(ops, "ACT_DTYPE", torch.float64)
    B = 2
    m = _student(name, img=img, embed=embed, seed=9)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(B, 3, img, img, generator=torch.Generator().manual_seed(4))
    teacher = torch.randn(B, 1024, embed, embed, generator=torch.Generator().manual_seed(5)).double()
    sizes = [(3, img, img * 3 // 4), (3, img * 2 // 3, img)]
    m.train()
    out = m(x)
    loss, _, _ = oracle_kd_loss(out, teacher, img, sizes, 1.0)
    loss.backward()
    sd_ref = {k: (v.double() if v.is_floating_point() else v) for k, v in _round_like_product(sd0, dw5_fp32=(variant == "b2")).items()}
    ref_out, _, sd = _oracle_step(sd_ref, x.double(), teacher, img, sizes, variant, embed, True)
    assert _rel(out.detach(), ref_out) < 1e-5
    num = den = 0.0
    for k, p in m.named_parameters():
        g = sd[k].grad.double()
        num += (p.grad.double() - g).pow(2).sum().item()
        den += g.pow(2).sum().item()
    assert (num / den) ** 0.5 < 1e-5, (num / den) ** 0.5


# ------------------------------------------------------------------------------------------------- TinyViT
def _round_like_product_tinyvit(sd):
    """bf16 in the product: every 1x1 Conv2d_BN weight, the second patch-embed conv, every nn.Linear weight, the head convs."""
    out = {}
    for k, v in sd.items():
        conv = (v.dim() == 4 and v.shape[1] > 1 and (k.endswith(".c.weight") or k in ("head.0.weight", "head.3.weight"))
                and not k.endswith("patch_embed.seq.0.c.weight"))
        lin = v.dim() == 2 and k.endswith(".weight") and (".qkv." in k or ".proj." in k or ".fc1." in k or ".fc2." in k)
        out[k] = v.to(torch.bfloat16).float() if (conv or lin) else v.clone()
    return out


@pytest.mark.parametrize("name,bn_train", [("tiny_vit_5m", True), ("tiny_vit_11m", False), ("tiny_vit_21m", True)])
def test_tinyvit_train_graph_exact(monkeypatch, name, bn_train):
    """TinyViT training graph (MBConv with the post-add GELU, PatchMerging, window attention with relative bias on maps padded to a
    window multiple -- 20 -> 21, 10 -> 14, 5 -> 7 at 160 px --, LayerNorm, GELU MLPs; DropPath rates set to 0) in fp64 emulation
    vs autograd of the oracle."""
    from efficientsam3_b200 import ops
    from oracle import tinyvit as TV
    emu_ops.install(monkeypatch)
    monkeypatch.setattr(emu_ops, "BF", torch.float64)
    monkeypatch.setattr(emu_ops, "CD", torch.float64)
    monkeypatch.setattr(ops, "ACT_DTYPE", torch.float64)
    img, embed, B = 160, 12, 2
    m = _student(name, img=img, embed=embed, seed=17)
    for mod in m.modules():
        if hasattr(mod, "drop_path_rate"):
            mod.drop_path_rate = 0.0
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(B, 3, img, img, generator=torch.Generator().manual_seed(1))
    teacher = torch.randn(B, 1024, embed, embed, generator=torch.Generator().manual_seed(2)).double()
    sizes = [(3, img, img)] * B
    m.train()
    if not bn_train:
        for mod in m.modules():
            if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
                mod.eval()
    out = m(x)
    loss, _, _ = oracle_kd_loss(out, teacher, img, sizes, 1.0)
    loss.backward()
    sd = {k: ((v.double().requires_grad_(True) if "running" not in k else v.double()) if v.is_floating_point() else v.clone())
          for k, v in _round_like_product_tinyvit(sd0).items()}
    if bn_train:
        with O.bn_batch_stats():
            ref_out = TV.image_student_encoder(sd, x.double(), embed, name)
    else:
        ref_out = TV.image_student_encoder(sd, x.double(), embed, name)
    rl, _, _ = oracle_kd_loss(ref_out, teacher, img, sizes, 1.0)
    rl.backward()
    assert _rel(out.detach(), ref_out.detach()) < 1e-5, _rel(out.detach(), ref_out.detach())
    gscale = max(v.grad.norm().item() for v in sd.values() if v.is_floating_point() and v.grad is not None)
    num = den = 0.0
    for k, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape, k
        g = sd[k].grad.double()
        err = (p.grad.double() - g).norm().item()
        assert err / max(g.norm().item(), 1e-3 * gscale) < 2e-4, (k, err / max(g.norm().item(), 1e-3 * gscale))
        num += err ** 2
        den += g.pow(2).sum().item()
    print(f"{name} bn_train={bn_train}: out {_rel(out.detach(), ref_out.detach()):.2e}, all grads {(num / den) ** 0.5:.2e}")
    assert (num / den) ** 0.5 < 2e-5


def test_drop_path_gate(monkeypatch):
    """timm DropPath in the TinyViT training graph: one Bernoulli(keep) draw per sample scaled by 1 / keep, the same gate in the backward,
    identity for rate 0 -- and the 11m builder keeps the reference's per-block rates (linspace(0, 0.1, 12))."""
    from efficientsam3_b200.backbones.tinyvit_train import DropPath
    from efficientsam3_b200.backbones.tiny_vit import tiny_vit_11m_224
    emu_ops.install(monkeypatch)
    torch.manual_seed(0)
    x = torch.randn(64, 3, 5, 16).to(torch.bfloat16)
    dp = DropPath(0.25)
    y = dp.forward(x)
    g = dp.gate[:, 0]
    assert all(v == 0.0 or abs(v - 1.0 / 0.75) < 1e-6 for v in g.tolist()) and 0 < (g == 0).sum().item() < 64
    assert torch.equal(y, (x.float() * g.view(-1, 1, 1, 1)).to(torch.bfloat16))
    d = torch.randn_like(x)
    assert torch.equal(dp.backward(d), (d.float() * g.view(-1, 1, 1, 1)).to(torch.bfloat16))
    assert DropPath(0.0).forward(x) is x
    m = tiny_vit_11m_224(img_size=224, num_classes=0)
    rates = [blk.drop_path_rate for layer in m.layers for blk in layer.blocks]
    assert len(rates) == 12 and rates[0] == 0.0 and abs(rates[-1] - 0.1) < 1e-7 and all(a <= b for a, b in zip(rates, rates[1:]))
