"""GPU: the student-backward kernels (efficientsam3_b200/csrc/train_bwd.cu) against their torch statements in
tests/emu_ops.py (which the CPU suite ties to autograd of the train-mode oracle), then whole training steps.

Tolerances: bf16 outputs 1e-2 of the tensor's scale (bf16 step 2^-8); fp32 reductions (statistics, parameter
gradients) 2e-3 of the tensor's scale (bf16 products, fp32 accumulation in a different order).  Whole-step parity of
parameter gradients: frozen-BN mode (well conditioned) rel-L2 <= 5e-2 over all gradients; batch-statistics mode on the
random-weight fixture is ill-conditioned (the fp32 oracle itself is 2.5e-3 from the fp64 one, bf16 storage of the
activations alone moves the gradients by ~12 %; tests/test_train_cpu.py) and is held to a loose bound, next to a
functional check: a few optimiser steps reduce the loss.

(The file name sorts last on purpose: it is the newest code of the round.)"""
import math
import os
import subprocess
import sys
from types import SimpleNamespace as NS

import pytest
import torch

import emu_ops as E

pytestmark = pytest.mark.gpu


def _bf(t):
    return t.to(torch.bfloat16)


def _close(got, ref, tol, what=""):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = ref.abs().max().item() + 1e-20
    err = (got - ref).abs().max().item() / scale
    assert math.isfinite(err) and err <= tol, f"{what}: max err / scale = {err:.3e} > {tol}"


def _g(seed):
    return torch.Generator().manual_seed(seed)


# --------------------------------------------------------------------------------------------- BatchNorm pieces
@pytest.mark.parametrize("M,C", [(1000, 16), (4099, 24), (777, 64), (20000, 128), (3000, 1024), (131, 2560)])
def test_bn_stats(cuda, M, C):
    from efficientsam3_b200 import ops
    g = _g(M + C)
    z = _bf(torch.randn(M, C, generator=g) * (torch.rand(C, generator=g) + 0.2) + torch.randn(C, generator=g) * 2)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    rm, rv, nbt = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5, torch.tensor(7)
    rm_d, rv_d, nbt_d = rm.clone().to(cuda), rv.clone().to(cuda), nbt.clone().to(cuda)
    got = ops.bn_stats(z.to(cuda), gamma.to(cuda), beta.to(cuda), 1e-5, 0.1, rm_d, rv_d, nbt_d)
    ref = E.bn_stats(z, gamma, beta, 1e-5, 0.1, rm, rv, nbt)
    for a, b, name in zip(got, ref, ("mean", "invstd", "scale", "shift")):
        _close(a, b, 1e-4, f"bn_stats {name}")
    _close(rm_d, rm, 1e-5, "running_mean")
    _close(rv_d, rv, 1e-4, "running_var")
    assert int(nbt_d) == 8


@pytest.mark.parametrize("act", [None, "hswish", "gelu", "relu"])
@pytest.mark.parametrize("M,C,res", [(513, 16, True), (1000, 256, False), (77, 1024, True)])
def test_affine_act(cuda, M, C, res, act):
    from efficientsam3_b200 import ops
    g = _g(M * 3 + C)
    z = _bf(torch.randn(M, C, generator=g) * 2)
    scale, shift = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    r = _bf(torch.randn(M, C, generator=g)) if res else None
    got = ops.affine_act(z.to(cuda), scale.to(cuda), shift.to(cuda), act, r.to(cuda) if res else None)
    _close(got, E.affine_act(z, scale, shift, act, r), 1e-2, f"affine_act {act}")
    got = ops.affine_act(z.to(cuda), None, shift.to(cuda), act)        # bias-only layers (fewer_norm MBConv)
    _close(got, E.affine_act(z, None, shift, act), 1e-2, "affine_act bias-only")


@pytest.mark.parametrize("mode", ["none", "eval", "batch"])
@pytest.mark.parametrize("act", [None, "hswish", "gelu"])
@pytest.mark.parametrize("M,C", [(2000, 16), (1111, 64), (300, 512)])
def test_bn_act_bwd(cuda, M, C, act, mode):
    from efficientsam3_b200 import ops
    g = _g(M + 7 * C)
    z = _bf(torch.randn(M, C, generator=g) * (torch.rand(C, generator=g) + 0.3) + torch.randn(C, generator=g))
    da = _bf(torch.randn(M, C, generator=g))
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.5
    if mode == "none":
        scale, shift, mean, invstd = None, beta, None, None
    elif mode == "eval":
        mean, invstd = torch.randn(C, generator=g) * 0.5, torch.rsqrt(torch.rand(C, generator=g) + 0.5)
        scale = gamma * invstd
        shift = beta - mean * scale
    else:
        mean, invstd, scale, shift = E.bn_stats(z, gamma, beta, 1e-5, 0.1)
    dg_ref, db_ref = torch.full((C,), 0.25), torch.full((C,), -0.5)     # the kernels accumulate (+=)
    dz_ref = E.bn_act_bwd(da, z, scale, shift, act, mode, mean, invstd, dg_ref if mode != "none" else None, db_ref)
    dev = lambda t: None if t is None else t.to(cuda)
    dg, db = torch.full((C,), 0.25, device=cuda), torch.full((C,), -0.5, device=cuda)
    dz = ops.bn_act_bwd(dev(da), dev(z), dev(scale), dev(shift), act, mode, dev(mean), dev(invstd), dg if mode != "none" else None, db)
    _close(dz, dz_ref, 1e-2, f"dz {mode} {act}")
    _close(db, db_ref, 2e-3, f"dbeta {mode} {act}")
    if mode != "none":
        _close(dg, dg_ref, 2e-3, f"dgamma {mode} {act}")
    # reductions only (bias gradient of the head's 3x3 conv)
    db2 = torch.zeros(C, device=cuda)
    assert ops.bn_act_bwd(dev(da), dev(da), None, None, None, "none", dbeta=db2, apply=False) is None
    _close(db2, da.float().sum(0), 2e-3, "column sums")


def test_add_bf16_strided(cuda):
    from efficientsam3_b200 import ops
    g = _g(4)
    big = _bf(torch.randn(999, 768, generator=g))
    b = _bf(torch.randn(999, 384, generator=g))
    got = ops.add_bf16(big.to(cuda)[:, :384], b.to(cuda))
    _close(got, E.add_bf16(big[:, :384], b), 1e-2, "add strided")
    got = ops.add_bf16(big.to(cuda)[:, 384:], b.to(cuda))
    _close(got, E.add_bf16(big[:, 384:], b), 1e-2, "add strided 2")


# --------------------------------------------------------------------------------------------- weight gradients
@pytest.mark.parametrize("M,N,K", [(1000, 64, 16), (4103, 16, 16), (2560, 32, 128), (777, 128, 512), (5000, 384, 384),
                                   (300, 1024, 256), (256, 24, 96), (20000, 16, 64), (3000, 16, 32), (3001, 32, 16), (999, 32, 32), (5555, 64, 32)])
def test_wgrad_pw(cuda, M, N, K):
    from efficientsam3_b200 import ops
    g = _g(M + N + K)
    dz, x = _bf(torch.randn(M, N, generator=g)), _bf(torch.randn(M, K, generator=g))
    dW_ref = torch.full((N, K), 0.5)
    E.wgrad_pw(dz, x, dW_ref)
    dW = torch.full((N, K), 0.5, device=cuda)
    ops.wgrad_pw(dz.to(cuda), x.to(cuda), dW)
    _close(dW, dW_ref, 2e-3, f"wgrad_pw {M}x{N}x{K}")


@pytest.mark.parametrize("M,N,K,ldz,ldx", [(64, 64, 64, 64, 64), (5000, 128, 64, 128, 64), (4099, 256, 512, 256, 512), (20000, 1024, 256, 1024, 256),
                                           (3000, 64, 256, 200, 264), (777, 192, 320, 192, 320), (100000, 384, 128, 768, 128), (1500, 512, 1024, 512, 1024)])
def test_wgrad_tc(cuda, M, N, K, ldz, ldx):
    """The wgmma split-K weight-gradient kernel (both operands MN-major) against the fp32 statement, incl. strided operand views,
    ragged pixel counts, tiles wider than the matrix, accumulation into a pre-filled dW, and bit-reproducibility."""
    from efficientsam3_b200 import ops, _lib
    g = _g(M + N + K)
    dzb, xb = _bf(torch.randn(M, ldz, generator=g)), _bf(torch.randn(M, ldx, generator=g))
    dz, x = dzb[:, ldz - N:], xb[:, :K]
    ref = torch.full((N, K), 0.25)
    E.wgrad_pw(dz, x, ref)
    outs = []
    for _ in range(2):
        dW = torch.full((N, K), 0.25, device=cuda)
        dzd, xd = dzb.to(cuda)[:, ldz - N:], xb.to(cuda)[:, :K]
        ws = torch.empty(_lib.size("es3_wgrad_tc_ws_floats", M, N, K), device=cuda)
        rc = _lib.call_rc("es3_wgrad_tc", dzd.data_ptr(), dzd.stride(0), xd.data_ptr(), xd.stride(0), M, N, K, ws.data_ptr(), dW.data_ptr(), K,
                          torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        outs.append(dW)
    _close(outs[0], ref, 2e-3, f"wgrad_tc {M}x{N}x{K}")
    assert torch.equal(outs[0], outs[1])
    # and the same shapes through the public op (which routes here)
    dW = torch.full((N, K), 0.25, device=cuda)
    ops.wgrad_pw(dzb.to(cuda)[:, ldz - N:], xb.to(cuda)[:, :K], dW)
    assert torch.equal(dW, outs[0])


def test_wgrad_pw_strided_operands(cuda):
    """dz is a channel slice of the LiteMLA gradient buffer (row stride 2*c3)."""
    from efficientsam3_b200 import ops
    g = _g(11)
    M, c3 = 1500, 96
    big, x = _bf(torch.randn(M, 2 * c3, generator=g)), _bf(torch.randn(M, c3, generator=g))
    ref = torch.zeros(c3, c3)
    E.wgrad_pw(big[:, c3:], x, ref)
    got = torch.zeros(c3, c3, device=cuda)
    ops.wgrad_pw(big.to(cuda)[:, c3:], x.to(cuda), got)
    _close(got, ref, 2e-3, "wgrad_pw strided")


@pytest.mark.parametrize("B,H,W,N,C", [(2, 9, 7, 32, 16), (1, 12, 12, 64, 128), (3, 5, 32, 1024, 64)])
def test_wgrad_pw_conv3x3_taps(cuda, B, H, W, N, C):
    """Nine shifted launches = the weight gradient of a dense 3x3 conv, written with the [N][C][3][3] strides."""
    import torch.nn.functional as F
    from efficientsam3_b200 import ops
    g = _g(B + H + N)
    dy, a = _bf(torch.randn(B, H, W, N, generator=g)), _bf(torch.randn(B, H, W, C, generator=g))
    w = torch.zeros(N, C, 3, 3, requires_grad=True)
    y = F.conv2d(a.float().permute(0, 3, 1, 2), w, padding=1)
    (ref,) = torch.autograd.grad(y, w, dy.float().permute(0, 3, 1, 2))
    got = torch.zeros(N, C, 3, 3, device=cuda)
    flat = got.view(-1)
    dy2, a2 = dy.to(cuda).view(-1, N), a.to(cuda).view(-1, C)
    for ky in range(3):
        for kx in range(3):
            ops.wgrad_pw(dy2, a2, flat[ky * 3 + kx:], ldn=9 * C, ldk=9, shift=(H, W, ky - 1, kx - 1))
    _close(got, ref, 2e-3, "conv3x3 wgrad")


@pytest.mark.parametrize("B,H,W,N,C", [(2, 9, 7, 32, 16), (1, 12, 12, 64, 128), (2, 32, 32, 1024, 256), (3, 5, 33, 128, 64)])
def test_conv3x3_wgrad_tc(cuda, B, H, W, N, C):
    """The wgmma route of the head.3 weight gradient: zero-framed transposes + nine GEMMs over the pixel index."""
    from efficientsam3_b200 import ops
    g = _g(B + H + N + 1)
    dy, a = _bf(torch.randn(B, H, W, N, generator=g)), _bf(torch.randn(B, H, W, C, generator=g))
    # the primitive first
    for dx in (-1, 0, 1):
        Wp = (W + 2 + 7) // 8 * 8
        assert torch.equal(ops.transpose_pad(a.to(cuda), Wp, dx).cpu(), E.transpose_pad(a, Wp, dx)), dx
    ref = torch.full((N, C, 3, 3), 0.5)
    E.conv3x3_wgrad(dy, a, ref)
    got = torch.full((N, C, 3, 3), 0.5, device=cuda)
    ops.conv3x3_wgrad(dy.to(cuda), a.to(cuda), got)
    _close(got, ref, 2e-3, "conv3x3_wgrad (wgmma)")


@pytest.mark.parametrize("B,H,W,C,ks,stride", [(2, 17, 23, 64, 3, 2), (1, 32, 32, 256, 3, 2), (2, 16, 16, 16, 3, 1), (1, 9, 11, 96, 5, 1),
                                               (2, 8, 8, 1024, 3, 2), (1, 21, 20, 128, 5, 2), (2, 13, 19, 64, 3, 1), (1, 7, 5, 32, 5, 1), (2, 64, 64, 384, 5, 1),
                                               (2, 40, 40, 512, 3, 1)])
def test_dwconv_gradients(cuda, B, H, W, C, ks, stride):
    from efficientsam3_b200 import ops
    g = _g(B * H + C + ks)
    pad = ks // 2
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    x = _bf(torch.randn(B, H, W, C, generator=g))
    dz = _bf(torch.randn(B, Ho, Wo, C, generator=g))
    w = torch.randn(ks * ks, C, generator=g) / ks
    _close(ops.dwconv_bwd_data(dz.to(cuda), w.to(cuda), H, W, ks, stride), E.dwconv_bwd_data(dz, w, H, W, ks, stride), 1e-2,
           "dwconv_bwd_data")
    if stride == 1:   # the route the training graph takes for stride 1: the forward kernel on the rotated taps
        _close(ops.dwconv(dz.to(cuda), w.flip(0).contiguous().to(cuda), None, ks, 1, None), E.dwconv_bwd_data(dz, w, H, W, ks, 1), 1e-2,
               "dwconv on flipped taps")
    ref = torch.full((C, 1, ks, ks), 0.125)
    E.dwconv_wgrad(dz, x, ref, ks, stride)
    got = torch.full((C, 1, ks, ks), 0.125, device=cuda)
    ops.dwconv_wgrad(dz.to(cuda), x.to(cuda), got, ks, stride)
    _close(got, ref, 2e-3, "dwconv_wgrad")


def test_dwconv_wgrad_channel_slice(cuda):
    """x is the qkv half of the LiteMLA multi-scale buffer (pixel stride 2*c3)."""
    from efficientsam3_b200 import ops
    g = _g(21)
    B, H, W, c3 = 2, 10, 10, 96
    ms = _bf(torch.randn(B, H, W, 2 * c3, generator=g))
    dz = _bf(torch.randn(B, H, W, c3, generator=g))
    ref = torch.zeros(c3, 1, 5, 5)
    E.dwconv_wgrad(dz, ms[..., :c3], ref, 5, 1)
    got = torch.zeros(c3, 1, 5, 5, device=cuda)
    ops.dwconv_wgrad(dz.to(cuda), ms.to(cuda)[..., :c3], got, 5, 1)
    _close(got, ref, 2e-3, "dwconv_wgrad slice")


@pytest.mark.parametrize("B,H,W,Cout", [(2, 64, 64, 16), (1, 37, 51, 8), (3, 32, 48, 24)])
def test_stem_wgrad(cuda, B, H, W, Cout):
    from efficientsam3_b200 import ops
    g = _g(B + H + Cout)
    img = torch.randn(B, 3, H, W, generator=g)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dz = _bf(torch.randn(B, Ho, Wo, Cout, generator=g))
    ref = torch.full((Cout, 3, 3, 3), 1.0)
    E.stem_wgrad(img, dz, ref)
    got = torch.full((Cout, 3, 3, 3), 1.0, device=cuda)
    ops.stem_wgrad(img.to(cuda), dz.to(cuda), got)
    _close(got, ref, 2e-3, "stem_wgrad")


@pytest.mark.parametrize("B,C,Hi,Wi,Ho,Wo", [(2, 64, 5, 5, 12, 12), (1, 1024, 32, 32, 64, 64), (2, 96, 10, 7, 9, 20), (1, 32, 16, 16, 6, 6)])
def test_bilinear_bwd(cuda, B, C, Hi, Wi, Ho, Wo):
    from efficientsam3_b200 import ops
    dout = torch.randn(B, C, Ho, Wo, generator=_g(B + C + Ho))
    _close(ops.bilinear_bwd(dout.to(cuda), Hi, Wi), E.bilinear_bwd(dout, Hi, Wi), 1e-2, "bilinear_bwd")


@pytest.mark.parametrize("B,H,W,heads2", [(2, 10, 10, 16), (1, 32, 32, 32), (2, 23, 29, 4)])
def test_litemla_attn_bwd(cuda, B, H, W, heads2):
    from efficientsam3_b200 import ops
    g = _g(B + H + heads2)
    ms = _bf(torch.randn(B, H, W, 48 * heads2, generator=g))
    datt = _bf(torch.randn(B, H, W, 16 * heads2, generator=g))
    att, kv = ops.litemla_attn(ms.to(cuda), heads2, 1e-15, return_kv=True)
    _close(att, E.litemla_attn(ms, heads2, 1e-15), 1e-2, "litemla_attn fwd")
    got = ops.litemla_attn_bwd(ms.to(cuda), datt.to(cuda), kv, heads2, 1e-15)
    _close(got, E.litemla_attn_bwd(ms, datt, None, heads2, 1e-15), 1.5e-2, "litemla_attn_bwd")


# --------------------------------------------------------------------------------------------- whole steps
def _student(name, img, embed, seed=3):
    from efficientsam3_b200.stage1.model import build_image_student_model
    from oracle.weights import fill_state_dict
    cfg = NS(MODEL=NS(BACKBONE=name), DATA=NS(IMG_SIZE=img), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=embed))
    m = build_image_student_model(cfg)
    m.load_state_dict(fill_state_dict(m.state_dict(), seed))
    return m


def _oracle_grads(sd0, x, teacher, img, sizes, variant, embed, bn_train, device="cpu", autocast=None):
    """Autograd of the oracle: fp32 on the CPU (the reference), or -- device="cuda", autocast=dtype -- the same graph the way the
    reference trains it (torch.autocast around the student forward, train_image_encoder_stage1.py:199-203), as a yardstick for what
    reduced-precision activations alone do to these gradients."""
    import contextlib
    from oracle import efficientvit as O
    from oracle.kd_loss import kd_loss
    sd = {k: (v.clone().to(device).requires_grad_(True) if (v.is_floating_point() and "running" not in k) else v.clone().to(device))
          for k, v in sd0.items()}
    x, teacher = x.to(device), teacher.to(device)
    with (torch.autocast("cuda", dtype=autocast) if autocast is not None else contextlib.nullcontext()):
        if bn_train:
            with O.bn_batch_stats():
                out = O.image_student_encoder(sd, x, embed, variant)
        else:
            out = O.image_student_encoder(sd, x, embed, variant)
    out = out.float()
    loss, _, _ = kd_loss(out, teacher, img, sizes, 1.0)
    loss.backward()
    return out.detach(), loss.item(), sd


@pytest.mark.parametrize("name,variant,bn_train", [("efficientvit_b1", "b1", False), ("efficientvit_b1", "b1", True),
                                                   ("efficientvit_b0", "b0", False)])
def test_student_training_step_matches_oracle_autograd(cuda, name, variant, bn_train):
    """preds = model(x); loss = KD(preds, teacher); loss.backward() on the native path vs autograd of the CPU oracle."""
    from efficientsam3_b200.stage1.optim import KDLossFunction
    img, embed, B = 320, 20, 4
    m = _student(name, img, embed)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(B, 3, img, img, generator=_g(1))
    teacher = torch.randn(B, 1024, embed, embed, generator=_g(2))
    sizes = [(3, img, img * 3 // 4) if i % 2 == 0 else (3, img * 2 // 3, img) for i in range(B)]
    m = m.to(cuda).train()
    if not bn_train:
        for mod in m.modules():
            if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
                mod.eval()
    out = m(x.to(cuda))
    assert out.requires_grad and out.dtype == torch.float32 and out.shape == (B, 1024, embed, embed)
    sz = torch.tensor([[s[1], s[2]] for s in sizes], dtype=torch.int32, device=cuda)
    loss = KDLossFunction.apply(out, teacher.to(cuda), sz, img, 1.0)
    loss.backward()
    torch.cuda.synchronize()
    ref_out, ref_loss, sd = _oracle_grads(sd0, x, teacher, img, sizes, variant, embed, bn_train)
    tol_out, tol_all = (0.15, 0.6) if bn_train else (2e-2, 5e-2)
    rel_out = ((out.detach().cpu().double() - ref_out.double()).norm() / ref_out.double().norm()).item()
    num = den = 0.0
    for k, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        g = sd[k].grad.double()
        num += (p.grad.cpu().double() - g).pow(2).sum().item()
        den += g.pow(2).sum().item()
    rel_all = (num / den) ** 0.5
    print(f"{name} bn_train={bn_train}: out rel-L2 {rel_out:.3e}, loss {loss.item():.5f} vs {ref_loss:.5f}, all-gradient rel-L2 {rel_all:.3e}")
    assert rel_out < tol_out, rel_out
    assert rel_all < tol_all, rel_all
    if bn_train:
        # yardstick: the SAME fp32 oracle graph under torch.autocast (how the reference itself trains) against the fp32 oracle.  The
        # batch-statistics gradients of this random-weight fixture move by a comparable amount from reduced-precision activations
        # alone, i.e. the distance above is the precision class, not a graph error (the graph is exact in fp64: tests/test_train_cpu.py)
        for dt in (torch.bfloat16, torch.float16):
            _, _, sda = _oracle_grads(sd0, x, teacher, img, sizes, variant, embed, True, device=cuda, autocast=dt)
            n = sum((sda[k].grad.cpu().double() - sd[k].grad.double()).pow(2).sum().item() for k, _ in m.named_parameters())
            rel_auto = (n / den) ** 0.5
            print(f"  torch.autocast({dt}) oracle vs fp32 oracle: all-gradient rel-L2 {rel_auto:.3e}")
            if dt is torch.bfloat16:
                assert rel_all < max(3.0 * rel_auto, 0.1), (rel_all, rel_auto)
    if bn_train:
        for k, v in m.state_dict().items():
            if k.endswith("num_batches_tracked"):
                assert int(v) == int(sd0[k]) + 1, k


def test_training_steps_reduce_the_loss_and_are_deterministic(cuda):
    """A few full KD steps (train-mode student -> KD loss -> backward -> FlatAdamW) on one fixed batch: the loss goes down,
    and two identical runs produce bit-identical parameters (fixed-order reductions, no atomics)."""
    from efficientsam3_b200.stage1.optim import FlatAdamW, KDLossFunction
    img, embed, B = 256, 16, 4
    x = torch.randn(B, 3, img, img, generator=_g(5)).to(cuda)
    teacher = (torch.randn(B, 1024, embed, embed, generator=_g(6)) * 0.5).to(cuda)
    sz = torch.tensor([[img, img]] * B, dtype=torch.int32, device=cuda)

    def run():
        m = _student("efficientvit_b1", img, embed).to(cuda).train()
        opt = FlatAdamW(m, lr=1e-4, weight_decay=0.01)   # 2e-3 diverges on this random-weight fixture (CPU emulation agrees)
        losses = []
        for _ in range(6):
            opt.zero_grad()
            loss = KDLossFunction.apply(m(x), teacher, sz, img, 1.0)
            loss.backward()
            opt.step(max_norm=5.0)
            losses.append(loss.item())
        return losses, opt.flat_param.clone()

    l1, p1 = run()
    l2, p2 = run()
    print("losses", [round(v, 4) for v in l1])
    assert all(math.isfinite(v) for v in l1)
    assert l1[-1] < 0.8 * l1[0] and all(b < a for a, b in zip(l1, l1[1:])), l1
    assert l1 == l2 and torch.equal(p1, p2)
    # and the eval-mode forward after training uses the updated weights (stale packed plans are dropped)
    m = _student("efficientvit_b1", img, embed).to(cuda)
    m.eval()
    e0 = m(x)
    m.train()
    opt = FlatAdamW(m, lr=1e-2, weight_decay=0.0)
    loss = KDLossFunction.apply(m(x), teacher, sz, img, 1.0)
    loss.backward()
    opt.step()
    m.eval()
    e1 = m(x)
    assert (e1 - e0).abs().max().item() > 1e-3


def test_direct_arena_gradients_equal_autograd_gradients(cuda):
    """FlatAdamW(direct_grads=True): the backward kernels accumulate straight into the flat gradient arena (the all-reduce buffer);
    direct_grads=False: per-parameter temporaries returned to autograd, which adds them into the same views.  Bit-identical."""
    from efficientsam3_b200.stage1.optim import FlatAdamW, KDLossFunction
    img, embed, B = 192, 12, 2
    x = torch.randn(B, 3, img, img, generator=_g(8)).to(cuda)
    teacher = torch.randn(B, 1024, embed, embed, generator=_g(9)).to(cuda)
    sz = torch.tensor([[img, img * 3 // 4]] * B, dtype=torch.int32, device=cuda)
    arenas = []
    for direct in (True, False):
        m = _student("efficientvit_b1", img, embed).to(cuda).train()
        opt = FlatAdamW(m, lr=1e-4, direct_grads=direct)
        assert (getattr(m, "_es3_grad_arena", None) is opt) == direct
        for _ in range(2):                                   # two backward passes: accumulation into the arena
            KDLossFunction.apply(m(x), teacher, sz, img, 1.0).backward()
        arenas.append(opt.flat_grad.clone())
    assert arenas[0].abs().sum().item() > 0 and torch.equal(arenas[0], arenas[1])


def test_cuda_graph_replay_equals_the_kernel_sequence(cuda):
    """enable_cuda_graphs(): the eval forward replayed from a CUDA graph is bit-identical to the host-launched kernel sequence, per
    input buffer; a parameter update invalidates the captured graph."""
    img, embed = 192, 12
    m = _student("efficientvit_b1", img, embed).to(cuda).eval()
    xs = [torch.randn(2, 3, img, img, generator=_g(20 + i)).to(cuda) for i in range(2)]
    ref = [m(x).clone() for x in xs]
    m.enable_cuda_graphs()
    for rep in range(3):
        for x, r in zip(xs, ref):
            assert torch.equal(m(x), r)
    assert len(m._graphs) == 2 and m.graph_launches_per_step > 0
    xs[0].mul_(0.5)                                          # same buffer, new contents: replay must read the new pixels
    assert torch.equal(m(xs[0]), m.forward_uncaptured(xs[0]))
    with torch.no_grad():
        m.head[3].bias.add_(1.0)                             # bumps the parameter version: the graph is captured again
    out = m(xs[1])
    assert torch.equal(out, m.forward_uncaptured(xs[1])) and not torch.equal(out, ref[1])
    m.enable_cuda_graphs(False)
    assert torch.equal(m(xs[1]), out)


@pytest.mark.parametrize("M,L,ld", [(1, 5, 5), (37, 130, 136), (4000, 784, 784), (11552, 9604, 9604), (3, 38416, 38416)])
def test_colsum_f32(cuda, M, L, ld):
    from efficientsam3_b200 import ops
    g = _g(M + L)
    src = torch.randn(M, ld, generator=g)
    out0 = torch.randn(L, generator=g)
    got = out0.clone().to(cuda)
    ops.colsum_f32(src.to(cuda)[:, :L], got)
    ref = out0.double() + src[:, :L].double().sum(0)
    err = (got.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-5, err
    again = out0.clone().to(cuda)
    ops.colsum_f32(src.to(cuda)[:, :L], again)
    assert torch.equal(got, again)                          # fixed reduction order


def test_half_width_image_batches(cuda):
    """bf16 image batches (half the host->device bytes) go through a device cast and then the same kernels: the result equals the forward
    of the rounded batch exactly, and is within the bf16 tolerance of the fp32 batch (the stem rounds its operands to bf16 itself)."""
    img, embed = 192, 9
    m = _student("efficientvit_b1", img, embed).to(cuda).eval()
    x = torch.randn(2, 3, img, img, generator=_g(3)).to(cuda)
    xb = x.to(torch.bfloat16)
    a, b, c = m(x), m(xb), m(xb.float())
    assert torch.equal(b, c)
    rel = ((a - b).double().norm() / a.double().norm()).item()
    print(f"bf16 image batch vs fp32 batch: rel-L2 {rel:.3e}, bit-identical: {torch.equal(a, b)}")
    assert rel < 1e-2


# ---------------------------------------------------------------------------------------------
# Training graphs of the three student families against autograd of the CPU oracle.
@pytest.mark.parametrize("bn_train", [False, True])
def test_repvit_training_step_matches_oracle_autograd(cuda, bn_train):
    from efficientsam3_b200.stage1.optim import KDLossFunction
    from oracle import efficientvit as O
    from oracle import repvit as R
    from oracle.kd_loss import kd_loss
    img, embed, B = 256, 16, 4
    m = _student("repvit_m1_1", img, embed, seed=11)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(B, 3, img, img, generator=_g(1))
    teacher = torch.randn(B, 1024, embed, embed, generator=_g(2))
    sizes = [(3, img, img * 3 // 4) if i % 2 == 0 else (3, img * 2 // 3, img) for i in range(B)]
    m = m.to(cuda).train()
    if not bn_train:
        for mod in m.modules():
            if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
                mod.eval()
    out = m(x.to(cuda))
    sz = torch.tensor([[s[1], s[2]] for s in sizes], dtype=torch.int32, device=cuda)
    loss = KDLossFunction.apply(out, teacher.to(cuda), sz, img, 1.0)
    loss.backward()
    torch.cuda.synchronize()
    sd = {k: (v.clone().requires_grad_(True) if (v.is_floating_point() and "running" not in k) else v.clone()) for k, v in sd0.items()}
    if bn_train:
        with O.bn_batch_stats():
            ref_out = R.image_student_encoder(sd, x, embed, "repvit_m1_1")
    else:
        ref_out = R.image_student_encoder(sd, x, embed, "repvit_m1_1")
    ref_loss, _, _ = kd_loss(ref_out, teacher, img, sizes, 1.0)
    ref_loss.backward()
    rel_out = ((out.detach().cpu().double() - ref_out.detach().double()).norm() / ref_out.detach().double().norm()).item()
    num = den = 0.0
    for k, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        g = sd[k].grad.double()
        num += (p.grad.cpu().double() - g).pow(2).sum().item()
        den += g.pow(2).sum().item()
    rel_all = (num / den) ** 0.5
    print(f"repvit_m1_1 bn_train={bn_train}: out rel-L2 {rel_out:.3e}, all-gradient rel-L2 {rel_all:.3e}")
    tol_out, tol_all = (0.15, 0.6) if bn_train else (2e-2, 5e-2)
    assert rel_out < tol_out and rel_all < tol_all, (rel_out, rel_all)


@pytest.mark.parametrize("B,H,W,C,ks,stride", [(2, 16, 16, 32, 3, 1), (1, 9, 11, 96, 5, 1), (2, 64, 64, 384, 5, 1), (2, 40, 37, 512, 3, 1),
                                               (1, 7, 5, 64, 5, 1), (2, 64, 64, 64, 3, 2), (1, 37, 51, 128, 3, 2), (3, 18, 70, 32, 3, 2),
                                               (1, 33, 33, 64, 5, 2), (2, 8, 100, 96, 3, 1)])
def test_dwconv_wgrad_win(cuda, B, H, W, C, ks, stride):
    """Sliding-window weight gradient (the default for C % 32 == 0) against the torch statement and against the direct kernels."""
    from efficientsam3_b200 import ops
    g = _g(B * H + C + ks + stride)
    ms = _bf(torch.randn(B, H, W, 2 * C, generator=g))
    Ho, Wo = (H + 2 * (ks // 2) - ks) // stride + 1, (W + 2 * (ks // 2) - ks) // stride + 1
    dz = _bf(torch.randn(B, Ho, Wo, C, generator=g))
    ref = torch.full((C, 1, ks, ks), 0.125)
    E.dwconv_wgrad(dz, ms[..., :C], ref, ks, stride)
    got = torch.full((C, 1, ks, ks), 0.125, device=cuda)
    ops.dwconv_wgrad(dz.to(cuda), ms.to(cuda)[..., :C], got, ks, stride, impl="win")
    _close(got, ref, 2e-3, "dwconv_wgrad win")
    direct = torch.full((C, 1, ks, ks), 0.125, device=cuda)
    ops.dwconv_wgrad(dz.to(cuda), ms.to(cuda)[..., :C], direct, ks, stride, impl="direct")
    _close(got, direct.cpu(), 1e-4, "dwconv_wgrad win vs direct")


@pytest.mark.parametrize("B,H,W,C", [(3, 16, 16, 64), (2, 9, 7, 128), (4, 32, 32, 256), (2, 5, 5, 2560)])
def test_se_bwd_batched(cuda, B, H, W, C):
    from efficientsam3_b200 import ops
    g = _g(B + H + C)
    dy, x = _bf(torch.randn(B, H, W, C, generator=g)), _bf(torch.randn(B, H, W, C, generator=g))
    gate, add = torch.rand(B, C, generator=g), torch.randn(B, C, generator=g) * 0.1
    _close(ops.se_bwd_dgate(dy.to(cuda), x.to(cuda)), E.se_bwd_dgate(dy, x), 2e-3, "se_bwd_dgate")
    _close(ops.se_bwd_apply(dy.to(cuda), gate.to(cuda), add.to(cuda)), E.se_bwd_apply(dy, gate, add), 1e-2, "se_bwd_apply")


def test_efficientsam3_student_segmenter_vs_oracles(cuda):
    """build_efficientsam3_point_segmenter("efficientvit", "b1"): image -> EV-M student -> 1024 x 72 x 72 -> SAM2-branch FPN -> point-prompt
    mask decoding, against the oracle composition (efficientvit + student head + neck + SAM heads)."""
    from efficientsam3_b200.model_builder import build_efficientsam3_point_segmenter
    from oracle import efficientvit as EV, necks as ON, sam_heads as OH
    from oracle.weights import fill_state_dict
    seg = build_efficientsam3_point_segmenter("efficientvit", "b1")
    sd = {k: v for k, v in fill_state_dict(seg.state_dict(), 47).items() if not v.is_complex()}
    seg.load_state_dict(sd, strict=False)
    B, S = 2, 1008
    g = torch.Generator().manual_seed(6)
    img = torch.randn(B, 3, S, S, generator=g)
    coords = torch.rand(B, 1, 2, generator=g) * S
    labels = torch.ones(B, 1, dtype=torch.int32)
    with torch.no_grad():
        vb = {k[len("backbone.vision_backbone."):]: v for k, v in sd.items() if k.startswith("backbone.vision_backbone.")}
        feats = EV.image_student_encoder({k[len("trunk.model."):]: v for k, v in vb.items() if k.startswith("trunk.model.")}, img, 72, "b1")
        l288, l144, l72 = ON.neck(vb, feats, prefix="sam2_convs.")[:3]
        sd_md = {k[len("sam_mask_decoder."):]: v for k, v in sd.items() if k.startswith("sam_mask_decoder.")}
        sd_pe = {k[len("sam_prompt_encoder."):]: v for k, v in sd.items() if k.startswith("sam_prompt_encoder.")}
        hr = OH.high_res_from_fpn(sd_md, "", l288, l144)
        ref = OH.forward_sam_heads(sd_pe, sd_md, l72 + sd["no_mem_embed"].reshape(1, -1, 1, 1), hr, coords, labels, S, multimask_output=True)
    seg = seg.to(cuda)
    out = seg.set_image_batch(img.to(cuda)).predict_batch(coords.to(cuda), labels.to(cuda), multimask_output=True, return_logits=True)
    low = out["low_res_multimasks"].cpu()
    e_low = ((low.double() - ref["low_res_multimasks"].double()).norm() / ref["low_res_multimasks"].double().norm()).item()
    agree = ((out["high_res"].cpu() > 0) == (ref["high_res_multimasks"] > 0)).float().mean().item()
    print(f"EfficientSAM3 (EV-M) point-prompt pipeline: low-res logits rel_l2={e_low:.3e}, binary mask agreement {agree:.5f}")
    assert e_low <= 3e-2 and agree >= 0.99
    assert torch.equal(out["best"].cpu(), ref["best"])


@pytest.mark.parametrize("B,H,W,heads2,dim", [(2, 10, 10, 8, 32), (1, 23, 29, 4, 32), (2, 12, 12, 6, 16)])
def test_litemla_attn_bwd_generic(cuda, B, H, W, heads2, dim):
    from efficientsam3_b200 import ops
    g = _g(B + H + heads2 + dim)
    ms = _bf(torch.randn(B, H, W, 3 * dim * heads2, generator=g))
    datt = _bf(torch.randn(B, H, W, dim * heads2, generator=g))
    att, kv = ops.litemla_attn_generic(ms.to(cuda), heads2, dim, 1e-15, return_kv=True)
    _close(att, E.litemla_attn_generic(ms, heads2, dim, 1e-15), 1e-2, "litemla_attn_generic fwd")
    got = ops.litemla_attn_bwd_generic(ms.to(cuda), datt.to(cuda), kv, heads2, dim, 1e-15)
    _close(got, E.litemla_attn_bwd_generic(ms, datt, None, heads2, dim, 1e-15), 1.5e-2, "litemla_attn_bwd_generic")


def test_efficientvit_b2_training_step_matches_oracle_autograd(cuda):
    from efficientsam3_b200.stage1.optim import KDLossFunction
    img, embed, B = 320, 20, 2
    m = _student("efficientvit_b2", img, embed)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(B, 3, img, img, generator=_g(1))
    teacher = torch.randn(B, 1024, embed, embed, generator=_g(2))
    sizes = [(3, img, img)] * B
    m = m.to(cuda).train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
            mod.eval()
    out = m(x.to(cuda))
    sz = torch.tensor([[img, img]] * B, dtype=torch.int32, device=cuda)
    loss = KDLossFunction.apply(out, teacher.to(cuda), sz, img, 1.0)
    loss.backward()
    torch.cuda.synchronize()
    ref_out, _, sd = _oracle_grads(sd0, x, teacher, img, sizes, "b2", embed, False)
    num = den = 0.0
    for k, p in m.named_parameters():
        g = sd[k].grad.double()
        num += (p.grad.cpu().double() - g).pow(2).sum().item()
        den += g.pow(2).sum().item()
    print(f"efficientvit_b2 (frozen BN): all-gradient rel-L2 {(num / den) ** 0.5:.3e}")
    assert (num / den) ** 0.5 < 5e-2


@pytest.mark.parametrize("M,C", [(1000, 64), (777, 448), (4100, 160), (300, 576)])
def test_layernorm_bwd(cuda, M, C):
    from efficientsam3_b200 import ops
    g = _g(M + C)
    x, dy = _bf(torch.randn(M, C, generator=g) * 2 + 0.5), _bf(torch.randn(M, C, generator=g))
    dres = _bf(torch.randn(M, C, generator=g))
    gamma = torch.rand(C, generator=g) + 0.5
    dg_ref, db_ref = torch.full((C,), 0.5), torch.full((C,), -1.0)
    ref = E.layernorm_bwd(x, dy, gamma, 1e-5, dg_ref, db_ref, dres)
    dg, db = torch.full((C,), 0.5, device=cuda), torch.full((C,), -1.0, device=cuda)
    got = ops.layernorm_bwd(x.to(cuda), dy.to(cuda), gamma.to(cuda), 1e-5, dg, db, dres.to(cuda))
    _close(got, ref, 1e-2, "layernorm_bwd dx")
    _close(dg, dg_ref, 2e-3, "layernorm_bwd dgamma")
    _close(db, db_ref, 2e-3, "layernorm_bwd dbeta")


@pytest.mark.parametrize("B,H,W,heads,ws", [(2, 14, 21, 4, 7), (1, 14, 28, 8, 14), (2, 7, 7, 5, 7)])
def test_win_attn_bias_bwd(cuda, B, H, W, heads, ws):
    from efficientsam3_b200 import ops
    g = _g(B + H + heads + ws)
    C, N = 32 * heads, ws * ws
    qkv = _bf(torch.randn(B * H * W, 3 * C, generator=g))
    dout = _bf(torch.randn(B * H * W, C, generator=g))
    bias = torch.randn(heads, N, N, generator=g) * 0.5
    scale = 32 ** -0.5
    fwd = ops.win_attn_bias(qkv.to(cuda), torch.zeros(3 * C, dtype=torch.bfloat16, device=cuda), bias.to(cuda), B, H, W, C, heads, ws, scale)
    _close(fwd, E.win_attn_bias(qkv, None, bias, B, H, W, C, heads, ws, scale), 1e-2, "win_attn_bias fwd")
    dq, db = ops.win_attn_bias_bwd(qkv.to(cuda), dout.to(cuda), bias.to(cuda), B, H, W, C, heads, ws, scale)
    rq, rb = E.win_attn_bias_bwd(qkv, dout, bias, B, H, W, C, heads, ws, scale)
    _close(dq, rq, 1.5e-2, "win_attn_bias_bwd dqkv")
    _close(db, rb, 2e-3, "win_attn_bias_bwd dbias")      # per-window dS in fp32, summed over the windows in fp32


def test_tinyvit_training_step_matches_oracle_autograd(cuda):
    from efficientsam3_b200.stage1.optim import KDLossFunction
    from oracle import tinyvit as TV
    from oracle.kd_loss import kd_loss
    img, embed, B = 224, 14, 2
    m = _student("tiny_vit_11m", img, embed, seed=17)
    for mod in m.modules():
        if hasattr(mod, "drop_path_rate"):
            mod.drop_path_rate = 0.0
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(B, 3, img, img, generator=_g(1))
    teacher = torch.randn(B, 1024, embed, embed, generator=_g(2))
    sizes = [(3, img, img)] * B
    m = m.to(cuda).train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
            mod.eval()
    out = m(x.to(cuda))
    sz = torch.tensor([[img, img]] * B, dtype=torch.int32, device=cuda)
    loss = KDLossFunction.apply(out, teacher.to(cuda), sz, img, 1.0)
    loss.backward()
    torch.cuda.synchronize()
    sd = {k: (v.clone().requires_grad_(True) if (v.is_floating_point() and "running" not in k) else v.clone()) for k, v in sd0.items()}
    ref_loss, _, _ = kd_loss(TV.image_student_encoder(sd, x, embed, "tiny_vit_11m"), teacher, img, sizes, 1.0)
    ref_loss.backward()
    num = den = 0.0
    for k, p in m.named_parameters():
        gq = sd[k].grad.double()
        num += (p.grad.cpu().double() - gq).pow(2).sum().item()
        den += gq.pow(2).sum().item()
    print(f"tiny_vit_11m (frozen BN, no DropPath): all-gradient rel-L2 {(num / den) ** 0.5:.3e}")
    assert (num / den) ** 0.5 < 8e-2
