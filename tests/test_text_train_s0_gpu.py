"""GPU: training MobileCLIP-S0 natively with frozen BatchNorm -- the RepMixerBlock backward kernels (csrc/repmixer_bwd.cu) against
fp64 torch autograd, whole training graphs against the oracle's autograd (with the bf16-autocast oracle as the precision yardstick),
the reference's frozen-BN iteration (tests/golden/gen_golden_text_train_s0.py) end to end from strings, the train-mode forward
against the eval fixtures, frozen running statistics, the optimiser interplay and the raise paths."""
import contextlib
import random

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from helpers import load_golden, max_err_over_scale, rel_l2
from oracle import text as OT
from oracle.weights import fill_state_dict
from test_text_cpu import oracle_cfg
from test_text_gpu import captions, check_memory, loaded_student
from test_text_train_cpu import build_train_student, fixture_permutations, grad_stats, ref_text_loss
from test_text_train_gpu import _all_grad_rel, _cfg_ns, _permuted, _student
from test_text_train_s0_cpu import oracle_sd

pytestmark = pytest.mark.gpu


def freeze_bn(m):
    """.train(), then every BatchNorm back in .eval() (set_bn_state with TRAIN.EVAL_BN_WHEN_TRAINING)."""
    m.train()
    for mod in m.modules():
        if isinstance(mod, nn.modules.batchnorm._BatchNorm):
            mod.eval()
    return m


# ------------------------------------------------------------------------------------------------ kernels vs fp64 autograd
def _block(C, seed, dev):
    from efficientsam3_b200.backbones.mobile_clip import RepMixerBlock, RepMixerUnit
    blk = RepMixerBlock(dim=C)
    sd = fill_state_dict(blk.state_dict(), seed)
    blk.load_state_dict(sd)
    blk = blk.to(dev).eval()
    sd64 = {k: v.to(dev, torch.float64) for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    return blk, RepMixerUnit(blk)._pack(), sd64


def _t(rows, B, L):
    """[B*L, C] -> [B, C, 1, L] fp64 leaf (the reference's layout)."""
    return rows.double().view(B, L, -1).permute(0, 2, 1).unsqueeze(2).clone().requires_grad_(True)


def _rows(t):
    return t.squeeze(2).permute(0, 2, 1).reshape(-1, t.shape[1])


def _leaves(sd64, names):
    return {n: sd64[n].clone().requires_grad_(True) for n in names}


def _acc(shape, dev):
    """A gradient destination pre-filled with 0.25: the kernels add into it."""
    return torch.full(shape, 0.25, device=dev)


def _check(got, ref, tol, what):
    err = max_err_over_scale(got.double().cpu(), ref.double().cpu())
    assert err <= tol, (what, err)


@pytest.mark.parametrize("C", [32, 512])
@pytest.mark.parametrize("L", [1, 4, 11, 16, 32, 77, 128])
@pytest.mark.parametrize("B", [1, 3, 64])
def test_repmixer_bwd_kernels(cuda, B, L, C):
    from efficientsam3_b200 import ops
    blk, p, sd = _block(C, 7 * L + C + B, cuda)
    gen = torch.Generator().manual_seed(B * 1000 + L * 10 + C)
    x, x1, g, du, y, e = (torch.randn(B * L, C, generator=gen).to(cuda) for _ in range(6))
    bn_names = ["token_mixer.mixer.rbr_skip", "token_mixer.mixer.rbr_conv.0.bn", "token_mixer.norm.rbr_skip"]
    bn_leaf = [f"{n}.{w}" for n in bn_names for w in ("weight", "bias")]

    def run():
        outs = {}
        outs["dls_blk"], outs["db2"] = _acc((C, 1, 1), cuda), _acc((C,), cuda)
        outs["dy"] = ops.repmixer_ls_bwd(g, y, p["lsb"], B, L, dls=outs["dls_blk"], dbias=outs["db2"])
        outs["dwf"], outs["dgf"], outs["dbf"] = _acc((C, 1, 1, 11), cuda), _acc((C,), cuda), _acc((C,), cuda)
        outs["e"] = ops.repmixer_ffn_bwd(x1, du, g, p["f_taps"], p["bnf"], B, L, dtaps=outs["dwf"], dgamma=outs["dgf"],
                                         dbeta=outs["dbf"])
        outs["dwm"], outs["dls_tm"] = _acc((C, 1, 1, 11), cuda), _acc((C, 1, 1), cuda)
        dbn = [_acc((C,), cuda) for _ in range(6)]
        outs["dx"], outs["dxb"] = ops.repmixer_tm_bwd(x, e, p["tm_taps"], p["bnp"], B, L, dtaps=outs["dwm"], dls=outs["dls_tm"],
                                                      dbn=dbn, want_bf16=True)
        for n, t in zip(bn_leaf, dbn):
            outs[n] = t
        return outs

    got = run()
    # layer scale: x2 = x1 + ls * y
    ls = sd["layer_scale"].reshape(-1)
    g64, y64 = g.double(), y.double()
    _check(got["dy"], ls * g64, 1e-2, "dy")
    _check(got["dls_blk"] - 0.25, (g64 * y64).sum(0).view(C, 1, 1), 2e-3, "d ls_blk")
    _check(got["db2"] - 0.25, (ls * g64).sum(0), 2e-3, "d fc2.bias")
    # ConvFFN.conv + BN_f: e = d/dx1 of (sum du * BN_f(dw(x1)) + sum g * x1)
    lv = _leaves(sd, ["convffn.conv.conv.weight", "convffn.conv.bn.weight", "convffn.conv.bn.bias"])
    t1 = _t(x1, B, L)
    u = OT._bn(OT._dw(t1, lv["convffn.conv.conv.weight"]), {**sd, **lv}, "convffn.conv.bn")
    ((u * _t(du, B, L).detach()).sum() + (t1 * _t(g, B, L).detach()).sum()).backward()
    _check(got["e"], _rows(t1.grad), 2e-3, "e")
    _check(got["dwf"] - 0.25, lv["convffn.conv.conv.weight"].grad, 2e-3, "d w_f")
    _check(got["dgf"] - 0.25, lv["convffn.conv.bn.weight"].grad, 2e-3, "d gamma_f")
    _check(got["dbf"] - 0.25, lv["convffn.conv.bn.bias"].grad, 2e-3, "d beta_f")
    # token mixer: dx = d/dx of sum e * (x + ls_tm (BN_ms(x) + BN_mc(dw(x)) - BN_ns(x)))
    lv = _leaves(sd, ["token_mixer.mixer.rbr_conv.0.conv.weight", "token_mixer.layer_scale", *bn_leaf])
    s = {**sd, **lv}
    t = _t(x, B, L)
    tm = "token_mixer"
    mixer = OT._bn(t, s, tm + ".mixer.rbr_skip") + OT._bn(OT._dw(t, s[tm + ".mixer.rbr_conv.0.conv.weight"]), s,
                                                          tm + ".mixer.rbr_conv.0.bn")
    out = t + s[tm + ".layer_scale"] * (mixer - OT._bn(t, s, tm + ".norm.rbr_skip"))
    (out * _t(e, B, L).detach()).sum().backward()
    _check(got["dx"], _rows(t.grad), 2e-3, "dx")
    _check(got["dxb"], _rows(t.grad), 1e-2, "dx bf16")
    assert torch.equal(got["dxb"], got["dx"].to(torch.bfloat16))
    _check(got["dwm"] - 0.25, lv[tm + ".mixer.rbr_conv.0.conv.weight"].grad, 2e-3, "d w_mc")
    _check(got["dls_tm"] - 0.25, lv[tm + ".layer_scale"].grad, 2e-3, "d ls_tm")
    for n in bn_leaf:
        _check(got[n] - 0.25, lv[n].grad, 2e-3, n)
    again = run()                                                    # fixed-order reductions: bit-identical
    for k in got:
        assert torch.equal(got[k], again[k]), k


def test_repmixer_bwd_host_checks(cuda):
    from efficientsam3_b200 import ops
    blk, p, _ = _block(32, 1, cuda)
    n0 = ops.launch_count
    for B, L, C in ((1, 129, 32), (2, 4, 48)):
        x = torch.zeros(B * L, C, device=cuda)
        taps, bnf, bnp, ls = (torch.zeros(r, C, device=cuda) for r in (11, 4, 13, 1))
        match = "1..128" if L > 128 else "multiple of 32"
        with pytest.raises(ValueError, match=match):
            ops.repmixer_ls_bwd(x, x, ls.view(-1), B, L)
        with pytest.raises(ValueError, match=match):
            ops.repmixer_ffn_bwd(x, x, x, taps, bnf, B, L)
        with pytest.raises(ValueError, match=match):
            ops.repmixer_tm_bwd(x, x, taps, bnp, B, L)
    assert ops.launch_count == n0


# ------------------------------------------------------------------------------------------------ whole graphs vs the oracle
def _oracle_grads(sd0, m, ids, perm_ids, teacher, valid, w_cos, w_con, dev, autocast=None):
    sd = oracle_sd(sd0, m, dev)
    cfg = oracle_cfg(m)
    ctx = torch.autocast("cuda", dtype=autocast) if autocast is not None else contextlib.nullcontext()
    with ctx:
        preds = OT.text_student(sd, ids.to(dev), cfg)[1].transpose(0, 1)
        perms = [OT.text_student(sd, q.to(dev), cfg)[1].transpose(0, 1) for q in perm_ids]
    preds, perms = preds.float(), [q.float() for q in perms]
    loss, _, _ = ref_text_loss(preds, teacher, valid, w_cos)
    for q in perms:
        loss = loss + w_con * F.mse_loss(preds.mean(1), q.mean(1))
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in sd.items()}


def _compare_s0(m, sd, caps, masked, w_con, dev, label):
    from efficientsam3_b200.stage1.losses import TextKDLossFunction
    w_cos = 1.0
    ids = m.tokenizer(caps, context_length=m.context_length)
    perm_caps = _permuted(caps, 5) if w_con > 0 else []
    perm_ids = [m.tokenizer(pc, context_length=m.context_length) for pc in perm_caps]
    teacher = torch.randn(len(caps), m.context_length, 256, generator=torch.Generator().manual_seed(9)).to(dev)
    valid = (ids != 0).float().to(dev) if masked else None
    freeze_bn(m)
    m.zero_grad(set_to_none=True)
    pad, mem, _ = m(caps)
    perms = [m(pc)[1].transpose(0, 1) for pc in perm_caps]
    loss_n, _, _, _ = TextKDLossFunction.apply(mem.transpose(0, 1), teacher, pad if masked else None, w_cos, w_con, *perms)
    loss_n.backward()
    got = {n: p.grad for n, p in m.named_parameters()}
    loss_r, ref = _oracle_grads(sd, m, ids, perm_ids, teacher, valid, w_cos, w_con, dev)
    _, ref_bf = _oracle_grads(sd, m, ids, perm_ids, teacher, valid, w_cos, w_con, dev, autocast=torch.bfloat16)
    assert got["encoder.projection_layer"] is None
    names = [n for n, _ in m.named_parameters() if n != "encoder.projection_layer"]
    rel = _all_grad_rel(got, ref, names)
    d_bf16 = _all_grad_rel(ref_bf, ref, names)
    print(f"  {label}: loss native {loss_n.item():.6f} oracle {loss_r.item():.6f}; all-gradient rel-L2 native {rel:.3e}, "
          f"torch.autocast(bf16) oracle {d_bf16:.3e}")
    assert abs(loss_n.item() - loss_r.item()) <= 2e-2 * abs(loss_r.item())
    assert rel <= 5e-2 and rel <= 3 * d_bf16, (rel, d_bf16)
    return got


def test_s0_shaped_depth1_masked_consistency(cuda):
    m, sd = _student("MobileCLIP-S0", cuda, layers=1, ctx=32, seed=61)
    _compare_s0(m, sd, captions(), masked=True, w_con=0.5, dev=cuda, label="S0-shaped depth 1, masked + consistency")


def test_s0_full_depth_table77_at_32(cuda):
    m, sd = _student("MobileCLIP-S0", cuda, ctx=32, table=77, seed=62)
    got = _compare_s0(m, sd, captions(), masked=True, w_con=0.0, dev=cuda, label="MobileCLIP-S0 full depth, table 77 at 32")
    assert got["encoder.positional_embedding.pos_embed.pos_embed"].abs().sum().item() > 0


# ------------------------------------------------------------------------------------------------ reference fixtures, eval fixtures
@pytest.mark.parametrize("name", ["text_train_s0_ctx16", "text_train_s0_ctx32"])
def test_s0_train_fixture_end_to_end_from_strings(cuda, name):
    """The reference's frozen-BN iteration natively from strings: permuted captions, loss terms and every parameter's gradient
    statistics, as test_train_fixture_end_to_end_from_strings checks the base students."""
    from efficientsam3_b200.stage1.losses import TextKDLossFunction
    g = load_golden(name)
    m, _ = build_train_student(g)
    m = freeze_bn(m.to(cuda))
    caps, perms = fixture_permutations(g)
    assert [list(p) for p in perms] == [[str(s) for s in row] for row in g["perm_strings"]]
    teacher = torch.from_numpy(g["teacher"]).float().to(cuda)
    pad, mem, _ = m(caps)
    assert torch.equal(pad.cpu(), torch.from_numpy(g["pad"]))
    qs = [m(p)[1].transpose(0, 1) for p in perms]
    loss, mse, cos, cons = TextKDLossFunction.apply(mem.transpose(0, 1), teacher, pad if int(g["masked"]) else None,
                                                    float(g["cosine"]), float(g["consistency"]), *qs)
    loss.backward()
    got_terms = [loss.item(), mse.item(), cos.item(), *cons.tolist()] + [0.0] * (2 - cons.numel())
    for a, b in zip(got_terms[:3], g["loss"][:3]):
        assert abs(a - b) <= 1e-2 * abs(b), (got_terms, g["loss"].tolist())
    e = 1e-2 * mem.detach().transpose(0, 1).mean(1).pow(2).mean().sqrt().item()
    for a, b in zip(got_terms[3:], g["loss"][3:]):
        assert abs(a - b) <= 2 * abs(b) ** 0.5 * e + e * e, (got_terms, g["loss"].tolist(), e)
    params = dict(m.named_parameters())
    got = torch.stack([grad_stats(params[str(n)].grad.cpu()) for n in g["grad_names"]])
    r = rel_l2(got, torch.from_numpy(g["grad_stats"]))
    print(f"  {name}: loss native {got_terms[0]:.6f} reference {g['loss'][0]:.6f}; gradient statistics rel-L2 {r:.3e}")
    assert r <= 5e-2, r
    assert params["encoder.projection_layer"].grad is None
    bufs = dict(m.named_buffers())
    for n, (rm, rv), nbt in zip(g["bn_names"], g["running"], g["num_batches_tracked"]):
        assert np.array_equal(bufs[f"{n}.running_mean"].cpu().numpy(), rm) and np.array_equal(bufs[f"{n}.running_var"].cpu().numpy(), rv)
        assert int(bufs[f"{n}.num_batches_tracked"]) == int(nbt)


@pytest.mark.parametrize("name", ["text_s0_ctx32", "text_s0_resize16", "text_s0_interp"])
def test_frozen_bn_train_mode_memory_matches_eval_fixture(cuda, name):
    g = load_golden(name)
    m = freeze_bn(loaded_student(g, cuda))
    mask, mem, emb = m(captions())
    assert mem.grad_fn is not None and not emb.requires_grad
    assert torch.equal(mask.cpu(), torch.from_numpy(g["mask"]))
    check_memory(mem.detach(), torch.from_numpy(g["memory"]))
    with torch.no_grad():                                       # train mode under no_grad: the eval path
        _, mem_ng, _ = m(captions())
    assert mem_ng.grad_fn is None
    check_memory(mem_ng, torch.from_numpy(g["memory"]))


# ------------------------------------------------------------------------------------------------ optimiser interplay
def _s0_steps(seed, n=3, dev="cuda"):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import text_kd_train_step
    from efficientsam3_b200.stage1.optim import FlatAdamW
    m, _ = _student("MobileCLIP-S0", dev, layers=1, ctx=16, seed=seed)
    freeze_bn(m)
    opt = FlatAdamW(m, lr=1e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    caps = captions()
    teacher = torch.randn(len(caps), 16, 256, generator=torch.Generator().manual_seed(seed)).to(dev)
    random.seed(seed)
    losses = [text_kd_train_step(m, opt, caps, teacher, cosine_weight=1.0, mask_pad_tokens=True, consistency_weight=0.5,
                                 clip_grad=5.0, lr=1e-3).item() for _ in range(n)]
    return m, opt, losses


def test_step_leaves_running_stats_and_reaches_every_parameter(cuda):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import text_kd_train_step
    from efficientsam3_b200.stage1.optim import FlatAdamW
    m, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=71)
    freeze_bn(m)
    bufs0 = {n: b.clone() for n, b in m.named_buffers()}
    opt = FlatAdamW(m, lr=1e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    caps = captions()
    teacher = torch.randn(len(caps), 16, 256, generator=torch.Generator().manual_seed(3)).to(cuda)
    random.seed(3)
    # consistency > 0: three forwards in the iteration; update=False keeps the gradients for inspection
    text_kd_train_step(m, opt, caps, teacher, cosine_weight=2.0, mask_pad_tokens=True, consistency_weight=0.05, update=False)
    torch.cuda.synchronize()
    for n, b in m.named_buffers():
        assert torch.equal(b, bufs0[n]), n
    assert sum(n.endswith("num_batches_tracked") for n in bufs0) == 8
    for n, p in m.named_parameters():
        if n == "encoder.projection_layer":
            assert p.grad is None
        else:
            assert p.grad is not None and torch.count_nonzero(p.grad).item() > 0, n
    rm = [n for n, _ in m.named_parameters() if n.startswith(("encoder.transformer.0.", "encoder.transformer.2."))]
    assert sum(n.endswith(("rbr_skip.weight", "bn.weight")) for n in rm) == 8
    assert sum(n.endswith("layer_scale") for n in rm) == 4


def test_s0_seeded_steps_bit_identical_and_loss_decreases(cuda):
    m1, opt1, l1 = _s0_steps(81)
    m2, _, l2 = _s0_steps(81)
    print(f"  S0 3 steps: losses {l1}")
    assert l1 == l2 and l1[-1] < l1[0]
    for (n, a), (_, b) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(a, b), n
    assert m1._es3_grad_arena is opt1


def test_s0_direct_arena_grads_equal_autograd_grads_and_accumulation(cuda):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import TextKDLossFunction
    from efficientsam3_b200.stage1.optim import FlatAdamW
    caps = captions()
    teacher = torch.randn(len(caps), 16, 256, generator=torch.Generator().manual_seed(2)).to(cuda)

    def backward(m, text):
        pad, mem, _ = m(text)
        loss, _, _, _ = TextKDLossFunction.apply(mem.transpose(0, 1), teacher, pad, 1.0, 0.0)
        loss.backward()

    m, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=91)
    freeze_bn(m)
    backward(m, caps)
    auto = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    m.zero_grad(set_to_none=True)
    backward(m, caps[::-1])
    auto2 = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    md, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=91)
    freeze_bn(md)
    opt = FlatAdamW(md, lr=1e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    backward(md, caps)
    for n, p in md.named_parameters():
        if n in auto:
            assert torch.equal(p.grad, auto[n]), n
    backward(md, caps[::-1])
    for n, p in md.named_parameters():
        if n in auto:
            r = rel_l2(p.grad.cpu(), (auto[n] + auto2[n]).cpu())
            assert r <= 1e-6, (n, r)
    assert md.encoder.projection_layer.grad is None and opt.flat_grad.numel() > 0


def _epoch_cfg(eval_bn):
    from types import SimpleNamespace as NS
    return NS(TRAIN=NS(ACCUMULATION_STEPS=2, EPOCHS=3, WARMUP_EPOCHS=1, MIN_LR=1e-5, WARMUP_LR=1e-6, CLIP_GRAD=5.0,
                       EVAL_BN_WHEN_TRAINING=eval_bn),
              DISTILL=NS(NUM_EMBED=16, EMBED_DIM=256, MASK_PAD_TOKENS=True, COSINE=2.0, CONSISTENCY_LOSS=0.05))


def test_train_text_one_epoch_s0_frozen_bn_matches_the_steps_it_composes(cuda):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import text_kd_train_step
    from efficientsam3_b200.stage1.optim import FlatAdamW
    from efficientsam3_b200.stage1.train import default_lr_at, lr_for_update, train_text_one_epoch
    cfg = _epoch_cfg(True)
    caps = captions()
    g = np.random.default_rng(0)
    embs = [[(g.standard_normal(16 * 256) * 0.5).astype(np.float16) for _ in caps] for _ in range(4)]
    loader = [[list(caps), [e, list(range(len(caps)))]] for e in embs]
    m1, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=95)
    m2, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=95)
    o1 = FlatAdamW(m1, lr=2e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    o2 = FlatAdamW(m2, lr=2e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    random.seed(7)
    losses = train_text_one_epoch(cfg, m1, loader, o1, epoch=1)
    bns = [b for b in m1.modules() if isinstance(b, nn.modules.batchnorm._BatchNorm)]
    assert len(bns) == 8 and m1.training and not any(b.training for b in bns)
    freeze_bn(m2)
    lr_at = default_lr_at(cfg, o2, len(loader))
    random.seed(7)
    want = []
    for idx, e in enumerate(embs):
        t = torch.from_numpy(np.stack(e)).float().view(len(caps), 16, 256).to(cuda)
        update = (idx + 1) % 2 == 0
        want.append(text_kd_train_step(m2, o2, caps, t, cosine_weight=2.0, mask_pad_tokens=True, consistency_weight=0.05,
                                       clip_grad=5.0, lr=lr_for_update(idx, 1, len(loader), 2, lr_at) if update else None,
                                       accumulation_steps=2, update=update))
    assert [x.item() for x in losses] == [x.item() for x in want]
    for (n, a), (_, b) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(a, b), n
    for (n, a), (_, b) in zip(m1.named_buffers(), m2.named_buffers()):
        assert torch.equal(a, b), n
    m3, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=95)
    o3 = FlatAdamW(m3, lr=2e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    with pytest.raises(NotImplementedError, match=r"RepMixerBlocks.*Call \.eval\(\) first\."):
        train_text_one_epoch(_epoch_cfg(False), m3, loader, o3, epoch=1)


# ------------------------------------------------------------------------------------------------ raise paths
def test_s0_raise_paths(cuda):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.model import build_text_student_model
    s0 = build_text_student_model(_cfg_ns("MobileCLIP-S0", 32)).to(cuda).train()
    msg = r"RepMixerBlocks.*EVAL_BN_WHEN_TRAINING.*Call \.eval\(\) first\."
    with pytest.raises(NotImplementedError, match=msg):
        s0(["a cat"])
    with torch.no_grad(), pytest.raises(NotImplementedError, match=msg):
        s0(["a cat"])
    freeze_bn(s0)
    s0.encoder.transformer[-1].convffn.conv.bn.train()          # one BatchNorm left in train mode: a mixed state
    with pytest.raises(NotImplementedError, match=msg):
        s0(["a cat"])
    freeze_bn(s0)
    with pytest.raises(NotImplementedError, match="strict"):
        with ops.strict_precision():
            s0(["a cat"])
    pad, mem, _ = s0(["a cat", "a dog on a mat"])               # frozen: trains
    mem.sum().backward()
    assert s0.encoder.transformer[0].token_mixer.layer_scale.grad is not None
