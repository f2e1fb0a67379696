"""GPU: training MobileCLIP-S0 natively with batch-statistics BatchNorm (TextStudentEncoder.enable_batch_stat_bn) -- the kernels of
csrc/repmixer_bn_train.cu against fp64 torch autograd and F.batch_norm, whole training graphs against the batch-statistics oracle's
autograd (tests/oracle_text_bn.py, with its bf16-autocast run as the precision yardstick), the reference's plain-.train() iteration
(tests/golden/gen_golden_text_train_s0_bn.py) end to end from strings, the train-mode forward under no_grad and the eval path after
it, the optimiser interplay and the raise paths."""
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
from oracle_text_bn import running_clones, text_student_bn
from test_text_cpu import oracle_cfg
from test_text_gpu import captions, check_memory
from test_text_train_cpu import build_train_student, fixture_permutations, grad_stats, ref_text_loss
from test_text_train_gpu import _all_grad_rel, _cfg_ns, _permuted, _student
from test_text_train_s0_cpu import oracle_sd
from test_text_train_s0_gpu import _acc, _check, _leaves, _rows, _t, freeze_bn

pytestmark = pytest.mark.gpu

BN = ["token_mixer.mixer.rbr_skip", "token_mixer.mixer.rbr_conv.0.bn", "token_mixer.norm.rbr_skip", "convffn.conv.bn"]


def bn_train(m):
    """Opt in and put everything in train mode, as train_text_one_epoch does with TRAIN.EVAL_BN_WHEN_TRAINING False."""
    return m.enable_batch_stat_bn().train()


# ------------------------------------------------------------------------------------------------ kernels vs fp64 autograd
def _bt(t, sd, p):
    """nn.BatchNorm2d in train mode without running buffers (fp64 reference)."""
    return F.batch_norm(t, None, None, sd[p + ".weight"], sd[p + ".bias"], True, 0.0, 1e-5)


def _stats64(t):
    m = t.mean((0, 2, 3))
    return m, t.var((0, 2, 3), unbiased=False)


@pytest.mark.parametrize("C", [32, 512])
@pytest.mark.parametrize("L", [1, 4, 11, 16, 32, 77, 128])
@pytest.mark.parametrize("B", [1, 3, 64])
def test_repmixer_bn_kernels(cuda, B, L, C):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.backbones.mobile_clip import RepMixerBlock, repmixer_bn_pack, repmixer_bns
    if B * L < 2:
        pytest.skip("batch statistics need B*L >= 2 (host rejection: test_repmixer_bn_host_checks)")
    blk = RepMixerBlock(dim=C)
    sd0 = fill_state_dict(blk.state_dict(), 11 * L + C + B)
    blk.load_state_dict(sd0)
    blk = blk.to(cuda).train()
    sd = {k: v.to(cuda, torch.float64) for k, v in sd0.items() if not k.endswith("num_batches_tracked")}
    p, bns = repmixer_bn_pack(blk), repmixer_bns(blk)
    run0 = [(bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()) for bn in bns]
    gen = torch.Generator().manual_seed(B * 1000 + L * 10 + C)
    offset = 100.0 if (B, C) == (3, 32) else 0.0            # |mean| >> std: the shifted statistics
    # the tap gradients sum d x with sum d = 0 under batch statistics: with |mean| = 100 std that sum cancels by ~100, and fp32
    # keeps about two fewer digits of it (any fp32 implementation does; the statistics are what the offset case checks)
    tap_tol = 2e-3 if offset == 0.0 else 2e-1
    x = (torch.randn(B * L, C, generator=gen) + offset).to(cuda)
    g, du, e = (torch.randn(B * L, C, generator=gen).to(cuda) for _ in range(3))
    bn_leaf = [f"{n}.{w}" for n in BN[:3] for w in ("weight", "bias")]

    def run():
        for bn, (rm, rv, nbt) in zip(bns, run0):
            bn.running_mean.copy_(rm); bn.running_var.copy_(rv); bn.num_batches_tracked.copy_(nbt)
        o = {}
        o["x1"], o["u"], o["fold"], o["stats"] = ops.repmixer_bn_fwd(x, B, L, p["taps"], p["aff"], bns)
        for i, bn in enumerate(bns):
            o[f"rm{i}"], o[f"rv{i}"], o[f"nbt{i}"] = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()
        o["dwf"], o["dgf"], o["dbf"] = _acc((C, 1, 1, 11), cuda), _acc((C,), cuda), _acc((C,), cuda)
        o["e"] = ops.repmixer_bn_ffn_bwd(o["x1"], du, g, p["taps"], p["aff"], o["stats"], B, L, dtaps=o["dwf"], dgamma=o["dgf"],
                                         dbeta=o["dbf"])
        o["dwm"], o["dls_tm"] = _acc((C, 1, 1, 11), cuda), _acc((C, 1, 1), cuda)
        dbn = [_acc((C,), cuda) for _ in range(6)]
        o["dx"], o["dxb"] = ops.repmixer_bn_tm_bwd(x, e, p["taps"], p["aff"], o["stats"], B, L, dtaps=o["dwm"], dls=o["dls_tm"],
                                                   dbn=dbn, want_bf16=True)
        for n, t in zip(bn_leaf, dbn):
            o[n] = t
        return o

    n0 = ops.launch_count
    got = run()
    assert ops.launch_count - n0 == 5 + 4 + 4
    # forward: batch statistics, running buffers, folded taps, x1 and u
    tm, f = "token_mixer", "convffn"
    t = _t(x, B, L).detach()
    c = OT._dw(t, sd[tm + ".mixer.rbr_conv.0.conv.weight"])
    t1 = _t(got["x1"], B, L).detach()
    fv = OT._dw(t1, sd[f + ".conv.conv.weight"])
    st = got["stats"].double()
    for i, v in enumerate((t, c, t, fv)):
        mean, var = _stats64(v)
        std = var.sqrt()
        assert ((st[2 * i] - mean).abs() / std).max().item() <= 1e-4, (BN[i], "mean")
        assert ((st[2 * i + 1] * (var + 1e-5).sqrt() - 1).abs()).max().item() <= 1e-4, (BN[i], "invstd")
        rm, rv = run0[i][0].double().clone(), run0[i][1].double().clone()
        F.batch_norm(v, rm, rv, None, None, True, 0.1, 1e-5)
        _check(got[f"rm{i}"], rm, 1e-5, f"{BN[i]} running_mean")
        _check(got[f"rv{i}"], rv, 1e-5, f"{BN[i]} running_var")
        assert int(got[f"nbt{i}"]) == int(run0[i][2]) + 1
    ref_x1 = t + sd[tm + ".layer_scale"] * (_bt(t, sd, tm + ".mixer.rbr_skip") + _bt(c, sd, tm + ".mixer.rbr_conv.0.bn")
                                            - _bt(t, sd, tm + ".norm.rbr_skip"))
    _check(got["x1"], _rows(ref_x1), 1e-5, "x1")
    _check(got["u"].float(), _rows(_bt(fv, sd, f + ".conv.bn")), 1e-2, "u")
    # the fold, restated from the fp64 statistics
    ls = sd[tm + ".layer_scale"].reshape(-1)
    inv = [1.0 / (_stats64(v)[1] + 1e-5).sqrt() for v in (t, c, t, fv)]
    mean = [_stats64(v)[0] for v in (t, c, t, fv)]
    s = [sd[f"{n}.weight"] * i for n, i in zip(BN, inv)]
    b = [sd[f"{n}.bias"] - m_ * s_ for n, m_, s_ in zip(BN, mean, s)]
    wm = sd[tm + ".mixer.rbr_conv.0.conv.weight"].reshape(C, 11).t() * (ls * s[1])
    wm[5] += 1.0 + ls * (s[0] - s[2])
    _check(got["fold"][:11], wm, 1e-4, "wm")
    _check(got["fold"][11], ls * (b[0] + b[1] - b[2]), 1e-4, "bm")
    _check(got["fold"][12:23], sd[f + ".conv.conv.weight"].reshape(C, 11).t() * s[3], 1e-4, "wf")
    _check(got["fold"][23], b[3], 1e-4, "bf")
    # ConvFFN.conv + BN_f (batch statistics of dw(x1)): e = d/dx1 of (sum du * BN_f(dw(x1)) + sum g * x1)
    lv = _leaves(sd, [f + ".conv.conv.weight", f + ".conv.bn.weight", f + ".conv.bn.bias"])
    t1 = t1.clone().requires_grad_(True)
    uu = _bt(OT._dw(t1, lv[f + ".conv.conv.weight"]), {**sd, **lv}, f + ".conv.bn")
    ((uu * _t(du, B, L).detach()).sum() + (t1 * _t(g, B, L).detach()).sum()).backward()
    _check(got["e"], _rows(t1.grad), 2e-3, "e")
    _check(got["dwf"] - 0.25, lv[f + ".conv.conv.weight"].grad, tap_tol, "d w_f")
    _check(got["dgf"] - 0.25, lv[f + ".conv.bn.weight"].grad, 2e-3, "d gamma_f")
    _check(got["dbf"] - 0.25, lv[f + ".conv.bn.bias"].grad, 2e-3, "d beta_f")
    # token mixer: dx = d/dx of sum e * (x + ls_tm (BN_ms(x) + BN_mc(dw(x)) - BN_ns(x))), batch statistics
    lv = _leaves(sd, [tm + ".mixer.rbr_conv.0.conv.weight", tm + ".layer_scale", *bn_leaf])
    s_ = {**sd, **lv}
    tx = _t(x, B, L)
    out = tx + s_[tm + ".layer_scale"] * (_bt(tx, s_, tm + ".mixer.rbr_skip")
                                          + _bt(OT._dw(tx, s_[tm + ".mixer.rbr_conv.0.conv.weight"]), s_, tm + ".mixer.rbr_conv.0.bn")
                                          - _bt(tx, s_, tm + ".norm.rbr_skip"))
    (out * _t(e, B, L).detach()).sum().backward()
    _check(got["dx"], _rows(tx.grad), 2e-3, "dx")
    _check(got["dxb"], _rows(tx.grad), 1e-2, "dx bf16")
    assert torch.equal(got["dxb"], got["dx"].to(torch.bfloat16))
    _check(got["dwm"] - 0.25, lv[tm + ".mixer.rbr_conv.0.conv.weight"].grad, tap_tol, "d w_mc")
    _check(got["dls_tm"] - 0.25, lv[tm + ".layer_scale"].grad, 2e-3, "d ls_tm")
    for n in bn_leaf:
        _check(got[n] - 0.25, lv[n].grad, 2e-3, n)
    again = run()                                                    # fixed-order reductions: bit-identical
    for k in got:
        assert torch.equal(got[k], again[k]), k


def test_repmixer_bn_host_checks(cuda):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.backbones.mobile_clip import RepMixerBlock, repmixer_bns
    n0 = ops.launch_count
    for B, L, C in ((1, 1, 32), (1, 129, 32), (2, 4, 48)):
        bns = repmixer_bns(RepMixerBlock(dim=C).to(cuda).train())
        x = torch.zeros(B * L, C, device=cuda)
        taps, aff, stats = torch.zeros(2, 11, C, device=cuda), torch.zeros(9, C, device=cuda), torch.zeros(8, C, device=cuda)
        match = "more than 1 value" if B * L == 1 else "1..128" if L > 128 else "multiple of 32"
        with pytest.raises(ValueError, match=match):
            ops.repmixer_bn_fwd(x, B, L, taps, aff, bns)
        with pytest.raises(ValueError, match=match):
            ops.repmixer_bn_ffn_bwd(x, x, x, taps, aff, stats, B, L)
        with pytest.raises(ValueError, match=match):
            ops.repmixer_bn_tm_bwd(x, x, taps, aff, stats, B, L)
    assert ops.launch_count == n0


# ------------------------------------------------------------------------------------------------ whole graphs vs the oracle
def _oracle(sd0, m, ids_list, dev, autocast=None, teacher=None, valid=None, w_cos=1.0, w_con=0.0):
    """The batch-statistics oracle on the forwards ids_list (the captions, then the permutations), with the loss and its backward
    when a teacher is given: (loss | None, {name: grad} | None, running buffers after the forwards)."""
    sd = oracle_sd(sd0, m, dev)
    run = {k: [v[0].to(dev), v[1].to(dev), v[2]] for k, v in running_clones(sd0).items()}
    cfg = oracle_cfg(m)
    ctx = torch.autocast("cuda", dtype=autocast) if autocast is not None else contextlib.nullcontext()
    with ctx:
        outs = [text_student_bn(sd, ids.to(dev), cfg, run)[1].transpose(0, 1) for ids in ids_list]
    if teacher is None:
        return None, None, run
    preds, perms = outs[0].float(), [q.float() for q in outs[1:]]
    loss, _, _ = ref_text_loss(preds, teacher, valid, w_cos)
    for q in perms:
        loss = loss + w_con * F.mse_loss(preds.mean(1), q.mean(1))
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in sd.items()}, run


def _running_err(m, run, block):
    """Largest max-error-over-scale of the running buffers of one RepMixerBlock (transformer index) against an oracle run."""
    bufs = dict(m.named_buffers())
    err = 0.0
    for n in BN:
        k = f"encoder.transformer.{block}.{n}"
        for j, s in enumerate(("running_mean", "running_var")):
            err = max(err, max_err_over_scale(bufs[f"{k}.{s}"].double().cpu(), torch.as_tensor(run[k][j]).double().cpu()))
        assert int(bufs[f"{k}.num_batches_tracked"]) == run[k][2], k
    return err


def _compare_s0_bn(m, sd, caps, masked, w_con, dev, label):
    from efficientsam3_b200.stage1.losses import TextKDLossFunction
    w_cos = 1.0
    ids = m.tokenizer(caps, context_length=m.context_length)
    perm_caps = _permuted(caps, 5) if w_con > 0 else []
    ids_list = [ids] + [m.tokenizer(pc, context_length=m.context_length) for pc in perm_caps]
    teacher = torch.randn(len(caps), m.context_length, 256, generator=torch.Generator().manual_seed(9)).to(dev)
    valid = (ids != 0).float().to(dev) if masked else None
    bn_train(m)
    m.zero_grad(set_to_none=True)
    pad, mem, _ = m(caps)
    perms = [m(pc)[1].transpose(0, 1) for pc in perm_caps]
    loss_n, _, _, _ = TextKDLossFunction.apply(mem.transpose(0, 1), teacher, pad if masked else None, w_cos, w_con, *perms)
    loss_n.backward()
    got = {n: p.grad for n, p in m.named_parameters()}
    loss_r, ref, run = _oracle(sd, m, ids_list, dev, None, teacher, valid, w_cos, w_con)
    _, ref_bf, run_bf = _oracle(sd, m, ids_list, dev, torch.bfloat16, teacher, valid, w_cos, w_con)
    assert got["encoder.projection_layer"] is None
    names = [n for n, _ in m.named_parameters() if n != "encoder.projection_layer"]
    rel = _all_grad_rel(got, ref, names)
    d_bf16 = _all_grad_rel(ref_bf, ref, names)
    last = len(m.encoder.transformer) - 1
    e0, e_last = _running_err(m, run, 0), _running_err(m, run, last)
    e_bf = max(_all_err(run_bf, run, last), 1e-4)
    print(f"  {label}: loss native {loss_n.item():.6f} oracle {loss_r.item():.6f}; all-gradient rel-L2 native {rel:.3e}, "
          f"torch.autocast(bf16) oracle {d_bf16:.3e}; running buffers block 0 {e0:.2e}, last block {e_last:.2e} (bf16 oracle "
          f"{e_bf:.2e})")
    assert abs(loss_n.item() - loss_r.item()) <= 2e-2 * abs(loss_r.item())
    assert rel <= 5e-2 and rel <= 3 * d_bf16, (rel, d_bf16)
    assert e0 <= 1e-4 and e_last <= 3 * e_bf, (e0, e_last, e_bf)
    return got


def _all_err(run_a, run_b, block):
    err = 0.0
    for n in BN:
        k = f"encoder.transformer.{block}.{n}"
        for j in range(2):
            err = max(err, max_err_over_scale(run_a[k][j].double().cpu(), run_b[k][j].double().cpu()))
    return err


def test_s0_bn_depth1_masked_consistency(cuda):
    m, sd = _student("MobileCLIP-S0", cuda, layers=1, ctx=32, seed=161)
    _compare_s0_bn(m, sd, captions(), masked=True, w_con=0.5, dev=cuda, label="S0-shaped depth 1, batch-stat BN, masked + consistency")


def test_s0_bn_full_depth_table77_at_32(cuda):
    m, sd = _student("MobileCLIP-S0", cuda, ctx=32, table=77, seed=162)
    got = _compare_s0_bn(m, sd, captions(), masked=True, w_con=0.0, dev=cuda, label="MobileCLIP-S0 full depth, batch-stat BN")
    assert got["encoder.positional_embedding.pos_embed.pos_embed"].abs().sum().item() > 0


# ------------------------------------------------------------------------------------------------ reference fixtures
@pytest.mark.parametrize("name", ["text_train_s0_bn_ctx16", "text_train_s0_bn_ctx32"])
def test_s0_bn_train_fixture_end_to_end_from_strings(cuda, name):
    """The reference's plain-.train() iteration natively from strings: loss terms, every parameter's gradient statistics,
    num_batches_tracked, and the running buffers (block 0 sees the exact fp32 embedding stream; the last block is held to the
    bf16-autocast oracle's distance)."""
    from efficientsam3_b200.stage1.losses import TextKDLossFunction
    g = load_golden(name)
    m, sd0 = build_train_student(g)
    m = bn_train(m.to(cuda))
    caps, perms = fixture_permutations(g)
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
    assert r <= 5e-2, r
    assert params["encoder.projection_layer"].grad is None
    ref = {str(n): [torch.from_numpy(rm), torch.from_numpy(rv), int(nbt)]
           for n, (rm, rv), nbt in zip(g["bn_names"], g["running"], g["num_batches_tracked"])}
    ids_list = [torch.from_numpy(g["ids"])] + [torch.from_numpy(p) for p in g["perm_ids"]]
    _, _, run_bf = _oracle(sd0, m, ids_list, cuda, torch.bfloat16)
    last = len(m.encoder.transformer) - 1
    e0, e_last = _running_err(m, ref, 0), _running_err(m, ref, last)
    e_bf = max(_all_err(run_bf, ref, last), 1e-4)
    print(f"  {name}: loss native {got_terms[0]:.6f} reference {g['loss'][0]:.6f}; gradient statistics rel-L2 {r:.3e}; running "
          f"buffers block 0 {e0:.2e}, last block {e_last:.2e} (bf16 oracle {e_bf:.2e})")
    assert e0 <= 1e-4 and e_last <= 3 * e_bf, (e0, e_last, e_bf)


# ------------------------------------------------------------------------------------------------ no_grad, then eval
def test_s0_bn_no_grad_forward_then_eval_sees_new_buffers(cuda):
    m, sd0 = _student("MobileCLIP-S0", cuda, layers=1, ctx=32, seed=171)
    caps = captions()
    ids = m.tokenizer(caps, context_length=32)
    cfg = oracle_cfg(m)
    m.eval()
    with torch.no_grad():
        m(caps)                                                   # an eval plan folded from the loaded running statistics
    freeze_bn(m)
    m(caps)[1].sum().backward()                                   # and a frozen-BN train fold
    bn_train(m)
    bufs0 = {n: b.clone() for n, b in m.named_buffers()}
    with torch.no_grad():
        _, mem, _ = m(caps)
    assert mem.grad_fn is None
    sd = oracle_sd(sd0, m, cuda)
    run = {k: [v[0].to(cuda), v[1].to(cuda), v[2]] for k, v in running_clones(sd0).items()}
    with torch.no_grad():
        ref = text_student_bn(sd, ids.to(cuda), cfg, run)[1]
    check_memory(mem, ref.cpu())
    for n, b in m.named_buffers():
        if n.endswith("num_batches_tracked"):
            assert int(b) == int(bufs0[n]) + 1, n                 # exactly one update per forward
    assert _running_err(m, run, 0) <= 1e-4
    # .eval() on the updated buffers: the cached folds were dropped
    sd_new = {k: v.to(cuda) for k, v in m.state_dict().items()}
    m.eval()
    with torch.no_grad():
        _, mem_e, _ = m(caps)
        ref_e = OT.text_student(sd_new, ids.to(cuda), cfg)[1]
    check_memory(mem_e, ref_e.cpu())
    freeze_bn(m)
    _, mem_f, _ = m(caps)
    check_memory(mem_f.detach(), ref_e.cpu())


# ------------------------------------------------------------------------------------------------ optimiser interplay
def _s0_bn_steps(seed, n=3, dev="cuda"):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import text_kd_train_step
    from efficientsam3_b200.stage1.optim import FlatAdamW
    m, _ = _student("MobileCLIP-S0", dev, layers=1, ctx=16, seed=seed)
    bn_train(m)
    opt = FlatAdamW(m, lr=1e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    caps = captions()
    teacher = torch.randn(len(caps), 16, 256, generator=torch.Generator().manual_seed(seed)).to(dev)
    random.seed(seed)
    losses = [text_kd_train_step(m, opt, caps, teacher, cosine_weight=1.0, mask_pad_tokens=True, consistency_weight=0.5,
                                 clip_grad=5.0, lr=1e-3).item() for _ in range(n)]
    return m, opt, losses


def test_s0_bn_step_moves_running_stats_and_reaches_every_parameter(cuda):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import text_kd_train_step
    from efficientsam3_b200.stage1.optim import FlatAdamW
    m, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=181)
    bn_train(m)
    bufs0 = {n: b.clone() for n, b in m.named_buffers()}
    opt = FlatAdamW(m, lr=1e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    caps = captions()
    teacher = torch.randn(len(caps), 16, 256, generator=torch.Generator().manual_seed(3)).to(cuda)
    random.seed(3)
    text_kd_train_step(m, opt, caps, teacher, cosine_weight=2.0, mask_pad_tokens=True, consistency_weight=0.05, update=False)
    torch.cuda.synchronize()
    for n, b in m.named_buffers():
        if n.endswith("num_batches_tracked"):
            assert int(b) == int(bufs0[n]) + 3, n                 # three forwards in the iteration
        else:
            assert not torch.equal(b, bufs0[n]), n
    for n, p in m.named_parameters():
        if n == "encoder.projection_layer":
            assert p.grad is None
        else:
            assert p.grad is not None and torch.count_nonzero(p.grad).item() > 0, n


def test_s0_bn_seeded_steps_bit_identical_and_loss_decreases(cuda):
    m1, opt1, l1 = _s0_bn_steps(191)
    m2, _, l2 = _s0_bn_steps(191)
    print(f"  S0 batch-stat BN, 3 steps: losses {l1}")
    assert l1 == l2 and l1[-1] < l1[0]
    for (n, a), (_, b) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(a, b), n
    for (n, a), (_, b) in zip(m1.named_buffers(), m2.named_buffers()):
        assert torch.equal(a, b), n
    assert m1._es3_grad_arena is opt1


def test_s0_bn_direct_arena_grads_equal_autograd_grads_and_accumulation(cuda):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import TextKDLossFunction
    from efficientsam3_b200.stage1.optim import FlatAdamW
    caps = captions()
    teacher = torch.randn(len(caps), 16, 256, generator=torch.Generator().manual_seed(2)).to(cuda)

    def backward(m, text):
        pad, mem, _ = m(text)
        loss, _, _, _ = TextKDLossFunction.apply(mem.transpose(0, 1), teacher, pad, 1.0, 0.0)
        loss.backward()

    m, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=193)
    bn_train(m)
    backward(m, caps)
    auto = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    m.zero_grad(set_to_none=True)
    backward(m, caps[::-1])
    auto2 = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    md, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=193)
    bn_train(md)
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
    for (n, a), (_, b) in zip(m.named_buffers(), md.named_buffers()):
        assert torch.equal(a, b), n
    assert md.encoder.projection_layer.grad is None and opt.flat_grad.numel() > 0


def test_train_text_one_epoch_s0_batch_stat_bn_matches_the_steps_it_composes(cuda):
    from types import SimpleNamespace as NS
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import text_kd_train_step
    from efficientsam3_b200.stage1.optim import FlatAdamW
    from efficientsam3_b200.stage1.train import default_lr_at, lr_for_update, train_text_one_epoch
    cfg = NS(TRAIN=NS(ACCUMULATION_STEPS=2, EPOCHS=3, WARMUP_EPOCHS=1, MIN_LR=1e-5, WARMUP_LR=1e-6, CLIP_GRAD=5.0,
                      EVAL_BN_WHEN_TRAINING=False),
             DISTILL=NS(NUM_EMBED=16, EMBED_DIM=256, MASK_PAD_TOKENS=True, COSINE=2.0, CONSISTENCY_LOSS=0.05))
    caps = captions()
    g = np.random.default_rng(0)
    embs = [[(g.standard_normal(16 * 256) * 0.5).astype(np.float16) for _ in caps] for _ in range(4)]
    loader = [[list(caps), [e, list(range(len(caps)))]] for e in embs]
    m1, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=195)
    m2, _ = _student("MobileCLIP-S0", cuda, layers=1, ctx=16, seed=195)
    m1.enable_batch_stat_bn()
    o1 = FlatAdamW(m1, lr=2e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    o2 = FlatAdamW(m2, lr=2e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    random.seed(7)
    losses = train_text_one_epoch(cfg, m1, loader, o1, epoch=1)
    bns = [b for b in m1.modules() if isinstance(b, nn.modules.batchnorm._BatchNorm)]
    assert len(bns) == 8 and all(b.training for b in bns) and all(int(b.num_batches_tracked) == 12 for b in bns)
    bn_train(m2)
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


# ------------------------------------------------------------------------------------------------ raise paths
def test_s0_bn_raise_paths(cuda):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.model import build_text_student_model
    s0 = bn_train(build_text_student_model(_cfg_ns("MobileCLIP-S0", 32)).to(cuda))
    n0 = ops.launch_count
    s0.encoder.transformer[-1].convffn.conv.bn.eval()              # a mixed state
    with pytest.raises(NotImplementedError, match="mixed"):
        s0(["a cat"])
    s0.train()
    s0.encoder.transformer[0].token_mixer.mixer.rbr_skip.momentum = None
    with pytest.raises(NotImplementedError, match="momentum=None"):
        s0(["a cat"])
    s0.encoder.transformer[0].token_mixer.mixer.rbr_skip.momentum = 0.1
    s0.encoder.transformer[0].convffn.conv.bn.track_running_stats = False
    with pytest.raises(NotImplementedError, match="track_running_stats"):
        s0(["a cat"])
    s0.encoder.transformer[0].convffn.conv.bn.track_running_stats = True
    with pytest.raises(NotImplementedError, match="strict"):
        with ops.strict_precision():
            s0(["a cat"])
    one = torch.tensor([[5]])
    with pytest.raises(ValueError, match="more than 1 value"):
        s0(one)
    with torch.no_grad(), pytest.raises(ValueError, match="more than 1 value"):
        s0(one)
    assert ops.launch_count == n0
    pad, mem, _ = s0(["a cat", "a dog on a mat"])                   # batch statistics: trains
    mem.sum().backward()
    assert s0.encoder.transformer[0].token_mixer.layer_scale.grad is not None
