"""CPU: the pieces of MobileCLIP-S0 training with batch-statistics BatchNorm that need no GPU -- the reference fixtures
(tests/golden/gen_golden_text_train_s0_bn.py) against the batch-statistics oracle's autograd (tests/oracle_text_bn.py), the
forward fold and backward formulas that csrc/repmixer_bn_train.cu implements (restated in fp64 torch) against fp64 autograd of
the oracle block in train mode, and the opt-in's host-side rules."""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from helpers import load_golden
from oracle_text_bn import running_clones, repmixer_block_bn, text_student_bn
from test_text_train_cpu import build_train_student, fixture_permutations, grad_stats
from test_text_train_s0_cpu import _dw, _dw_t, _dw_taps, oracle_sd, repmixer_block_sd

BN_FIXTURES = ["text_train_s0_bn_ctx16", "text_train_s0_bn_ctx32"]


def s0_bn_oracle_train_grads(g, sd0, m):
    """The reference iteration on the batch-statistics oracle: (loss terms, {name: grad}, running buffers after the iteration)."""
    from test_text_cpu import oracle_cfg
    from test_text_train_cpu import ref_text_loss
    sd = oracle_sd(sd0, m)
    run = running_clones(sd0)
    cfg = oracle_cfg(m)
    ids = torch.from_numpy(g["ids"])
    preds = text_student_bn(sd, ids, cfg, run)[1].transpose(0, 1)
    valid = (ids != 0).float() if int(g["masked"]) else None
    loss, mse, cos = ref_text_loss(preds, torch.from_numpy(g["teacher"]).float(), valid, float(g["cosine"]))
    cons = []
    for pid in g["perm_ids"]:
        q = text_student_bn(sd, torch.from_numpy(pid), cfg, run)[1].transpose(0, 1)
        c = F.mse_loss(preds.mean(1), q.mean(1))
        loss = loss + float(g["consistency"]) * c
        cons.append(c.item())
    loss.backward()
    return [loss.item(), mse.item(), cos.item(), *cons] + [0.0] * (2 - len(cons)), {k: v.grad for k, v in sd.items()}, run


@pytest.mark.parametrize("name", BN_FIXTURES)
def test_s0_bn_fixture_inputs_and_running_stats_moved(name):
    g = load_golden(name)
    m, sd = build_train_student(g)
    caps, perms = fixture_permutations(g)
    assert torch.equal(m.tokenizer(caps, context_length=m.context_length), torch.from_numpy(g["ids"]))
    assert [list(p) for p in perms] == [[str(s) for s in row] for row in g["perm_strings"]]
    names = [str(n) for n in g["bn_names"]]
    assert len(names) == 8 and all(n.startswith(("encoder.transformer.0.", "encoder.transformer.2.")) for n in names)
    forwards = 1 + len(g["perm_ids"])
    assert forwards == (3 if float(g["consistency"]) > 0 else 1)
    for n, (rm, rv), nbt in zip(names, g["running"], g["num_batches_tracked"]):
        assert int(nbt) == int(sd[n + ".num_batches_tracked"]) + forwards, n
        assert not np.array_equal(rm, sd[n + ".running_mean"].numpy()), n


@pytest.mark.parametrize("name", BN_FIXTURES)
def test_s0_bn_fixture_oracle_loss_gradients_and_running_stats(name):
    """The batch-statistics oracle against the reference's plain-.train() iteration: loss terms rtol 1e-5, gradient statistics
    within 1e-4 of each gradient's norm, running buffers within 1e-5 of their scale, num_batches_tracked equal."""
    g = load_golden(name)
    m, sd = build_train_student(g)
    terms, grads, run = s0_bn_oracle_train_grads(g, sd, m)
    for a, b in zip(terms, g["loss"]):
        assert abs(a - b) <= 1e-5 * max(abs(b), 1e-12), (terms, g["loss"].tolist())
    names = [str(n) for n in g["grad_names"]]
    assert names == [n for n, _ in m.named_parameters() if n != "encoder.projection_layer"]
    for n, ref in zip(names, g["grad_stats"]):
        err = np.abs(grad_stats(grads[n]).numpy() - ref).max() / ref[0]
        assert err <= 1e-4, (n, err)
    for n, (rm, rv), nbt in zip([str(n) for n in g["bn_names"]], g["running"], g["num_batches_tracked"]):
        for got, ref in zip(run[n][:2], (rm, rv)):
            err = np.abs(got.numpy() - ref).max() / np.abs(ref).max()
            assert err <= 1e-5, (n, err)
        assert run[n][2] == int(nbt), n


# ------------------------------------------------------------------------------------------------ the kernels' formulas
def _batch_stats(v):
    """Per-channel mean and biased variance over (B, L) of v [B, L, C]."""
    mean = v.mean((0, 1))
    return mean, ((v - mean) ** 2).mean((0, 1))


def repmixer_bn_formula(x, g, sd, p, momentum=0.1, eps=1e-5):
    """The batch-statistics RepMixerBlock as repmixer_bn_train.cu computes it (fp64 torch): the forward fold from batch statistics
    and the sums / apply backward.  x, g [B, L, C] -> (x2, dx, {name: grad}, {BN prefix: (running_mean, running_var)})."""
    tm, f = p + ".token_mixer", p + ".convffn"
    M = x.shape[0] * x.shape[1]
    w_mc = sd[tm + ".mixer.rbr_conv.0.conv.weight"].reshape(-1, 11)
    w_f = sd[f + ".conv.conv.weight"].reshape(-1, 11)
    ls_tm, ls_blk = sd[tm + ".layer_scale"].reshape(-1), sd[p + ".layer_scale"].reshape(-1)
    gam = {k: sd[f"{k}.weight"] for k in (tm + ".mixer.rbr_skip", tm + ".mixer.rbr_conv.0.bn", tm + ".norm.rbr_skip", f + ".conv.bn")}
    bet = {k: sd[f"{k}.bias"] for k in gam}
    ms, mc, ns, bf_ = list(gam)
    W1, b1 = sd[f + ".fc1.weight"].flatten(1), sd[f + ".fc1.bias"]
    W2, b2 = sd[f + ".fc2.weight"].flatten(1), sd[f + ".fc2.bias"]
    running = {}

    def update(k, mean, var):
        running[k] = ((1 - momentum) * sd[k + ".running_mean"] + momentum * mean,
                      (1 - momentum) * sd[k + ".running_var"] + momentum * var * M / (M - 1))
        return 1.0 / torch.sqrt(var + eps)

    # forward: statistics of x and c -> folded token-mixer taps; statistics of f -> folded ConvFFN taps
    c = _dw(x, w_mc)
    mx, vx = _batch_stats(x)
    mcm, vc = _batch_stats(c)
    i_ms, i_mc, i_ns = update(ms, mx, vx), update(mc, mcm, vc), update(ns, mx, vx)
    s_ms, s_mc, s_ns = gam[ms] * i_ms, gam[mc] * i_mc, gam[ns] * i_ns
    wm = w_mc * (ls_tm * s_mc)[:, None]
    wm[:, 5] += 1.0 + ls_tm * (s_ms - s_ns)
    bm = ls_tm * (bet[ms] - mx * s_ms + bet[mc] - mcm * s_mc - (bet[ns] - mx * s_ns))
    x1 = _dw(x, wm) + bm
    fv = _dw(x1, w_f)
    mf, vf = _batch_stats(fv)
    i_f = update(bf_, mf, vf)
    s_f = gam[bf_] * i_f
    u = _dw(x1, w_f * s_f[:, None]) + (bet[bf_] - mf * s_f)
    z = u @ W1.t() + b1
    h = F.gelu(z)
    y = h @ W2.t() + b2
    x2 = x1 + ls_blk * y
    # backward
    gr = {}
    gr[p + ".layer_scale"] = (g * y).sum((0, 1)).reshape(-1, 1, 1)
    dy = ls_blk * g
    gr[f + ".fc2.bias"] = dy.sum((0, 1))
    gr[f + ".fc2.weight"] = torch.einsum("bln,blk->nk", dy, h).reshape(W2.shape[0], -1, 1, 1)
    dz = (dy @ W2) * (0.5 * (1 + torch.erf(z / math.sqrt(2))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi))
    gr[f + ".fc1.bias"] = dz.sum((0, 1))
    gr[f + ".fc1.weight"] = torch.einsum("bln,blk->nk", dz, u).reshape(W1.shape[0], -1, 1, 1)
    du = dz @ W1
    # ConvFFN: sums pass, then the corrected df and the taps on it
    fh = (fv - mf) * i_f
    S0, S1 = du.sum((0, 1)), (du * fh).sum((0, 1))
    gr[bf_ + ".bias"], gr[bf_ + ".weight"] = S0, S1
    df = s_f * (du - S0 / M - fh * S1 / M)
    gr[f + ".conv.conv.weight"] = _dw_taps(df, x1).reshape(-1, 1, 1, 11)
    e = g + _dw_t(df, w_f)
    # token mixer: sums pass (e', e' chat, e' (x - mean)), then dc, dx, the taps and the layer scale
    ep = ls_tm * e
    chat, xc = (c - mcm) * i_mc, x - mx
    T0, T1, T2 = ep.sum((0, 1)), (ep * chat).sum((0, 1)), (ep * xc).sum((0, 1))
    gr[ms + ".bias"], gr[mc + ".bias"], gr[ns + ".bias"] = T0, T0, -T0
    gr[mc + ".weight"], gr[ms + ".weight"], gr[ns + ".weight"] = T1, i_ms * T2, -i_ns * T2
    r = (gam[ms] * i_ms - gam[ns] * i_ns) * xc + gam[mc] * chat + bet[ms] + bet[mc] - bet[ns]
    gr[tm + ".layer_scale"] = (e * r).sum((0, 1)).reshape(-1, 1, 1)
    dc = s_mc * (ep - T0 / M - chat * T1 / M)
    gr[tm + ".mixer.rbr_conv.0.conv.weight"] = _dw_taps(dc, x).reshape(-1, 1, 1, 11)
    dx = e + (s_ms - s_ns) * (ep - T0 / M) - (s_ms * i_ms ** 2 - s_ns * i_ns ** 2) * xc * T2 / M + _dw_t(dc, w_mc)
    return x2, dx, gr, running


@pytest.mark.parametrize("B,L", [(2, 1), (3, 11), (3, 77), (2, 128)])
def test_repmixer_bn_formulas_match_oracle_autograd(B, L):
    C = 32
    sd0 = repmixer_block_sd(C, 80 + L)
    g_ = torch.Generator().manual_seed(L)
    x = torch.randn(B, L, C, generator=g_, dtype=torch.float64) * 1.5 + 0.3
    gout = torch.randn(B, L, C, generator=g_, dtype=torch.float64)
    sd = {k: v.clone().requires_grad_(not k.endswith(("running_mean", "running_var"))) for k, v in sd0.items()}
    run = running_clones(sd0)
    xr = x.clone().requires_grad_(True)
    out = repmixer_block_bn(xr, sd, "blk", run)
    out.backward(gout)
    x2, dx, gr, running = repmixer_bn_formula(x, gout, sd0, "blk")
    assert torch.allclose(x2, out.detach(), rtol=1e-10, atol=1e-12 * out.abs().max().item())
    assert torch.allclose(dx, xr.grad, rtol=1e-8, atol=1e-10 * xr.grad.abs().max().item())
    names = [k for k, v in sd.items() if v.grad is not None]
    assert sorted(names) == sorted(gr), sorted(set(names) ^ set(gr))
    for k in names:
        ref = sd[k].grad
        assert gr[k].shape == ref.shape, k
        assert torch.allclose(gr[k], ref, rtol=1e-8, atol=1e-10 * max(ref.abs().max().item(), 1e-30)), k
    for k, (rm, rv) in running.items():
        assert torch.allclose(rm, run[k][0], rtol=1e-12, atol=1e-14) and torch.allclose(rv, run[k][1], rtol=1e-12, atol=1e-14), k
        assert run[k][2] == 1


# ------------------------------------------------------------------------------------------------ the opt-in's host rules
def _s0_cpu():
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.model import text_student_cfg
    cfg = text_student_cfg("MobileCLIP-S0")
    cfg.update(n_transformer_layers=1, context_length=16)
    return TextStudentEncoder(cfg=cfg, context_length=16, output_dim=256)


def test_batch_stat_flag_is_not_state_and_raise_rules_fire():
    from efficientsam3_b200.backbones.mobile_clip import check_trainable
    m = _s0_cpu()
    keys = list(m.state_dict())
    assert m.enable_batch_stat_bn() is m and m.encoder.batch_stat_bn
    assert list(m.state_dict()) == keys and not any("batch_stat" in k for k in keys)
    m.train()
    assert m.encoder.batch_stat_active()
    with pytest.raises(RuntimeError, match="CUDA device"):          # every BN rule passes; the CPU module is then rejected
        check_trainable(m, m.encoder, "S0")
    m.encoder.transformer[-1].convffn.conv.bn.eval()                # a mixed state
    with pytest.raises(NotImplementedError, match="mixed"):
        check_trainable(m, m.encoder, "S0")
    m.train()
    m.encoder.transformer[0].token_mixer.norm.rbr_skip.momentum = None
    with pytest.raises(NotImplementedError, match="momentum=None"):
        check_trainable(m, m.encoder, "S0")
    m = _s0_cpu().enable_batch_stat_bn().train()
    m.encoder.transformer[0].convffn.conv.bn.track_running_stats = False
    with pytest.raises(NotImplementedError, match="track_running_stats"):
        check_trainable(m, m.encoder, "S0")
    m = _s0_cpu().enable_batch_stat_bn().train()
    for mod in m.modules():                                         # every BN in eval: the frozen path, flag or not
        if isinstance(mod, nn.BatchNorm2d):
            mod.eval()
    assert not m.encoder.batch_stat_active()
    m.enable_batch_stat_bn(False).train()
    with pytest.raises(NotImplementedError, match=r"RepMixerBlocks.*EVAL_BN_WHEN_TRAINING.*enable_batch_stat_bn\(\).*"
                                                  r"Call \.eval\(\) first\."):
        check_trainable(m, m.encoder, "S0")
