"""CPU: the pieces of MobileCLIP-S0 training with frozen BatchNorm that need no GPU -- the reference fixtures
(tests/golden/gen_golden_text_train_s0.py) against the oracle's autograd, the RepMixerBlock backward formulas that
csrc/repmixer_bwd.cu implements (restated in fp64 torch) against autograd of oracle.text.repmixer_block, and FlatAdamW's
weight-decay groups on S0's parameters."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden
from test_text_train_cpu import build_train_student, fixture_permutations, grad_stats

S0_FIXTURES = ["text_train_s0_ctx16", "text_train_s0_ctx32"]


def oracle_sd(sd0, m, device="cpu", dtype=torch.float32):
    """The state dict as oracle leaves: parameters require grad, BatchNorm buffers (batch_norm takes no gradient for them) do not."""
    params = {n for n, _ in m.named_parameters()}
    return {k: v.detach().clone().to(device, dtype).requires_grad_(k in params) for k, v in sd0.items()}


def s0_oracle_train_grads(g, sd0, m):
    """oracle_train_grads (tests/test_text_train_cpu.py) on a state dict with BatchNorm buffers: (loss terms, {name: grad})."""
    from oracle import text as OT
    from test_text_cpu import oracle_cfg
    from test_text_train_cpu import ref_text_loss
    sd = oracle_sd(sd0, m)
    cfg = oracle_cfg(m)
    ids = torch.from_numpy(g["ids"])
    preds = OT.text_student(sd, ids, cfg)[1].transpose(0, 1)
    valid = (ids != 0).float() if int(g["masked"]) else None
    loss, mse, cos = ref_text_loss(preds, torch.from_numpy(g["teacher"]).float(), valid, float(g["cosine"]))
    cons = []
    for pid in g["perm_ids"]:
        q = OT.text_student(sd, torch.from_numpy(pid), cfg)[1].transpose(0, 1)
        c = F.mse_loss(preds.mean(1), q.mean(1))
        loss = loss + float(g["consistency"]) * c
        cons.append(c.item())
    loss.backward()
    return [loss.item(), mse.item(), cos.item(), *cons] + [0.0] * (2 - len(cons)), {k: v.grad for k, v in sd.items()}


@pytest.mark.parametrize("name", S0_FIXTURES)
def test_s0_fixture_ids_permutations_keys_and_running_stats(name):
    from test_text_cpu import sig
    g = load_golden(name)
    m, sd = build_train_student(g)
    assert sig(m.state_dict()) == [str(k) for k in g["keys"]]
    caps, perms = fixture_permutations(g)
    assert torch.equal(m.tokenizer(caps, context_length=m.context_length), torch.from_numpy(g["ids"]))
    assert torch.equal(torch.from_numpy(g["pad"]), torch.from_numpy(g["ids"]) == 0)
    assert [list(p) for p in perms] == [[str(s) for s in row] for row in g["perm_strings"]]
    for p, pid in zip(perms, g["perm_ids"]):
        assert torch.equal(m.tokenizer(p, context_length=m.context_length), torch.from_numpy(pid))
    # the trunk is RepMixerBlock, TransformerEncoder, RepMixerBlock: 8 BatchNorms, frozen by the reference's set_bn_state
    names = [str(n) for n in g["bn_names"]]
    assert len(names) == 8 and all(n.startswith(("encoder.transformer.0.", "encoder.transformer.2.")) for n in names)
    for n, (rm, rv), nbt in zip(names, g["running"], g["num_batches_tracked"]):
        assert np.array_equal(rm, sd[n + ".running_mean"].numpy()) and np.array_equal(rv, sd[n + ".running_var"].numpy()), n
        assert int(nbt) == int(sd[n + ".num_batches_tracked"]), n


@pytest.mark.parametrize("name", S0_FIXTURES)
def test_s0_fixture_oracle_loss_and_gradients(name):
    """oracle/text.py (running-statistics BatchNorm) against the reference's frozen-BN train-mode iteration: loss terms rtol 1e-5,
    every gradient statistic within 1e-4 of that parameter's gradient norm."""
    g = load_golden(name)
    m, sd = build_train_student(g)
    terms, grads = s0_oracle_train_grads(g, sd, m)
    for a, b in zip(terms, g["loss"]):
        assert abs(a - b) <= 1e-5 * max(abs(b), 1e-12), (terms, g["loss"].tolist())
    names = [str(n) for n in g["grad_names"]]
    assert names == [n for n, _ in m.named_parameters() if n != "encoder.projection_layer"]
    for n, ref in zip(names, g["grad_stats"]):
        err = np.abs(grad_stats(grads[n]).numpy() - ref).max() / ref[0]
        assert err <= 1e-4, (n, err)


# ------------------------------------------------------------------------------------------------ the backward formulas
def _shift(t, s):
    """t [B, L, C] -> t[:, l + s] (zero outside the sequence)."""
    L = t.shape[1]
    out = torch.zeros_like(t)
    lo, hi = max(0, -s), min(L, L - s)
    if lo < hi:
        out[:, lo:hi] = t[:, lo + s:hi + s]
    return out


def _dw(t, w):
    """Depthwise (1, 11) conv along the sequence, zero padding 5: sum_k w[c, k] t[l + k - 5]; w [C, 11]."""
    return sum(w[:, k] * _shift(t, k - 5) for k in range(11))


def _dw_t(d, w):
    """Its transpose: sum_k w[c, k] d[l - k + 5]."""
    return sum(w[:, k] * _shift(d, 5 - k) for k in range(11))


def _dw_taps(d, t):
    """Tap gradient [C, 11]: sum over (b, l) of d[l] t[l + k - 5]."""
    return torch.stack([(d * _shift(t, k - 5)).sum((0, 1)) for k in range(11)], 1)


def _bn_affine(sd, p, eps=1e-5):
    inv = 1.0 / torch.sqrt(sd[p + ".running_var"] + eps)
    s = sd[p + ".weight"] * inv
    return s, sd[p + ".bias"] - sd[p + ".running_mean"] * s, sd[p + ".running_mean"], inv


def repmixer_formula_backward(x, g, sd, p):
    """The frozen-BN RepMixerBlock backward as the kernels compute it (fp64 torch): x, g [B, L, C] -> (dx, {name: grad})."""
    tm, f = p + ".token_mixer", p + ".convffn"
    s_ms, b_ms, rm_ms, inv_ms = _bn_affine(sd, tm + ".mixer.rbr_skip")
    s_mc, b_mc, rm_mc, inv_mc = _bn_affine(sd, tm + ".mixer.rbr_conv.0.bn")
    s_ns, b_ns, rm_ns, inv_ns = _bn_affine(sd, tm + ".norm.rbr_skip")
    s_f, b_f, rm_f, inv_f = _bn_affine(sd, f + ".conv.bn")
    w_mc = sd[tm + ".mixer.rbr_conv.0.conv.weight"].reshape(-1, 11)
    w_f = sd[f + ".conv.conv.weight"].reshape(-1, 11)
    ls_tm, ls_blk = sd[tm + ".layer_scale"].reshape(-1), sd[p + ".layer_scale"].reshape(-1)
    W1, b1 = sd[f + ".fc1.weight"].flatten(1), sd[f + ".fc1.bias"]
    W2, b2 = sd[f + ".fc2.weight"].flatten(1), sd[f + ".fc2.bias"]
    # forward
    c = _dw(x, w_mc)
    r = s_ms * x + b_ms + s_mc * c + b_mc - (s_ns * x + b_ns)
    x1 = x + ls_tm * r
    fv = _dw(x1, w_f)
    u = s_f * fv + b_f
    z = u @ W1.t() + b1
    h = F.gelu(z)
    y = h @ W2.t() + b2
    # backward
    gr = {}
    gr[p + ".layer_scale"] = (g * y).sum((0, 1)).reshape(-1, 1, 1)
    dy = ls_blk * g
    gr[f + ".fc2.bias"] = dy.sum((0, 1))
    gr[f + ".fc2.weight"] = torch.einsum("bln,blk->nk", dy, h).reshape(W2.shape[0], -1, 1, 1)
    dh = dy @ W2
    dz = dh * (0.5 * (1 + torch.erf(z / math.sqrt(2))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi))
    gr[f + ".fc1.bias"] = dz.sum((0, 1))
    gr[f + ".fc1.weight"] = torch.einsum("bln,blk->nk", dz, u).reshape(W1.shape[0], -1, 1, 1)
    du = dz @ W1
    gr[f + ".conv.bn.weight"] = (du * (fv - rm_f) * inv_f).sum((0, 1))
    gr[f + ".conv.bn.bias"] = du.sum((0, 1))
    df = s_f * du
    gr[f + ".conv.conv.weight"] = _dw_taps(df, x1).reshape(-1, 1, 1, 11)
    e = g + _dw_t(df, w_f)
    gr[tm + ".layer_scale"] = (e * r).sum((0, 1)).reshape(-1, 1, 1)
    ep = ls_tm * e
    gr[tm + ".mixer.rbr_skip.weight"] = (ep * (x - rm_ms) * inv_ms).sum((0, 1))
    gr[tm + ".norm.rbr_skip.weight"] = -(ep * (x - rm_ns) * inv_ns).sum((0, 1))
    gr[tm + ".mixer.rbr_conv.0.bn.weight"] = (ep * (c - rm_mc) * inv_mc).sum((0, 1))
    sb = ep.sum((0, 1))
    gr[tm + ".mixer.rbr_skip.bias"], gr[tm + ".mixer.rbr_conv.0.bn.bias"], gr[tm + ".norm.rbr_skip.bias"] = sb, sb, -sb
    dc = s_mc * ep
    gr[tm + ".mixer.rbr_conv.0.conv.weight"] = _dw_taps(dc, x).reshape(-1, 1, 1, 11)
    dx = e + (s_ms - s_ns) * ep + _dw_t(dc, w_mc)
    return dx, gr


def repmixer_block_sd(C, seed):
    """A fill_state_dict-initialised RepMixerBlock state dict under the prefix "blk", in fp64."""
    from efficientsam3_b200.backbones.mobile_clip import RepMixerBlock
    from oracle.weights import fill_state_dict
    sd = fill_state_dict(RepMixerBlock(dim=C).state_dict(), seed)
    return {"blk." + k: v.double() for k, v in sd.items() if not k.endswith("num_batches_tracked")}


@pytest.mark.parametrize("L", [1, 4, 11, 77])
def test_repmixer_backward_formulas_match_oracle_autograd(L):
    from oracle import text as OT
    B, C = 3, 32
    sd0 = repmixer_block_sd(C, 40 + L)
    g_ = torch.Generator().manual_seed(L)
    x = torch.randn(B, L, C, generator=g_, dtype=torch.float64)
    gout = torch.randn(B, L, C, generator=g_, dtype=torch.float64)
    sd = {k: v.clone().requires_grad_(not k.endswith(("running_mean", "running_var"))) for k, v in sd0.items()}
    xr = x.clone().requires_grad_(True)
    OT.repmixer_block(xr, sd, "blk").backward(gout)
    dx, gr = repmixer_formula_backward(x, gout, sd0, "blk")
    assert torch.allclose(dx, xr.grad, rtol=1e-9, atol=1e-11 * xr.grad.abs().max().item())
    names = [k for k, v in sd.items() if v.grad is not None]
    assert sorted(names) == sorted(gr), sorted(set(names) ^ set(gr))
    for k in names:
        ref = sd[k].grad
        assert gr[k].shape == ref.shape, k
        assert torch.allclose(gr[k], ref, rtol=1e-9, atol=1e-11 * max(ref.abs().max().item(), 1e-30)), k


def test_flat_adamw_weight_decay_groups_of_s0():
    """set_weight_decay (stage1/optimizer.py:33-46): 1-D parameters and biases skip decay.  On S0 that puts every BatchNorm
    gamma / beta and every bias in the no-decay group, while the [C, 1, 1] layer scales and the depthwise taps decay."""
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.model import text_student_cfg
    from efficientsam3_b200.stage1.optim import FlatAdamW
    from test_text_cpu import BPE
    cfg = text_student_cfg("MobileCLIP-S0")
    cfg.update(n_transformer_layers=1, context_length=16)
    m = TextStudentEncoder(cfg=cfg, context_length=16, output_dim=256, bpe_path=BPE)
    opt = FlatAdamW(m, lr=1e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    decay = {n for n, o in zip(opt.names, opt.offsets) if o < opt.n_decay}
    no_decay = set(opt.names) - decay
    params = dict(m.named_parameters())
    rm = [n for n in params if n.startswith(("encoder.transformer.0.", "encoder.transformer.2."))]
    assert len(rm) == 2 * 16          # 2 layer scales, 4 BNs x (gamma, beta), 2 tap sets, fc1 and fc2 (weight, bias)
    for n in rm:
        p = params[n]
        if ".rbr_skip." in n or ".bn." in n or n.endswith(".bias"):
            assert n in no_decay and p.dim() == 1, n
        else:
            assert n in decay, n
    layer_scales = [n for n in rm if n.endswith("layer_scale")]
    assert len(layer_scales) == 4 and all(params[n].shape == (512, 1, 1) and n in decay for n in layer_scales)
    taps = [n for n in rm if n.endswith("conv.weight") and params[n].shape[-1] == 11]
    assert len(taps) == 4 and all(n in decay for n in taps)
