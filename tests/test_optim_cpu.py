"""CPU: host logic of the optimiser side of the KD step (efficientsam3_b200/stage1/optim.py): parameter grouping, arena
layout, LR schedule, checkpoint interop with torch.optim.AdamW.  The update itself is a CUDA kernel (tests/test_optim_gpu.py)."""
import math

import pytest
import torch

from efficientsam3_b200.stage1 import optim as O


def _student():
    from types import SimpleNamespace as NS
    from efficientsam3_b200.stage1.model import build_image_student_model
    cfg = NS(MODEL=NS(BACKBONE="tiny_vit_5m"), DATA=NS(IMG_SIZE=224), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=14))
    return build_image_student_model(cfg)


def test_decay_groups_follow_the_reference_rule():
    m = _student()
    decay, no_decay = O.split_decay(m.named_parameters(), skip_keywords=("attention_biases",))
    names_d, names_n = {n for n, _ in decay}, {n for n, _ in no_decay}
    assert names_d.isdisjoint(names_n) and len(names_d) + len(names_n) == sum(1 for _ in m.parameters())
    for n, p in m.named_parameters():
        expect_no_decay = p.dim() == 1 or n.endswith(".bias") or "attention_biases" in n
        assert (n in names_n) == expect_no_decay, n
    assert any("attention_biases" in n for n in names_n)


def test_arena_layout_and_views():
    m = _student()
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    opt = O.FlatAdamW(m, lr=1e-3, weight_decay=0.05)
    assert opt.numel >= sum(p.numel() for p in m.parameters()) and opt.numel % 4 == 0
    lo, hi = opt.flat_param.data_ptr(), opt.flat_param.data_ptr() + opt.numel * 4
    for name, p, o in zip(opt.names, opt.params, opt.offsets):
        assert lo <= p.data_ptr() < hi and (p.data_ptr() - lo) == o * 4 and o % 4 == 0
        assert torch.equal(p.detach(), before[name])                 # values survived the move into the arena
        assert p.grad.data_ptr() == opt.flat_grad.data_ptr() + o * 4
        assert (o < opt.n_decay) == (not (p.dim() == 1 or name.endswith(".bias")))
    opt.params[0].grad.fill_(3.0)
    assert opt.flat_grad[: opt.params[0].numel()].eq(3.0).all()
    opt.zero_grad()
    assert opt.flat_grad.abs().sum().item() == 0
    with pytest.raises(RuntimeError):
        opt.step()                                                   # no CPU fallback for the update


def test_cosine_schedule_matches_restated_timm_rule():
    base, t_init, lr_min, wt, wl = 2e-3, 1000, 1e-5, 100, 1e-6
    assert O.cosine_lr(0, base, t_init, lr_min, wt, wl) == wl
    assert math.isclose(O.cosine_lr(50, base, t_init, lr_min, wt, wl), wl + 50 * (base - wl) / wt)
    # warmup_prefix=False: the cosine is evaluated at t, not t - warmup_t
    assert math.isclose(O.cosine_lr(100, base, t_init, lr_min, wt, wl), lr_min + 0.5 * (base - lr_min) * (1 + math.cos(math.pi * 0.1)))
    assert math.isclose(O.cosine_lr(500, base, t_init, lr_min, wt, wl), lr_min + 0.5 * (base - lr_min))
    assert O.cosine_lr(1000, base, t_init, lr_min, wt, wl) == lr_min and O.cosine_lr(5000, base, t_init, lr_min, wt, wl) == lr_min
    lrs = [O.cosine_lr(t, base, t_init, lr_min, wt, wl) for t in range(wt, t_init)]
    assert all(a >= b for a, b in zip(lrs, lrs[1:]))
    assert O.scaled_lr(1e-3, 32, 8) == 1e-3 * 256 / 512


def test_state_dict_round_trips_through_torch_adamw():
    torch.manual_seed(1)
    m = torch.nn.Sequential(torch.nn.Linear(6, 4), torch.nn.LayerNorm(4), torch.nn.Linear(4, 2))
    opt = O.FlatAdamW(m, lr=3e-4, betas=(0.9, 0.95), weight_decay=0.1, loss_scale=1024.0)
    opt.exp_avg.normal_(); opt.exp_avg_sq.uniform_(); opt.state[2] = 7
    sd = opt.state_dict()
    d, n = O.split_decay(m.named_parameters())
    ref = torch.optim.AdamW([{"params": [p for _, p in d]}, {"params": [p for _, p in n], "weight_decay": 0.0}], lr=1.0)
    ref.load_state_dict({k: v for k, v in sd.items() if k != "amp_scaler"})       # torch accepts the format
    assert ref.param_groups[0]["weight_decay"] == 0.1 and ref.param_groups[1]["weight_decay"] == 0.0
    assert ref.param_groups[0]["lr"] == 3e-4 and ref.param_groups[0]["betas"] == (0.9, 0.95)
    for i, p in enumerate(opt.params):
        assert torch.equal(ref.state[p]["exp_avg"], sd["state"][i]["exp_avg"]) and float(ref.state[p]["step"]) == 7.0
    opt2 = O.FlatAdamW(torch.nn.Sequential(torch.nn.Linear(6, 4), torch.nn.LayerNorm(4), torch.nn.Linear(4, 2)), lr=1.0)
    back = ref.state_dict()
    back["amp_scaler"] = sd["amp_scaler"]
    opt2.load_state_dict(back)
    for p_, o in zip(opt.params, opt.offsets):          # (alignment padding between parameters is not part of the state)
        sl = slice(o, o + p_.numel())
        assert torch.equal(opt2.exp_avg[sl], opt.exp_avg[sl]) and torch.equal(opt2.exp_avg_sq[sl], opt.exp_avg_sq[sl])
    assert opt2.lr == 3e-4 and float(opt2.state[0]) == 1024.0 and float(opt2.state[2]) == 7.0


def test_packed_weight_cache_follows_the_parameter():
    """nn_utils.cached_pack: one packed copy per parameter state -- rebuilt after a torch-side write (version counter), after the fused
    AdamW kernel moved the parameters through raw pointers (WEIGHTS_EPOCH), and after the parameter moved (data_ptr)."""
    import torch
    from efficientsam3_b200 import nn_utils as U
    conv = torch.nn.Conv2d(8, 16, 1, bias=False)
    a = U.pw_weight(conv)
    assert U.pw_weight(conv) is a and U.pw_weight_t(conv).shape == (8, 16)
    with torch.no_grad():
        conv.weight.mul_(2.0)
    b = U.pw_weight(conv)
    assert b is not a and torch.equal(b.float(), (conv.weight.detach().reshape(16, 8)).to(torch.bfloat16).float())
    conv.weight.data.view(-1)[0] = 123.0           # a raw write: the version counter of `.data` is not the parameter's
    U.bump_weights_epoch()                          # ... which is why FlatAdamW.step bumps the epoch
    c = U.pw_weight(conv)
    assert c is not b and float(c[0, 0]) == 123.0
    dw = torch.nn.Conv2d(8, 8, 3, padding=1, groups=8, bias=False)
    r = U.dw_weight_rot(dw)
    assert torch.equal(r, U.dw_weight(dw, None).flip(0)) and U.dw_weight_rot(dw) is r


def test_folded_pointwise_weight_is_the_scaled_weight_rounded_once():
    """nn_utils.pw_weight_scaled: W * s in fp32, then ONE bf16 rounding (not bf16(W) * s, which would round twice)."""
    from efficientsam3_b200.nn_utils import pw_weight, pw_weight_scaled
    torch.manual_seed(3)
    conv = torch.nn.Conv2d(24, 40, 1, bias=False)
    s = torch.rand(40) * 3 + 0.1
    wf = pw_weight_scaled(conv, s)
    assert wf.dtype == torch.bfloat16 and wf.shape == (40, 24) and wf.is_contiguous()
    exact = conv.weight.detach().reshape(40, 24) * s.view(-1, 1)
    assert torch.equal(wf, exact.to(torch.bfloat16))
    assert ((wf.float() - exact).abs() <= exact.abs() * 2.0 ** -8).all()
    assert torch.equal(pw_weight_scaled(conv, None), pw_weight(conv))


def test_tensor_core_tap_operand_is_cached_per_tensor_and_version(monkeypatch):
    """ops._tc_taps: the sum-preserving bf16 taps are computed once per weight tensor object and recomputed after an in-place update."""
    from efficientsam3_b200 import ops
    calls = []

    def fake_round(w):
        calls.append(w._version)
        return w.to(torch.bfloat16).float()
    monkeypatch.setattr(ops, "round_taps_sum_bf16", fake_round)
    w = torch.randn(9, 32)
    a = ops._tc_taps(w)
    b = ops._tc_taps(w)
    assert a is b and len(calls) == 1
    w.mul_(2.0)                                   # an optimiser step on the flat arena bumps the version of its views
    c = ops._tc_taps(w)
    assert c is not a and len(calls) == 2 and torch.equal(c, w.to(torch.bfloat16).float())
    assert ops._tc_taps(torch.randn(9, 32)) is not c and len(calls) == 3


def test_step_without_clipping_passes_max_norm_0(monkeypatch):
    """TRAIN.CLIP_GRAD None or 0 means no clipping (NativeScalerWithGradNormCount): FlatAdamW.step hands es3_adamw_flat max_norm 0,
    as kd_train_step(clip_grad=None) and text_kd_train_step do through it.  The two kernels are replaced by recorders and the arena
    is taken for a device one, so the host side runs without a GPU."""
    from efficientsam3_b200 import ops
    m = torch.nn.Sequential(torch.nn.Linear(6, 4), torch.nn.LayerNorm(4))
    opt = O.FlatAdamW(m, lr=1e-3)
    seen = []
    monkeypatch.setattr(ops, "grad_norm", lambda *a: None)
    monkeypatch.setattr(ops, "adamw_flat", lambda *a, **k: seen.append(float(a[9])))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda t: True))
    for clip in (None, 0, 0.0, 5.0):
        opt.step(max_norm=clip)
    monkeypatch.undo()
    assert seen == [0.0, 0.0, 0.0, 5.0]
