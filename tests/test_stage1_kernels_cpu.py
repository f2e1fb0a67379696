"""tests/ref_stage1.py on the CPU: each statement is tied to the reference it restates -- the exact valid mask to the oracle's
build_valid_mask (fp32 F.interpolate), the forward to the oracle's loss, the backward to the torch semantics of
F.cosine_similarity below its eps, AdamW to torch.optim.AdamW after clip_grad_norm_, the scaler to torch's GradScaler update --
and the bounds are shown to hold for an fp32 restatement of the fixed KD backward and to reject the formula it replaced."""
import numpy as np
import pytest
import torch

import ref_stage1 as R
from bounds import U


def _oracle_masks(img, E, sizes):
    from oracle.kd_loss import build_valid_mask
    return build_valid_mask(img, [(3, h, w) for h, w in sizes], (E, E))[:, 0] > 0


@pytest.mark.parametrize("img,E", [(1008, 72), (1024, 64), (100, 7), (252, 18), (1000, 63), (512, 37), (800, 50), (32, 64)])
def test_exact_mask_is_the_oracles(img, E):
    """Every h at w = img / 2 + 1 and every w at h = img // 3, in batches, against build_valid_mask's fp32 F.interpolate."""
    sizes = [(h, img // 2 + 1) for h in range(1, img + 1, max(1, img // 200))] + \
            [(img // 3, w) for w in range(1, img + 1, max(1, img // 200))] + [(1, 1), (img, img)]
    for i in range(0, len(sizes), 64):
        chunk = sizes[i:i + 64]
        assert torch.equal(R.valid_masks(img, E, chunk), _oracle_masks(img, E, chunk)), (img, E, chunk)


def _kd_case(B=3, C=16, E=9, img=144, seed=0):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(B, C, E, E, generator=g, dtype=torch.float64)
    t = torch.randn(B, C, E, E, generator=g, dtype=torch.float64)
    sizes = [(img, img * 3 // 4), (img * 2 // 3, img), (img, img)][:B]
    return p, t, sizes, img


def test_forward_statement_is_the_oracle_loss():
    from oracle.kd_loss import kd_loss
    p, t, sizes, img = _kd_case()
    mask = R.valid_masks(img, p.shape[-1], sizes)
    ref = R.kd_fwd(p, t, mask, 0.7)
    loss, mse, cos = kd_loss(p, t, img, [(3, h, w) for h, w in sizes], 0.7)
    assert torch.allclose(ref["out3"][0], torch.stack([loss, mse, cos]), rtol=1e-7, atol=0)    # oracle's eps is the double 1e-8
    assert torch.equal(ref["per_sample"][0][:, 2], mask.sum((1, 2)).double())


def _tiny_case(C):
    """One sample, pixels 0..4 of row 0 with |pred| 0, 3e-9, 7e-9, 9.9e-9, 2e-8 along the teacher (|cos| ~ 0.9)."""
    g = torch.Generator().manual_seed(C)
    E = 7
    t = torch.randn(1, C, E, E, generator=g)
    p = torch.randn(1, C, E, E, generator=g)
    for j, r in enumerate([0.0, 3e-9, 7e-9, 9.9e-9, 2e-8]):
        d = t[0, :, 0, j] + 0.3 * torch.randn(C, generator=g)
        p[0, :, 0, j] = d / d.norm() * r if r > 0 else 0.0
    return p, t, torch.ones(1, E, E, dtype=torch.bool)


def _kernel_bwd32(p, t, w, g, fixed):
    """kd_loss_bwd_kernel restated in fp32 torch on an all-valid mask: the fixed k_a = w up dot / (na^2 |p| nt) (0 at p = 0), or the
    formula it replaced, w up dot / (na^3 nt)."""
    f = torch.float32
    dot, np2, nt2 = (p * t).sum(1), (p * p).sum(1), (t * t).sum(1)
    np_ = np2.sqrt()
    na, nt = np_.clamp_min(R.COS_EPS), nt2.sqrt().clamp_min(R.COS_EPS)
    up = torch.tensor(g, dtype=f) / (p.shape[0] * float(p.shape[2] * p.shape[3]))
    k_t = -w * up / (na * nt)
    if fixed:
        k_a = torch.where(np_ > 0, w * up * dot / (na * na * np_ * nt), torch.zeros_like(dot))
    else:
        k_a = w * up * dot / (na * na * na * nt)
    return 2 * up * (p - t) + k_t[:, None] * t + k_a[:, None] * p


@pytest.mark.parametrize("C", [1, 32, 1024])
def test_backward_bound_holds_for_the_fixed_kernel_and_rejects_the_old_one(C):
    """Below the 1e-8 clamp torch's gradient keeps |p|'s own derivative p / |p|: an fp32 restatement of the fixed backward stays
    inside kd_bwd's bound on every element, the replaced na^3 formula falls outside it on the pixels with 0 < |p| < 1e-8 only."""
    p, t, mask = _tiny_case(C)
    ref, bound = R.kd_bwd(p.double(), t.double(), mask, 1.0, 0.75)
    err = lambda fixed: (_kernel_bwd32(p, t, 1.0, 0.75, fixed).double() - ref).abs() / bound
    assert err(True).max() <= 1.0
    bad = (err(False) > 1.0).any(1)[0]                                   # [E, E]: pixels with an element outside
    want = torch.zeros_like(bad)
    want[0, 1:4] = True                                                  # |p| = 3e-9, 7e-9, 9.9e-9
    assert torch.equal(bad, want), bad.nonzero().tolist()


def test_adamw_statement_is_torch_adamw_after_clipping():
    """With double scalars ref_stage1.adamw is torch.optim.AdamW (float64) on gradients unscaled by world x scale and clipped by
    clip_grad_norm_, the decay group first."""
    g0 = torch.Generator().manual_seed(5)
    n, nd, lr, betas, eps, wd, scale, world, max_norm = 37, 20, 3e-3, (0.9, 0.999), 1e-8, 0.05, 1024.0, 4, 1.0
    p = torch.randn(n, generator=g0, dtype=torch.float64)
    m = torch.randn(n, generator=g0, dtype=torch.float64) * 1e-2
    v = torch.rand(n, generator=g0, dtype=torch.float64) * 1e-4
    g = torch.randn(n, generator=g0, dtype=torch.float64) * scale * world
    step = 6
    a, b = p[:nd].clone().requires_grad_(True), p[nd:].clone().requires_grad_(True)
    opt = torch.optim.AdamW([{"params": [a]}, {"params": [b], "weight_decay": 0.0}], lr=lr, betas=betas, eps=eps, weight_decay=wd)
    for q, sl in ((a, slice(0, nd)), (b, slice(nd, n))):
        q.grad = g[sl] / (scale * world)
        opt.state[q] = {"step": torch.tensor(float(step), dtype=torch.float64), "exp_avg": m[sl].clone(), "exp_avg_sq": v[sl].clone()}
    total = float(torch.nn.utils.clip_grad_norm_([a, b], max_norm))
    assert total > max_norm
    opt.step()
    ref = R.adamw(p, g, m, v, nd, lr, betas, eps, wd, max_norm, 1.0 / world, float((g * g).sum()), scale, float(step))
    got = torch.cat([a.detach(), b.detach()])
    assert torch.allclose(ref["p"][0], got, rtol=1e-12, atol=1e-15)
    assert torch.allclose(ref["m"][0], torch.cat([opt.state[a]["exp_avg"], opt.state[b]["exp_avg"]]), rtol=1e-12, atol=1e-18)
    assert torch.allclose(ref["v"][0], torch.cat([opt.state[a]["exp_avg_sq"], opt.state[b]["exp_avg_sq"]]), rtol=1e-12, atol=1e-20)


def test_beta_rounding_and_powf_terms_are_the_documented_size():
    """The two named differences from torch's double-precision bias correction at t = 1, b2 = 0.999: fp32 rounds b2 so that 1 - b2
    is 1.3e-5 relative off, and powf's 4 ulp of b2^t, charged at 2u |b2^t| each, are 4.8e-4 of 1 - b2^t (the cancellation)."""
    b2 = R.f32(0.999)
    assert 1.2e-5 < abs((1 - b2) - 0.001) / 0.001 < 1.4e-5
    assert 4e-4 < R.POWF_ULP * 2 * U * b2 / (1 - b2) < 5e-4


def test_scaler_state_is_gradscaler_update():
    """ref_stage1.scaler_state's scale and growth tracker follow torch._amp_update_scale_ (GradScaler.update) over a sequence of
    clean and non-finite steps with growth interval 3; the step count moves on clean steps only."""
    scale, tracker = torch.tensor([65536.0]), torch.tensor([0], dtype=torch.int32)
    state = np.array([65536.0, 0, 0, 0], dtype=np.float32)
    for bad in [False, False, True, False, False, False, True, False, False, False, False, True]:
        torch._amp_update_scale_(scale, tracker, torch.tensor([1.0 if bad else 0.0]), 2.0, 0.5, 3)
        state = R.scaler_state(state, 4.0, bad, 1.0, True, 3)
        assert state[0] == float(scale) and state[1] == int(tracker)
    assert state[2] == 9
