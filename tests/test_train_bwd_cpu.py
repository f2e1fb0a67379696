"""The fp64 statements of tests/ref_train_bwd.py against torch.autograd of each forward operation in float64, on the CPU, at small
shapes: the references the backward-kernel GPU tests hold the kernels to are themselves right.  Each bound is finite and >= 0."""
import pytest
import torch
import torch.nn.functional as F

import ref_train_bwd as R

D = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close(a, b):
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.allclose(a, b, rtol=1e-10, atol=1e-11), (a - b).abs().max().item()


def _bound_ok(bound):
    assert torch.isfinite(bound).all() and (bound > 0).all()


def _grads(f, inputs, dout):
    ins = [t.clone().requires_grad_(True) for t in inputs]
    return torch.autograd.grad(f(*ins), ins, dout)


@pytest.mark.parametrize("shift", [None, (5, 7, -1, 1), (5, 7, 1, 0), (5, 7, 0, -1)])
def test_wgrad_reference(shift):
    g = _g(1)
    M, N, K = 70, 6, 9
    dz, x, w, dW0 = torch.randn(M, N, generator=g, dtype=D), torch.randn(M, K, generator=g, dtype=D), torch.randn(N, K, generator=g,
                                                                                                                      dtype=D), torch.randn(N, K, generator=g, dtype=D)
    if shift is None:
        (gw,) = _grads(lambda ww: x @ ww.t(), [w], dz)
        ref, bound = R.wgrad(dz, x, dW0)
    else:                                   # one tap of a dense 3x3 conv's weight gradient
        H, W, dy, dx = shift
        a = x.reshape(2, H, W, K).permute(0, 3, 1, 2)
        w9 = torch.randn(N, K, 3, 3, generator=g, dtype=D)
        (g9,) = _grads(lambda ww: F.conv2d(a, ww, padding=1), [w9], dz.reshape(2, H, W, N).permute(0, 3, 1, 2))
        gw = g9[..., dy + 1, dx + 1]
        ref, bound = R.wgrad(dz, R.shift_rows(x, H, W, dy, dx), dW0)
    _close(ref, dW0 + gw)
    _bound_ok(bound)


@pytest.mark.parametrize("H,W,ks,stride", [(7, 9, 3, 2), (8, 8, 3, 2), (9, 6, 5, 2), (6, 7, 3, 1), (5, 5, 5, 1)])
def test_dwconv_references(H, W, ks, stride):
    g = _g(H * W + ks)
    B, C = 2, 3
    x = torch.randn(B, H, W, C, generator=g, dtype=D)
    w = torch.randn(ks * ks, C, generator=g, dtype=D)
    f = lambda xx, ww: F.conv2d(xx.permute(0, 3, 1, 2), R.dw_weight(ww), stride=stride, padding=ks // 2, groups=C)
    Ho, Wo = f(x, w).shape[2:]
    dz = torch.randn(B, Ho, Wo, C, generator=g, dtype=D)
    gx, gw = _grads(f, [x, w], dz.permute(0, 3, 1, 2))
    ref, bound = R.dwconv_bwd_data(dz, w, H, W, ks, stride)
    _close(ref, gx)
    _bound_ok(bound)
    dW0 = torch.randn(C, 1, ks, ks, generator=g, dtype=D)
    ref, bound = R.dwconv_wgrad(dz, x, dW0, ks, stride)
    _close(ref, dW0 + R.dw_weight(gw))
    _bound_ok(bound)


def test_stem_and_conv3x3_wgrad_references():
    g = _g(3)
    img = torch.randn(2, 3, 9, 11, generator=g, dtype=D)
    w = torch.randn(8, 3, 3, 3, generator=g, dtype=D)
    dz = torch.randn(2, 5, 6, 8, generator=g, dtype=D)
    (gw,) = _grads(lambda ww: F.conv2d(img, ww, stride=2, padding=1), [w], dz.permute(0, 3, 1, 2))
    ref, bound = R.stem_wgrad(img, dz, w)
    _close(ref, w + gw)
    _bound_ok(bound)
    a, dy = torch.randn(2, 5, 7, 4, generator=g, dtype=D), torch.randn(2, 5, 7, 6, generator=g, dtype=D)
    w3 = torch.randn(6, 4, 3, 3, generator=g, dtype=D)
    (gw,) = _grads(lambda ww: F.conv2d(a.permute(0, 3, 1, 2), ww, padding=1), [w3], dy.permute(0, 3, 1, 2))
    ref, bound = R.conv3x3_wgrad(dy, a, w3)
    _close(ref, w3 + gw)
    _bound_ok(bound)


def test_transpose_pad_reference():
    x = torch.arange(2 * 3 * 5 * 2, dtype=D).reshape(2, 3, 5, 2) + 1
    for dx in (-1, 0, 1):
        t = R.transpose_pad(x, 8, dx).reshape(2, 2, 5, 8)
        assert t.sum() == x.sum() and (t != 0).sum() == x.numel()
        assert torch.equal(t[:, :, 1:4, 1 - dx:6 - dx], x.permute(3, 0, 1, 2))


def test_bn_stats_reference():
    g = _g(4)
    M, C = 50, 5
    z = torch.randn(M, C, generator=g, dtype=D) + 10
    gamma, beta = torch.rand(C, generator=g, dtype=D) + 0.5, torch.randn(C, generator=g, dtype=D)
    rm, rv = torch.randn(C, generator=g, dtype=D), torch.rand(C, generator=g, dtype=D) + 0.5
    rm2, rv2 = rm.clone(), rv.clone()
    y = F.batch_norm(z, rm2, rv2, gamma, beta, training=True, momentum=0.1, eps=1e-5)
    ref = R.bn_stats(z, gamma, beta, 1e-5, 0.1, rm, rv)
    _close(ref["running_mean"][0], rm2)
    _close(ref["running_var"][0], rv2)
    _close(z * ref["scale"][0] + ref["shift"][0], y)
    _close(ref["mean"][0], z.mean(0))
    for _, b in ref.values():
        _bound_ok(b)


@pytest.mark.parametrize("mode", ["none", "eval", "batch"])
@pytest.mark.parametrize("act", [None, "relu", "hswish", "gelu"])
def test_bn_act_bwd_reference(mode, act):
    """dz, dgamma, dbeta against autograd of act(norm(z)): bias only, frozen BN, batch-statistics BN."""
    g = _g(5)
    M, C, eps = 40, 4, 1e-5
    z = torch.randn(M, C, generator=g, dtype=D) * 2 + 0.5
    da = torch.randn(M, C, generator=g, dtype=D)
    gamma, beta = torch.rand(C, generator=g, dtype=D) + 0.5, torch.randn(C, generator=g, dtype=D)
    dg0, db0 = torch.full((C,), 0.25, dtype=D), torch.full((C,), -0.5, dtype=D)
    act_f = lambda u: R._act64(u, act)
    if mode == "none":
        scale = gamma
        gz, gb = _grads(lambda zz, bb: act_f(zz * scale + bb), [z, beta], da)
        ref = R.bn_act_bwd(da, z, scale, beta, act, mode, None, None, dg0, db0)
        gg = None
    else:
        if mode == "eval":
            mean, invstd = torch.randn(C, generator=g, dtype=D), torch.rand(C, generator=g, dtype=D) + 0.5
            f = lambda zz, gm, bb: act_f((zz - mean) * invstd * gm + bb)
        else:
            mean, invstd = z.mean(0), (z.var(0, unbiased=False) + eps).rsqrt()
            f = lambda zz, gm, bb: act_f(F.batch_norm(zz, None, None, gm, bb, training=True, eps=eps))
        gz, gg, gb = _grads(f, [z, gamma, beta], da)
        scale = gamma * invstd
        ref = R.bn_act_bwd(da, z, scale, beta - mean * scale, act, mode, mean, invstd, dg0, db0)
        _close(ref["dgamma"][0], dg0 + gg)
    _close(ref["dz"][0], gz)
    _close(ref["dbeta"][0], db0 + gb)
    for _, b in ref.values():
        _bound_ok(b)


def test_act_grad_and_kink_band():
    x = torch.tensor([-4.0, -3.0, -1.0, 0.0, 1e-9, 2.0, 3.0, 5.0], dtype=D)
    for act in ("relu", "hswish", "gelu"):
        xr = x.clone().requires_grad_(True)
        (gx,) = torch.autograd.grad(R._act64(xr, act).sum(), xr)
        keep = ~R.kink_band(x, act)
        assert torch.allclose(R.act_grad(x, act)[keep], gx[keep])
    assert R.kink_band(x, "hswish").tolist() == [False, True, False, False, False, False, True, False]
    assert R.kink_band(x, "relu")[3] and not R.kink_band(x, "gelu").any()


@pytest.mark.parametrize("act", [None, "relu", "hswish", "gelu"])
def test_affine_act_reference(act):
    g = _g(6)
    z, s, b, r = (torch.randn(10, 4, generator=g, dtype=D), torch.rand(4, generator=g, dtype=D), torch.randn(4, generator=g, dtype=D),
                  torch.randn(10, 4, generator=g, dtype=D))
    ref, bound = R.affine_act(z, s, b, act, r)
    _close(ref, R._act64(z * s + b, act) + r)
    _bound_ok(bound)


def test_se_references():
    g = _g(7)
    dy, x = torch.randn(2, 9, 4, generator=g, dtype=D), torch.randn(2, 9, 4, generator=g, dtype=D)
    gate, add, dg0 = torch.rand(2, 4, generator=g, dtype=D), torch.randn(2, 4, generator=g, dtype=D), torch.randn(2, 4, generator=g, dtype=D)
    gx, gg = _grads(lambda xx, gt: xx * gt[:, None], [x, gate], dy)
    ref, bound = R.se_dgate(dy, x, dg0)
    _close(ref, dg0 + gg)
    _bound_ok(bound)
    ref, bound = R.se_apply(dy, gate, add)
    _close(ref, dy * gate[:, None] + add[:, None])
    _close(R.se_apply(dy, gate, torch.zeros_like(add))[0], _grads(lambda xx: xx * gate[:, None], [x], dy)[0])
    _bound_ok(bound)


@pytest.mark.parametrize("Hi,Wi,Ho,Wo", [(4, 5, 8, 10), (3, 4, 11, 15), (9, 7, 4, 3)])
def test_bilinear_bwd_reference_is_the_adjoint(Hi, Wi, Ho, Wo):
    """<resize(x), d> = <x, bwd(d)> with the resize written out explicitly (align_corners=False source coordinates)."""
    g = _g(8)
    x = torch.randn(2, 3, Hi, Wi, generator=g, dtype=D)
    d = torch.randn(2, 3, Ho, Wo, generator=g, dtype=D)

    def axis(n_in, n_out):
        A = torch.zeros(n_out, n_in, dtype=D)
        for o in range(n_out):
            f = max((o + 0.5) * n_in / n_out - 0.5, 0.0)
            i0 = min(int(f), n_in - 1)
            i1 = min(i0 + 1, n_in - 1)
            A[o, i0] += 1 - (f - i0)
            A[o, i1] += f - i0
        return A
    y = torch.einsum("oi,bcij,pj->bcop", axis(Hi, Ho), x, axis(Wi, Wo))
    ref, bound = R.bilinear_bwd(d, Hi, Wi)
    assert abs((y * d).sum() - (x.permute(0, 2, 3, 1) * ref).sum()) < 1e-10
    _bound_ok(bound)


def test_colsum_reference():
    s, o = torch.randn(7, 3, generator=_g(9), dtype=D), torch.randn(3, generator=_g(10), dtype=D)
    ref, bound = R.colsum(s, o)
    _close(ref, o + s.sum(0))
    _bound_ok(bound)


def _lite(ms, heads2, dim, eps):
    B, HW, _ = ms.shape
    t = ms.reshape(B, HW, heads2, 3 * dim)
    q, k, v = F.relu(t[..., :dim]), F.relu(t[..., dim:2 * dim]), t[..., 2 * dim:]
    vpad = torch.cat([v, torch.ones_like(v[..., :1])], -1)
    kv = torch.einsum("bnhj,bnhi->bhji", vpad, k)
    o = torch.einsum("bhji,bnhi->bnhj", kv, q)
    return (o[..., :dim] / (o[..., dim:] + eps)).reshape(B, HW, heads2 * dim), kv


@pytest.mark.parametrize("dim,HW", [(16, 5), (16, 130), (32, 77)])
def test_litemla_bwd_reference(dim, HW):
    """Against autograd of the ReLU linear attention; the KV partial sums are split over three chunks as the forward leaves them."""
    g = _g(dim + HW)
    B, heads2 = 2, 3
    ms = torch.randn(B, HW, heads2 * 3 * dim, generator=g, dtype=D)
    dy = torch.randn(B, HW, heads2 * dim, generator=g, dtype=D)
    (gms,) = _grads(lambda m: _lite(m, heads2, dim, 1e-15)[0], [ms], dy)
    kv = _lite(ms, heads2, dim, 1e-15)[1]
    part = torch.randn(B, heads2, 3, dim + 1, dim, generator=g, dtype=D)
    part[:, :, 2] = kv - part[:, :, :2].sum(2)
    ref, bound = R.litemla_bwd(ms, dy, part, heads2, dim, 1e-15)
    _close(ref, gms)
    _bound_ok(bound)


@pytest.mark.parametrize("dres", [False, True])
def test_layernorm_bwd_reference(dres):
    g = _g(11)
    M, C = 6, 10
    x, dy = torch.randn(M, C, generator=g, dtype=D) * 2 + 0.5, torch.randn(M, C, generator=g, dtype=D)
    gamma, beta = torch.rand(C, generator=g, dtype=D) + 0.5, torch.randn(C, generator=g, dtype=D)
    r = torch.randn(M, C, generator=g, dtype=D) if dres else None
    gx, gg, gb = _grads(lambda xx, gm, bb: F.layer_norm(xx, (C,), gm, bb, 1e-5), [x, gamma, beta], dy)
    dg0, db0 = torch.full((C,), 0.5, dtype=D), torch.full((C,), -1.0, dtype=D)
    ref = R.layernorm_bwd(x, dy, gamma, 1e-5, dg0, db0, r)
    _close(ref["dx"][0], gx + (r if dres else 0))
    _close(ref["dgamma"][0], dg0 + gg)
    _close(ref["dbeta"][0], db0 + gb)
    for _, b in ref.values():
        _bound_ok(b)


@pytest.mark.parametrize("B,H,W,heads,ws", [(2, 4, 6, 2, 2), (1, 3, 3, 1, 3)])
def test_win_attn_bias_bwd_reference(B, H, W, heads, ws):
    """dqkv against autograd of windowed attention with a per-head bias; dS of each window against the gradient of a bias that is
    separate per window (its sum over the windows is the shared bias's gradient)."""
    g = _g(12)
    C, N = 32 * heads, ws * ws
    qkv = torch.randn(B * H * W, 3 * C, generator=g, dtype=D)
    dout = torch.randn(B * H * W, C, generator=g, dtype=D)
    tok = R.win_attn_tokens(B, H, W, ws)
    nwin = tok.shape[0]
    bias = torch.randn(heads, N, N, generator=g, dtype=D)
    scale = 32 ** -0.5

    def f(qq, bw):                          # bw: [nwin, heads, N, N] per-window bias
        t = qq[tok].reshape(nwin, N, heads, 3, 32).permute(3, 0, 2, 1, 4)
        p = torch.softmax(scale * t[0] @ t[1].transpose(-1, -2) + bw, -1)
        o = (p @ t[2]).permute(0, 2, 1, 3).reshape(nwin * N, C)
        out = torch.empty(B * H * W, C, dtype=D)
        out = out.index_put((tok.reshape(-1),), o)
        return out
    gq, gbw = _grads(f, [qkv, bias.expand(nwin, -1, -1, -1).contiguous()], dout)
    ref = R.win_attn_bias_bwd(qkv, dout, bias, B, H, W, C, heads, ws, scale)
    _close(ref["dqkv"][0], gq)
    _close(ref["dS"][0], gbw)
    for _, b in ref.values():
        _bound_ok(b)
