"""The fp64 statements of tests/ref_text.py against textbook float64 torch (softmax attention with a causal mask, F.layer_norm,
F.conv1d, F.embedding, F.interpolate, F.cosine_similarity, F.mse_loss; autograd for the backward ones), and the bound logic on
constructed cases: the online-softmax rescale charge, the fp32 resize weights, the cosine gradient at the norm clamp.  No GPU."""
import zlib

import pytest
import torch
import torch.nn.functional as F

import ref_text as R

D = torch.float64


def _g(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _bf(t):
    return t.to(torch.bfloat16).to(D)


def _within(ref, bound, other, what):
    err = (ref - other).abs()
    assert (err <= bound).all(), f"{what}: {int((err > bound).sum())} elements outside the bound (max err {err.max():.3g})"
    assert (bound > 0).all()


def _close(a, b, what=""):
    assert torch.allclose(a, b, rtol=1e-10, atol=1e-12), (what, (a - b).abs().max().item())


def _grads(f, xs, gout):
    xs = [x.clone().requires_grad_(True) for x in xs]
    y = f(*xs)
    return torch.autograd.grad(y, xs, gout)


def _textbook(qkv, B, L, heads, scale, causal):
    q, k, v = qkv.reshape(B, L, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = scale * q @ k.transpose(-1, -2)
    if causal:
        s = s + torch.full((L, L), float("-inf"), dtype=D).triu(1)
    return q, k, v, s


# ----------------------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("L,causal,kernel", [(1, True, "mma"), (17, True, "mma"), (77, False, "mma"), (128, True, "mma"),
                                             (128, False, "tc"), (100, False, "mma")])
def test_attention_statement(L, causal, kernel):
    """Against softmax attention with the unnormalised probabilities rounded to bf16 (through fp32) before PV and the row sums
    taken before that rounding; the statement's bound is positive everywhere."""
    g = _g("attn", L, causal)
    B, heads = 2, 2
    qkv = _bf(torch.randn(B * L, 3 * 64 * heads, generator=g, dtype=D) * 1.5)
    ref, bound = R.attention(qkv, B, L, heads, 0.125, causal, kernel)
    q, k, v, s = _textbook(qkv, B, L, heads, 0.125, causal)
    p = torch.exp(s - s.amax(-1, keepdim=True))
    o = (p.float().to(torch.bfloat16).to(D) @ v) / p.sum(-1, keepdim=True)
    _within(ref, bound, R._tokens(o), "attention")
    exact = R._tokens(torch.softmax(s, -1) @ v)
    assert ((ref - exact).abs() <= 2.0 ** -8 * (R._tokens(torch.softmax(s, -1) @ v.abs())) + 1e-12).all()


def test_online_softmax_charge_where_the_running_max_rises():
    """A row whose maximum sits in the second 64-key tile is rounded by the mma.sync kernel against the first tile's max: those
    elements carry a full bf16 rounding (2^-8 p) in the bound; with the maximum in the first tile they carry only band()."""
    B, heads, L = 1, 1, 100
    qkv = torch.zeros(B * L, 3 * 64)
    qkv[:, :64] = 1.0
    qkv[:, 64:128] = _bf(torch.randn(L, 64, generator=_g("rise"), dtype=D) * 0.1)
    qkv[:, 128:] = 1.0                       # v = 1: the output is exactly 1, its bound is the charge
    late = qkv.clone()
    late[90, 64:128] = 0.5                   # key 90 (tile 1) dominates every row
    early = qkv.clone()
    early[10, 64:128] = 0.5                  # key 10 (tile 0) dominates
    _, b_late = R.attention(late, B, L, heads, 0.125, False, "mma")
    _, b_early = R.attention(early, B, L, heads, 0.125, False, "mma")
    _, b_tc = R.attention(late, B, L, heads, 0.125, False, "tc")
    assert (b_late > b_early).all() and (b_late > b_tc).all()


@pytest.mark.parametrize("L,causal", [(1, True), (9, True), (33, False), (70, True)])
def test_attention_bwd_statement(L, causal):
    """dqkv against float64 autograd of softmax attention when the given O is the exact forward output (the statement's D is then
    rowsum(P dP)); with another O, D moves by exactly sum_c dO (O' - O)."""
    g = _g("attn_bwd", L, causal)
    B, heads, C = 2, 2, 128
    qkv = torch.randn(B * L, 3 * C, generator=g, dtype=D)
    dout = torch.randn(B * L, C, generator=g, dtype=D)

    def f(x):
        q, k, v, s = _textbook(x, B, L, heads, 0.125, causal)
        return R._tokens(torch.softmax(s, -1) @ v)
    o = f(qkv)
    (gq,) = _grads(f, [qkv], dout)
    ref, bound = R.attention_bwd(qkv, o, dout, B, L, heads, 0.125, causal)
    _close(ref, gq, "attention bwd")
    assert (bound > 0).all()
    o2 = o + 0.01
    ref2, _ = R.attention_bwd(qkv, o2, dout, B, L, heads, 0.125, causal)
    _close(ref2[:, 2 * C:], gq[:, 2 * C:], "dv")                              # dv does not read D
    if L > 1:
        assert not torch.allclose(ref2[:, :C], gq[:, :C])


# ----------------------------------------------------------------------------------------------------------- LayerNorm
def test_layernorm_f32_statement_with_tiled_pos():
    g = _g("lnf")
    M, C, H, W, ps = 2 * 6 * 5, 256, 6, 5, 2
    x = torch.randn(M, C, generator=g, dtype=D) * 2 + 3
    pos = torch.randn(ps * ps, C, generator=g, dtype=D)
    gm, bt = torch.randn(C, generator=g, dtype=D), torch.randn(C, generator=g, dtype=D)
    ref, bound = R.layernorm_f32(x, gm, bt, 1e-5, pos, ps, H, W)
    t = torch.arange(M) % (H * W)
    xp = x + pos[((t // W) % ps) * ps + (t % W) % ps]
    _close(ref, F.layer_norm(xp, (C,), gm, bt, 1e-5))
    assert (bound > 4 * 2.0 ** -24 * ref.abs()).all()
    ref_b, bound_b = R.layernorm_f32(x, gm, bt, 1e-5, bf16=True)
    _close(ref_b, F.layer_norm(x, (C,), gm, bt, 1e-5))
    assert (bound_b >= 2.0 ** -8 * ref_b.abs()).all()


def test_layernorm_bwd_f32_statement():
    g = _g("lnb")
    M, C = 7, 132
    x, dy = torch.randn(M, C, generator=g, dtype=D) * 2 + 0.5, torch.randn(M, C, generator=g, dtype=D)
    gm, bt = torch.rand(C, generator=g, dtype=D) + 0.5, torch.randn(C, generator=g, dtype=D)
    r = torch.randn(M, C, generator=g, dtype=D)
    gx, gg, gb = _grads(lambda xx, w, b: F.layer_norm(xx, (C,), w, b, 1e-5), [x, gm, bt], dy)
    dg0, db0 = torch.randn(C, generator=g, dtype=D), torch.randn(C, generator=g, dtype=D)
    ref = R.layernorm_bwd_f32(x, dy, gm, 1e-5, dg0, db0, r)
    _close(ref["dx"][0], gx + r)
    _close(ref["dgamma"][0], dg0 + gg)
    _close(ref["dbeta"][0], db0 + gb)
    as_bf16 = R.layernorm_bwd(x, dy, gm, 1e-5, dg0, db0, r)["dx"][1]
    assert (ref["dx"][1] < as_bf16).all() and (ref["dx"][1] > 0).all()         # an fp32 store: no bf16 half-step


# ----------------------------------------------------------------------------------------------------------- RepMixer
def test_repmixer_statement():
    g = _g("rm")
    B, L, C = 3, 13, 64
    x = torch.randn(B * L, C, generator=g, dtype=D)
    wm, wf = torch.randn(11, C, generator=g, dtype=D) * 0.3, torch.randn(11, C, generator=g, dtype=D) * 0.3
    bm, bf = torch.randn(C, generator=g, dtype=D), torch.randn(C, generator=g, dtype=D)
    (x1, b1), (u, bu) = R.repmixer(x, wm, bm, wf, bf, B, L)

    def dw(t, w, b):
        t = t.view(B, L, C).permute(0, 2, 1)
        return F.conv1d(t, w.t().unsqueeze(1), b, padding=5, groups=C).permute(0, 2, 1).reshape(B * L, C)
    _close(x1, dw(x, wm, bm))
    _close(u, dw(dw(x, wm, bm), wf, bf))
    assert (bu >= 2.0 ** -8 * u.abs()).all() and (b1 > 0).all()


# ----------------------------------------------------------------------------------------------------------- embedding gradients
def test_embed_and_pos_grad_statements():
    g = _g("emb")
    V, C, B, L = 50, 8, 3, 7
    ids = torch.randint(0, 10, (B, L), generator=g)
    dx = torch.randn(B * L, C, generator=g, dtype=D)
    g0 = torch.randn(V, C, generator=g, dtype=D)
    ref, bound = R.embed_grad(dx, ids, g0)
    (gt,) = _grads(lambda t: F.embedding(ids, t), [torch.zeros(V, C, dtype=D)], dx.view(B, L, C))
    _close(ref, g0 + gt)
    unused = torch.ones(V, dtype=torch.bool)
    unused[ids.unique()] = False
    assert torch.equal(ref[unused], g0[unused])
    for N, LL in ((77, 32), (16, 32), (32, 32), (1, 5), (9, 1)):
        pe = torch.randn(1, 1, N, C, generator=g, dtype=D)
        dxl = torch.randn(B, LL, C, generator=g, dtype=D)
        gp0 = torch.randn(N, C, generator=g, dtype=D)
        if N != LL:
            ref_r, bound_r = R.pos_resize(pe.view(N, C), LL)
            tab = F.interpolate(pe, size=(LL, C), mode="bilinear", align_corners=False).view(LL, C)
            assert ((ref_r - tab).abs() <= 1e-6 * pe.abs().max()).all()           # the fp32 weights are within 1e-6 of exact
            (gpe,) = _grads(lambda t: F.interpolate(t, size=(LL, C), mode="bilinear", align_corners=False).view(1, LL, C)
                            .expand(B, LL, C), [pe], dxl)
        else:
            gpe = dxl.sum(0)
        ref_p, bound_p = R.pos_grad(dxl, N, gp0)
        assert ((ref_p - gp0 - gpe.reshape(N, C)).abs() <= 1e-6 * dxl.abs().sum(0).max()).all(), (N, LL)


def test_resize_weights_follow_fp32_order():
    """The weights of N -> L rows: each row's weights sum to 1 within an fp32 rounding, lie in [0, 1], and at L = 32 (a power of
    two) the fp32 source coordinate is exact, so they equal torch's float64 interpolation weights."""
    for N, L in ((77, 32), (16, 32), (77, 16), (5, 77)):
        w = R.pos_weights(N, L)
        assert ((w.sum(1) - 1).abs() <= 2 ** -23).all() and (w >= 0).all() and (w <= 1).all()
        if L == 32:
            eye = torch.eye(N, dtype=D).view(N, 1, N, 1)
            exact = F.interpolate(eye, size=(L, 1), mode="bilinear", align_corners=False).view(N, L).t()
            _close(w, exact)


# ----------------------------------------------------------------------------------------------------------- KD loss
def _kd_inputs(B, L, Dm, g):
    p = torch.randn(B, L, Dm, generator=g, dtype=D)
    t = torch.randn(B, L, Dm, generator=g, dtype=D)
    p[0, 0] = 0.0                                              # p = 0: cp := 0
    if L > 1:
        p[0, 1] = p[0, 1] / p[0, 1].norm() * 1e-9              # |p| below the 1e-8 clamp
        t[1 % B, 1] = 0.0                                      # t = 0
    pad = torch.zeros(B, L, dtype=torch.bool)
    pad[:, L // 2 + 1:] = True
    pad[-1] = True                                             # a sample without a valid token
    return p, t, pad


@pytest.mark.parametrize("masked", [False, True])
def test_kd_loss_statements(masked):
    """ws / out3 against the loss terms summed in float64; dp against autograd; and the kernel's explicit dcos/dp (the bound's form)
    equals autograd of F.cosine_similarity at |p| = 1, below the clamp and at p = 0."""
    g = _g("kd", masked)
    B, L, Dm = 3, 6, 33
    p, t, pad = _kd_inputs(B, L, Dm, g)
    pd = pad if masked else None
    (ws, bws), cl = R.kd_partials(p, t, pd)
    v = (~pad).double() if masked else torch.ones(B, L, dtype=D)
    _close(ws[:, 0], (v * ((p - t) ** 2).sum(-1)).sum(1))
    _close(ws[:, 1], (v * (1 - F.cosine_similarity(p, t, dim=-1, eps=R.COS_EPS))).sum(1))
    out, _ = R.kd_out3(ws, bws, L, Dm, masked, 0.7)
    _close(out[0], R.kd_loss64(p, t, pd, 0.7))
    if not masked:
        _close(out[1], F.mse_loss(p, t))
    ref, bound = R.kd_bwd(p, t, pd, ws[:, 2], 0.7, 3.0)
    pr = p.clone().requires_grad_(True)
    (gp,) = torch.autograd.grad(3.0 * R.kd_loss64(pr, t, pd, 0.7), pr)
    _close(ref, gp)
    if masked:
        assert (ref[pad] == 0).all()
    for tok in ((0, 0), (0, 1), (0, 2)):                       # p = 0, |p| = 1e-9, an ordinary token
        a, b = p[tok], t[tok]
        pa = a.clone().requires_grad_(True)
        (gc,) = torch.autograd.grad(F.cosine_similarity(pa, b, dim=0, eps=R.COS_EPS), pa)
        npc, ntc = max(a.norm().item(), R.COS_EPS), max(b.norm().item(), R.COS_EPS)
        cp = (a @ b) / (npc * npc * ntc * a.norm()) if a.norm() > 0 else 0.0
        mine = b / (npc * ntc) - a * cp
        assert torch.allclose(mine, gc, rtol=1e-12, atol=1e-12 * gc.abs().max().item()), tok


def test_consistency_statements():
    g = _g("con")
    B, L, Dm = 3, 5, 7
    p, q = torch.randn(B, L, Dm, generator=g, dtype=D), torch.randn(B, L, Dm, generator=g, dtype=D)
    r = R.consistency_fwd(p, q, 0.3, torch.tensor(1.5, dtype=D))
    _close(r["value"][0][0], F.mse_loss(p.mean(1), q.mean(1)))
    _close(r["loss"][0][0], 1.5 + 0.3 * F.mse_loss(p.mean(1), q.mean(1)))
    dp0 = torch.randn(B, L, Dm, generator=g, dtype=D)
    b = R.consistency_bwd(r["mdiff"][0], L, 0.3, 2.0, dp0)
    gp, gq = _grads(lambda a, c: 2.0 * 0.3 * F.mse_loss(a.mean(1), c.mean(1)), [p, q], torch.tensor(1.0, dtype=D))
    _close(b["dp"][0], dp0 + gp)
    _close(b["dq"][0], gq)


# ----------------------------------------------------------------------------------------------------------- RepMixerBlock backward
def _bn(v, gamma, beta, rm, rv):
    return gamma * (v - rm) / torch.sqrt(rv + 1e-5) + beta


def _bn_pack(gamma, beta, rm, rv):
    inv = 1 / torch.sqrt(rv + 1e-5)
    s = gamma * inv
    return torch.stack([s, beta - rm * s, rm, inv])


def test_repmixer_bwd_statements():
    """The frozen-BN RepMixerBlock backward statements, on taps and packed (s, b, rm, invstd) rows, against float64 autograd of the
    block's pieces written with nn.BatchNorm's eval formula: x2 = x1 + ls y (+ the fc2 bias inside ls y), u = BN_f(dw(x1; w_f)),
    x1 = x + ls_tm (BN_ms(x) + BN_mc(dw(x; w_mc)) - BN_ns(x)); every gradient accumulates into a prior value."""
    g = _g("rmb")
    B, L, C = 2, 13, 32
    r = lambda *s: torch.randn(*s, generator=g, dtype=D)
    bns = [(r(C), r(C), r(C), torch.rand(C, generator=g, dtype=D) + 0.5) for _ in range(4)]     # ms, mc, ns, f
    x, x1, gg, du, y, e = (r(B * L, C) for _ in range(6))
    ls, ls_tm, wf, wmc = r(C), r(C), r(11, C) * 0.3, r(11, C) * 0.3

    def dw(v, w):
        t = v.view(B, L, C).permute(0, 2, 1)
        return F.conv1d(t, w.t().unsqueeze(1), padding=5, groups=C).permute(0, 2, 1).reshape(B * L, C)

    dls0, db0 = r(C), r(C)
    o = R.repmixer_ls_bwd(gg, y, ls, B, L, dls0, db0)
    _close(o["dy"][0], ls * gg)
    _close(o["dls"][0], dls0 + (gg * y).sum(0))
    _close(o["dbias"][0], db0 + (ls * gg).sum(0))

    dwf0, dgf0, dbf0 = r(C, 11), r(C), r(C)
    bnf = _bn_pack(*bns[3])
    o = R.repmixer_ffn_bwd(x1, du, gg, wf, bnf, B, L, dwf0, dgf0, dbf0)
    gx, gw, ggm, gbt = _grads(lambda a, w, gm, bt: (du * _bn(dw(a, w), gm, bt, bns[3][2], bns[3][3])).sum() + (gg * a).sum(),
                              [x1, wf, bns[3][0], bns[3][1]], torch.tensor(1.0, dtype=D))
    _close(o["e"][0], gx)
    _close(o["dwf"][0], dwf0 + gw.t())
    _close(o["dgamma"][0], dgf0 + ggm)
    _close(o["dbeta"][0], dbf0 + gbt)

    bnp = torch.cat([_bn_pack(*bns[0]), _bn_pack(*bns[1]), _bn_pack(*bns[2]), ls_tm[None]])
    dwmc0, dlt0 = r(C, 11), r(C)
    dbn0 = [r(C) for _ in range(6)]
    o = R.repmixer_tm_bwd(x, e, wmc, bnp, B, L, dwmc0, dlt0, dbn0)

    def tm(a, w, lt, g0, b0, g1, b1, g2, b2):
        mix = _bn(a, g0, b0, *bns[0][2:]) + _bn(dw(a, w), g1, b1, *bns[1][2:]) - _bn(a, g2, b2, *bns[2][2:])
        return (e * (a + lt * mix)).sum()
    grads = _grads(tm, [x, wmc, ls_tm, bns[0][0], bns[0][1], bns[1][0], bns[1][1], bns[2][0], bns[2][1]], torch.tensor(1.0, dtype=D))
    _close(o["dx"][0], grads[0])
    _close(o["dwmc"][0], dwmc0 + grads[1].t())
    _close(o["dls"][0], dlt0 + grads[2])
    for name, i, k in (("dg_ms", 3, 0), ("db_ms", 4, 1), ("dg_mc", 5, 2), ("db_mc", 6, 3), ("dg_ns", 7, 4), ("db_ns", 8, 5)):
        _close(o[name][0], dbn0[k] + grads[i], name)
    for v in o.values():
        assert (v[1] > 0).all()
