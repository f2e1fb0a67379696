"""The fp64 statements of tests/ref_sam.py against textbook float64 torch (F.scaled_dot_product_attention, F.layer_norm, F.gelu,
F.conv2d, F.interpolate) and oracle/sam_heads.py (dense_pe, _embed_coords, mask_downscaling, layernorm2d), and the bound logic on
constructed cases: fp32 executions of the kernels' arithmetic -- lanes that hold no key, a peaked softmax, a flat LayerNorm patch at
rstd = 1 / sqrt(eps), a bilinear sample on a source pixel -- lie within the bounds.  No GPU."""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

import ref_sam as R
from oracle import sam_heads as O

D = torch.float64


def _g(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _within(ref, bound, other, what):
    err = (ref - other).abs()
    assert (err <= bound).all(), f"{what}: {int((err > bound).sum())} elements outside the bound (max err/bound {(err / bound).max():.3g})"
    assert (bound > 0).all()


def _close(a, b, what="", tol=1e-10):
    assert torch.allclose(a, b, rtol=tol, atol=tol), (what, (a - b).abs().max().item())


def _f32(t):
    return t.float().double()


# ----------------------------------------------------------------------------------------------------------- positional encodings
def test_dense_pe_statement():
    g = _f32(torch.randn(2, 64, generator=_g("pe")) * 3)
    ref, bound = R.dense_pe(g, 9, 7)
    ys, xs = torch.meshgrid((torch.arange(9, dtype=D) + 0.5) / 9, (torch.arange(7, dtype=D) + 0.5) / 7, indexing="ij")
    a = 2 * math.pi * (torch.stack([xs, ys], -1).reshape(-1, 2) * 2 - 1) @ g
    _close(ref, torch.cat([a.sin(), a.cos()], -1), "dense_pe")
    orc = O.dense_pe({"pe_layer.positional_encoding_gaussian_matrix": g.float()}, "", 9, 7)[0].permute(1, 2, 0).reshape(63, 128)
    _within(ref, bound + 2e-6, orc.double(), "dense_pe vs the fp32 oracle")
    assert bound.max() < 1e-4


def test_point_embed_statement_and_labels():
    """Labels -1 (not_a_point exactly), 0..3 (their row added), 4 and -2 (the pe unchanged), the padding point; against
    oracle._embed_coords on the +0.5 coordinates."""
    g = _f32(torch.randn(2, 64, generator=_g("pt")))
    nap, rows = _f32(torch.randn(128, generator=_g("nap"))), _f32(torch.randn(4, 128, generator=_g("rows")))
    coords = _f32(torch.tensor([[[0.0, 0.0], [1007.0, 1007.0], [-5.0, 12.0], [1100.0, 300.0], [500.0, 20.0], [3.0, 4.0], [7.0, 9.0]]]))
    labels = torch.tensor([[-1, 0, 1, 2, 3, 4, -2]])
    ref, bound, exact = R.point_embed(coords, labels, g, nap, rows, 1008.0, 1008.0, pad=True)
    assert ref.shape == (1, 8, 128) and bool(exact[0, 0].all()) and bool(exact[0, 7].all()) and not bool(exact[0, 1:7].any())
    _close(ref[0, 0], nap)
    _close(ref[0, 7], nap)
    pe, _ = R.pe(g, (coords[..., 0] + 0.5) / 1008, (coords[..., 1] + 0.5) / 1008)
    for i in range(4):
        _close(ref[0, 1 + i], pe[0, 1 + i] + rows[i])
    _close(ref[0, 5:7], pe[0, 5:7])
    sd = {"pe_layer.positional_encoding_gaussian_matrix": g.float(), "not_a_point_embed.weight": nap.float()[None],
          **{f"point_embeddings.{i}.weight": rows[i].float()[None] for i in range(4)}}
    orc = O._embed_coords(sd, "", coords.float() + 0.5, labels, (1008, 1008))
    _within(ref[:, :7], bound[:, :7] + 1e-5, orc.double(), "point_embed vs the fp32 oracle")
    # dropping the +0.5 pixel-centre offset moves the angle far outside the bound
    moved, _ = R.pe(g, coords[..., 0] / 1008, coords[..., 1] / 1008)
    assert ((moved[0, 5] - pe[0, 5]).abs() > bound[0, 5]).any()


# ----------------------------------------------------------------------------------------------------------- attention
def _fp32_few_queries(q, k, v, heads, scale):
    """The few-query kernel's arithmetic in fp32 (torch.exp for __expf): lane j holds keys j, j + 32, ..., merged like the warp."""
    B, Tq, Dm = q.shape
    Tk, hd = k.shape[1], Dm // heads
    qh = (q.float() * scale).reshape(B, Tq, heads, hd).transpose(1, 2)
    kh, vh = (t.float().reshape(B, Tk, heads, hd).transpose(1, 2) for t in (k, v))
    nl = -(-Tk // 32)
    m = torch.full((B, heads, Tq, 32), -math.inf)
    l = torch.zeros(B, heads, Tq, 32)
    acc = torch.zeros(B, heads, Tq, 32, hd)
    for step in range(nl):
        js = torch.arange(step * 32, min(Tk, step * 32 + 32))
        n = js.numel()
        s = qh @ kh[:, :, js].transpose(-1, -2)                            # [B, h, Tq, n]
        mn = torch.maximum(m[..., :n], s)
        corr, p = torch.exp(m[..., :n] - mn), torch.exp(s - mn)
        l[..., :n] = l[..., :n] * corr + p
        acc[..., :n, :] = p[..., None] * vh[:, :, js][:, :, None] + acc[..., :n, :] * corr[..., None]
        m[..., :n] = mn
    mw = m.amax(-1, keepdim=True)
    f = torch.where(m == -math.inf, torch.zeros(()), torch.exp(m - mw))
    y = (acc * f[..., None]).sum(-2) / (l * f).sum(-1, keepdim=True)
    return y.transpose(1, 2).reshape(B, Tq, Dm).double()


def _fp32_few_keys(q, k, v, heads, scale, strict):
    B, Nq, Dm = q.shape
    Tk, hd = k.shape[1], Dm // heads
    qh = q.float().reshape(B, Nq, heads, hd).transpose(1, 2)
    kh, vh = (t.float().reshape(B, Tk, heads, hd).transpose(1, 2) for t in (k, v))
    if strict:
        s = (qh @ kh.transpose(-1, -2)) * scale
        p = torch.exp(s - s.amax(-1, keepdim=True))
        l = torch.zeros(p.shape[:-1] + (1,))
        for t in range(Tk):
            l = l + p[..., t:t + 1]
        y = (p * (1 / l)) @ vh
    else:
        s = (qh * scale) @ kh.transpose(-1, -2)
        mx, l, o = torch.full(s.shape[:-1] + (1,), -math.inf), torch.zeros(s.shape[:-1] + (1,)), torch.zeros(qh.shape)
        for t in range(Tk):
            a = s[..., t:t + 1]
            mn = torch.maximum(mx, a)
            corr, p = torch.exp(mx - mn), torch.exp(a - mn)
            l = l * corr + p
            o = p * vh[:, :, t:t + 1] + o * corr
            mx = mn
        y = (o / l).to(torch.bfloat16).float()
    return y.transpose(1, 2).reshape(B, Nq, Dm).double()


def _qkv(kind, B, Nq, Tk, Dm, g):
    q, k, v = (torch.randn(B, n, Dm, generator=g, dtype=D) for n in (Nq, Tk, Tk))
    if kind == "peaked":
        q, k = q * 6, k * 6
    elif kind == "flat":
        q = q * 0
    elif kind == "tied":
        k = k[:, torch.arange(Tk) % 3]
    return q, k, v


@pytest.mark.parametrize("Tk", [1, 5, 31, 32, 33, 100])
@pytest.mark.parametrize("kind", ["random", "peaked", "flat", "tied"])
def test_attn_few_queries_statement(Tk, kind):
    """Against F.scaled_dot_product_attention; an fp32 execution of the lane-strided softmax and its merge lies within the bound,
    Tk < 32 (lanes without a key, f = 0) included."""
    q, k, v = _qkv(kind, 2, 7, Tk, 32, _g("fq", Tk, kind))
    k, v = (t.to(torch.bfloat16).double() for t in (k, v))
    q = _f32(q)
    ref, bound = R.attn_few_queries(q, k, v, 2, 16 ** -0.5)
    _close(ref, R._sdpa(q, k, v, 2, 16 ** -0.5), "few_queries vs sdpa")
    _within(ref, bound, _fp32_few_queries(q, k, v, 2, 16 ** -0.5), f"fp32 few_queries Tk{Tk} {kind}")


@pytest.mark.parametrize("Tk", [1, 7, 16, 17, 33])
@pytest.mark.parametrize("kind", ["random", "peaked", "flat", "tied"])
@pytest.mark.parametrize("strict", [False, True])
def test_attn_few_keys_statement(Tk, kind, strict):
    q, k, v = _qkv(kind, 2, 40, Tk, 32, _g("fk", Tk, kind))
    q = q.to(torch.bfloat16).double() if not strict else _f32(q)
    k, v = _f32(k), _f32(v)
    ref, bound = R.attn_few_keys(q, k, v, 2, 0.25, strict)
    _close(ref, R._sdpa(q, k, v, 2, 0.25), "few_keys vs sdpa")
    _within(ref, bound, _fp32_few_keys(q, k, v, 2, 0.25, strict), f"fp32 few_keys Tk{Tk} {kind} strict={strict}")


def test_peaked_softmax_bound_stays_at_the_output_rounding():
    """A near one-hot row: the result is the winning value, and the bf16-mode bound is dominated by the output's half-step."""
    q, k, v = _qkv("peaked", 1, 8, 16, 16, _g("peak"))
    q = q.to(torch.bfloat16).double()
    k, v = _f32(k * 5), _f32(v)
    ref, bound = R.attn_few_keys(q, k, v, 1, 0.25, False)
    inner = bound - 2.0 ** -8 * ref.abs()
    assert (inner <= 1e-2 * v.abs().amax() + 2.0 ** -8 * bound).all()


# ----------------------------------------------------------------------------------------------------------- LayerNorm + GELU
def _fp32_ln_gelu(x, w, b, eps, strict):
    xf = x.float()
    mu = xf.sum(1, keepdim=True) / x.shape[1]
    d = xf - mu
    rstd = 1 / torch.sqrt((d * d).sum(1, keepdim=True) / x.shape[1] + eps)
    y = F.gelu(d * rstd * w.float() + b.float())
    return y.double() if strict else y.to(torch.bfloat16).double()


@pytest.mark.parametrize("kind", ["random", "constant", "shifted", "near_flat"])
@pytest.mark.parametrize("strict", [False, True])
def test_ln_rows_gelu_statement(kind, strict):
    """Against F.layer_norm + F.gelu; constant rows (variance 0: rstd = 1 / sqrt(eps) = 1000, y = gelu(b)), rows whose mean is 1000x
    their spread, and rows whose variance is comparable to eps: an fp32 execution lies within the bound."""
    g = _g("ln", kind)
    M, C = 40, 64
    x = torch.randn(M, C, generator=g, dtype=D)
    if kind == "constant":
        x = x[:, :1].expand(M, C).clone()
    elif kind == "shifted":
        x = x * 1e-2 + 10.0
    elif kind == "near_flat":
        x = x * 1e-3 + 0.3
    x, w, b = _f32(x), _f32(torch.randn(C, generator=g, dtype=D)), _f32(torch.randn(C, generator=g, dtype=D))
    ref, bound = R.ln_rows_gelu(x, w, b, 1e-6, strict)
    _close(ref, F.gelu(F.layer_norm(x, (C,), w, b, 1e-6)), "ln_rows_gelu", 1e-9)
    _within(ref, bound, _fp32_ln_gelu(x, w, b, 1e-6, strict), f"fp32 ln_rows_gelu {kind}")
    if kind == "near_flat":                    # eps x 10 moves the output far outside the bound
        other, _ = R.ln_rows_gelu(x, w, b, 1e-5, strict)
        assert ((other - ref).abs() > bound).float().mean() > 0.5
    if kind == "random":                       # the variance over C - 1 does too
        unb = F.gelu((x - x.mean(1, keepdim=True)) / (x.var(1, keepdim=True) + 1e-6).sqrt() * w + b)
        assert ((unb - ref).abs() > bound).any()


# ----------------------------------------------------------------------------------------------------------- mask tail
def test_hyper_masks_statement_and_gate():
    g = _g("hm")
    up, hyper = _f32(torch.randn(4, 300, 32, generator=g, dtype=D)), _f32(torch.randn(4, 4, 32, generator=g, dtype=D))
    obj = torch.tensor([1.0, 0.0, -0.0, float("nan")], dtype=D)
    ref, bound, gated = R.hyper_masks(up, hyper, obj, -1024.0, 3, 1)
    assert gated.reshape(-1).tolist() == [False, True, True, True]
    _close(ref[0], torch.einsum("kc,pc->kp", hyper[0, 1:], up[0]))
    assert (ref[1:] == -1024.0).all() and (bound[1:] == 0).all()
    # the oracle's gate is where(obj > 0, masks, NO_OBJ_SCORE): the same rule
    assert torch.equal(torch.where(obj.reshape(-1, 1, 1) > 0, ref, torch.full_like(ref, O.NO_OBJ_SCORE)), ref)
    short = torch.einsum("kc,pc->kp", hyper[0, 1:, :31], up[0, :, :31])            # a sum that drops channel 31
    assert ((short - ref[0]).abs() > bound[0]).float().mean() > 0.5


def _fp32_bilinear(x, Ho, Wo):
    """es3_bilinear_nchw_f32's arithmetic in fp32."""
    P, Hi, Wi = x.shape
    xf = x.float()
    sy, sx = torch.tensor(Hi / Ho, dtype=torch.float32), torch.tensor(Wi / Wo, dtype=torch.float32)
    fy = ((torch.arange(Ho, dtype=torch.float32) + 0.5) * sy - 0.5).clamp_min(0)
    fx = ((torch.arange(Wo, dtype=torch.float32) + 0.5) * sx - 0.5).clamp_min(0)
    y0, x0 = fy.long().clamp_max(Hi - 1), fx.long().clamp_max(Wi - 1)
    y1, x1 = (y0 + 1).clamp_max(Hi - 1), (x0 + 1).clamp_max(Wi - 1)
    ly, lx = (fy - y0)[:, None], (fx - x0)[None, :]
    g = lambda yy, xx: xf[:, yy][:, :, xx]
    v = (1 - ly) * ((1 - lx) * g(y0, x0) + lx * g(y0, x1)) + ly * ((1 - lx) * g(y1, x0) + lx * g(y1, x1))
    return v.double()


@pytest.mark.parametrize("Hi,Wi,Ho,Wo", [(12, 12, 42, 42), (12, 12, 13, 17), (12, 12, 5, 3), (9, 9, 3, 3), (7, 5, 7, 5), (16, 16, 9, 9)])
def test_bilinear_statement(Hi, Wi, Ho, Wo):
    """Against F.interpolate(align_corners=False) by the textbook formula; an fp32 execution lies within the bound; a 3x downscale
    samples exactly on source pixels; the identity is the input."""
    x = _f32(torch.randn(3, Hi, Wi, generator=_g("bl", Hi, Ho, Wo), dtype=D) * 4)
    ref, bound = R.bilinear(x, Ho, Wo)
    _within(ref, bound, _fp32_bilinear(x, Ho, Wo), f"fp32 bilinear {Hi}x{Wi} -> {Ho}x{Wo}")
    fy = ((torch.arange(Ho, dtype=D) + 0.5) * Hi / Ho - 0.5).clamp_min(0)
    fx = ((torch.arange(Wo, dtype=D) + 0.5) * Wi / Wo - 0.5).clamp_min(0)
    y0, x0 = fy.floor().long(), fx.floor().long()
    y1, x1 = (y0 + 1).clamp_max(Hi - 1), (x0 + 1).clamp_max(Wi - 1)
    ly, lx = (fy - y0)[:, None], (fx - x0)[None, :]
    g = lambda yy, xx: x[:, yy][:, :, xx]
    _close(ref, (1 - ly) * ((1 - lx) * g(y0, x0) + lx * g(y0, x1)) + ly * ((1 - lx) * g(y1, x0) + lx * g(y1, x1)))
    if (Hi, Ho) == (9, 3):
        assert torch.equal(ref, x[:, 1::3, 1::3])
    if (Hi, Wi) == (Ho, Wo):
        assert torch.equal(ref, x)
    if Wo > Wi:                  # clamping fx after the floor: column 0 extrapolates with lx = fx < 0, outside the bound
        lx0 = 0.5 * Wi / Wo - 0.5
        rows = R.bilinear(x, Ho, Wi)[0]
        moved = (1 - lx0) * rows[:, :, 0] + lx0 * rows[:, :, 1]
        assert ((moved - ref[:, :, 0]).abs() > bound[:, :, 0]).any()


# ----------------------------------------------------------------------------------------------------------- mask prompt
def _mask_sd(g, C, flat=False):
    sd = {"mask_downscaling.0.weight": torch.randn(4, 1, 2, 2, generator=g) * 0.5, "mask_downscaling.0.bias": torch.randn(4, generator=g),
          "mask_downscaling.1.weight": torch.randn(4, generator=g) + 1, "mask_downscaling.1.bias": torch.randn(4, generator=g) * 0.1,
          "mask_downscaling.3.weight": torch.randn(16, 4, 2, 2, generator=g) * 0.3, "mask_downscaling.3.bias": torch.randn(16, generator=g),
          "mask_downscaling.4.weight": torch.randn(16, generator=g) + 1, "mask_downscaling.4.bias": torch.randn(16, generator=g) * 0.1,
          "mask_downscaling.6.weight": torch.randn(C, 16, 1, 1, generator=g) * 0.25, "mask_downscaling.6.bias": torch.randn(C, generator=g)}
    if flat:                                   # the first LayerNorm sees a spread comparable to sqrt(eps)
        sd["mask_downscaling.0.weight"] *= 1e-3
        sd["mask_downscaling.0.bias"] = 0.5 + 1e-3 * torch.randn(4, generator=g)
    return {k: _f32(v) for k, v in sd.items()}


def mask_wts(sd):
    q = "mask_downscaling."
    return (sd[q + "0.weight"].reshape(4, 4), sd[q + "0.bias"], sd[q + "1.weight"], sd[q + "1.bias"], sd[q + "3.weight"].reshape(16, 16),
            sd[q + "3.bias"], sd[q + "4.weight"], sd[q + "4.bias"], sd[q + "6.weight"].reshape(-1, 16), sd[q + "6.bias"])


@pytest.mark.parametrize("kind", ["random", "saturated", "flat"])
def test_mask_downscale_statement(kind):
    """Against oracle.mask_downscaling (F.conv2d, layernorm2d, F.gelu) in float64 and an fp32 execution of the same graph; the
    flat case puts the first LayerNorm's variance near eps, where eps x 10 leaves the bound."""
    g = _g("md", kind)
    sd = _mask_sd(g, 32, flat=kind == "flat")
    B, h, w = 2, 5, 7
    m = torch.randn(B, 1, 4 * h, 4 * w, generator=g, dtype=D) * 3
    if kind == "saturated":
        m = torch.where(m > 0, 1024.0, -1024.0).to(D)
    elif kind == "flat":
        m = torch.full_like(m, 0.25)
    m = _f32(m)
    base = _f32(torch.randn(h * w, 32, generator=g, dtype=D))
    ref, bound = R.mask_downscale(m, mask_wts(sd), 1e-6, base)
    orc = O.mask_downscaling(sd, "", m).permute(0, 2, 3, 1).reshape(B * h * w, 32) + base.repeat(B, 1)
    _close(ref, orc, "mask_downscale vs the oracle", 1e-9)
    sd32 = {k: v.float() for k, v in sd.items()}
    f32 = O.mask_downscaling(sd32, "", m.float()).permute(0, 2, 3, 1).reshape(B * h * w, 32) + base.float().repeat(B, 1)
    _within(ref, bound, f32.double(), f"fp32 mask_downscale {kind}")
    ln = O.layernorm2d(sd, "mask_downscaling.1", F.conv2d(m, sd["mask_downscaling.0.weight"], sd["mask_downscaling.0.bias"], stride=2))
    t = F.conv2d(m, sd["mask_downscaling.0.weight"], sd["mask_downscaling.0.bias"], stride=2)
    _close(ln, F.layer_norm(t.permute(0, 2, 3, 1), (4,), sd["mask_downscaling.1.weight"], sd["mask_downscaling.1.bias"], 1e-6)
           .permute(0, 3, 1, 2), "layernorm2d")
    if kind == "flat":
        other, _ = R.mask_downscale(m, mask_wts(sd), 1e-5, base)
        assert ((other - ref).abs() > bound).float().mean() > 0.25
