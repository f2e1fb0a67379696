"""The fp64 statements of tests/ref_strict.py against textbook float64 torch (F.conv2d with groups = C and tests/emu_strict.py,
F.interpolate, oracle/efficientvit.py's LiteMLA), float32 restatements of each strict student kernel's arithmetic order inside
their bounds, and restatements with a known fault outside them: a depthwise tap shifted by one row at a stride-2 border, the scale
dropped on one channel, a LiteMLA chunk that skips its last 32-pixel block, the bilinear x and y weights swapped, and the
activation applied on the wrong side of the residual.  No GPU."""
import zlib

import pytest
import torch
import torch.nn.functional as F

import emu_strict as E
import ref_strict as R

D = torch.float64


def _g(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _close(a, b, what=""):
    assert torch.allclose(a, b, rtol=1e-12, atol=1e-12), (what, (a - b).abs().max().item())


def _within(ref, bound, other, what):
    err = (ref - other).abs()
    assert (err <= bound).all(), f"{what}: {int((err > bound).sum())} elements outside the bound (max err/bound {(err / bound).max():.3g})"
    assert (bound > 0).all()


def _outside(ref, bound, other, what):
    assert ((ref - other).abs() > bound).any(), f"{what}: the fault stays inside the bound"


def _f32_act(v, act):
    return E._act(v, act)


# ----------------------------------------------------------------------------------------------------------- depthwise
def dwconv_f32(x, w, scale, bias, ks, stride, act, shift_top_row=False, drop_scale_at=None):
    """es3_dwconv_f32 in float32: the taps in (ky, kx) order from 0 (a product and a sum each, no fma), then scale, bias and act.
    shift_top_row: output row 0 reads every tap one source row lower; drop_scale_at: channel whose scale is not applied."""
    B, H, W, C = x.shape
    p = ks // 2
    Ho, Wo = (H + 2 * p - ks) // stride + 1, (W + 2 * p - ks) // stride + 1
    xp = F.pad(x, (0, 0, p, p + 1, p, p))                                        # one spare row below for the shifted tap
    acc = torch.zeros(B, Ho, Wo, C, dtype=torch.float32)
    for ky in range(ks):
        for kx in range(ks):
            t = xp[:, ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride].clone()
            if shift_top_row:
                t[:, 0] = xp[:, ky + 1, kx:kx + stride * (Wo - 1) + 1:stride]
            acc = acc + t * w[ky * ks + kx]
    if scale is not None:
        s = scale.clone()
        if drop_scale_at is not None:
            s[drop_scale_at] = 1.0
        acc = acc * s
    if bias is not None:
        acc = acc + bias
    return _f32_act(acc, act)


def _dw_case(B, H, W, C, ks, stride, seed):
    g = _g("dw", B, H, W, C, ks, stride, seed)
    x = torch.randn(B, H, W, C, generator=g)
    w = torch.randn(ks * ks, C, generator=g) / ks
    return x, w, torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)


@pytest.mark.parametrize("B,H,W,C,ks,stride,act", [(2, 9, 11, 5, 3, 1, "hswish"), (1, 7, 8, 3, 5, 2, "gelu"), (2, 2, 3, 4, 7, 1, None),
                                                   (1, 6, 5, 16, 3, 2, "relu")])
def test_dwconv_statement(B, H, W, C, ks, stride, act):
    """Against F.conv2d(groups = C) through emu_strict.dwconv_f32; the float32 restatement inside the bound."""
    x, w, sc, bi = _dw_case(B, H, W, C, ks, stride, 0)
    ref, bound = R.dwconv(x.double(), w.double(), sc.double(), bi.double(), ks, stride, act)
    _close(ref, E.dwconv_f32(x.double(), w.double(), sc.double(), bi.double(), ks, stride, act))
    _within(ref, bound, dwconv_f32(x, w, sc, bi, ks, stride, act).double(), "fp32 dwconv")


def test_valid_taps_counts_the_border():
    n = R.valid_taps(1, 5, 6, 3, 2, torch.zeros(1, dtype=D))
    assert n.shape == (1, 3, 3, 1) and n[0, 0, 0, 0] == 4 and n[0, 1, 1, 0] == 9 and n[0, 2, 2, 0] == 6


def test_dwconv_faults_leave_the_bound():
    """A tap shifted by one row on the top border at stride 2, and the scale dropped on one channel."""
    x, w, sc, bi = _dw_case(2, 9, 9, 8, 3, 2, 1)
    ref, bound = R.dwconv(x.double(), w.double(), sc.double(), bi.double(), 3, 2, "hswish")
    _within(ref, bound, dwconv_f32(x, w, sc, bi, 3, 2, "hswish").double(), "fp32 dwconv")
    _outside(ref, bound, dwconv_f32(x, w, sc, bi, 3, 2, "hswish", shift_top_row=True).double(), "tap shifted at the border")
    _outside(ref, bound, dwconv_f32(x, w, sc, bi, 3, 2, "hswish", drop_scale_at=5).double(), "scale dropped on channel 5")


# ----------------------------------------------------------------------------------------------------------- LiteMLA
def litemla_f32(ms, B, HW, heads, dim, eps, skip_last_block=False):
    """es3_litemla_attn_f32 in float32: per chunk a running sum over its pixels (product and sum, no fma), the chunks summed in
    order, then num and den as running sums over j and out = num * (1 / (den + eps)).  skip_last_block: chunk 0 leaves out its
    last 32 pixels."""
    chunk, nch = R.litemla_chunks(HW)
    t = ms.view(B, HW, -1)
    out = torch.empty(B, HW, heads * dim, dtype=torch.float32)
    for h in range(heads):
        c = 3 * dim * h
        q, k, v = F.relu(t[..., c:c + dim]), F.relu(t[..., c + dim:c + 2 * dim]), t[..., c + 2 * dim:c + 3 * dim]
        v1 = torch.cat([v, torch.ones_like(v[..., :1])], -1)
        kv = torch.zeros(B, dim + 1, dim, dtype=torch.float32)
        for ch in range(nch):
            p0, p1 = ch * chunk, min(HW, (ch + 1) * chunk)
            if skip_last_block and ch == 0:
                p1 = p0 + ((p1 - p0 - 1) // 32) * 32
            part = torch.zeros_like(kv)
            for p in range(p0, p1):
                part = part + v1[:, p, :, None] * k[:, p, None, :]
            kv = kv + part
        nd = torch.zeros(B, HW, dim + 1, dtype=torch.float32)
        for j in range(dim):
            nd = nd + kv[:, None, :, j] * q[:, :, j, None]
        out[..., dim * h:dim * (h + 1)] = nd[..., :dim] * (1.0 / (nd[..., dim:] + eps))
    return out.view(B * HW, -1)


def _ms(B, HW, heads, dim, seed):
    ms = torch.randn(B * HW, 3 * dim * heads, generator=_g("ms", B, HW, heads, dim, seed))
    ms[3::7, :dim] = -ms[3::7, :dim].abs() - 0.1                                 # head 0's q all negative on every 7th pixel
    return ms


def test_litemla_statement_against_the_oracle():
    """oracle/efficientvit.py's lite_mla with identity qkv, aggregation and projection weights runs its attention on ms = (x, x):
    the statement on the same ms agrees to 1e-12."""
    from oracle import efficientvit as O
    B, H, W, heads, dim = 2, 6, 7, 2, 8
    c3 = 3 * dim * heads
    x = torch.randn(B, c3, H, W, generator=_g("oracle mla"), dtype=D)
    agg = torch.zeros(c3, 1, 5, 5, dtype=D)
    agg[:, 0, 2, 2] = 1.0
    gs = c3 // (3 * heads)
    sd = {"m.qkv.conv.weight": torch.eye(c3, dtype=D)[:, :, None, None], "m.aggreg.0.0.weight": agg,
          "m.aggreg.0.1.weight": torch.eye(gs, dtype=D).repeat(3 * heads, 1)[:, :, None, None],
          "m.proj.conv.weight": torch.eye(2 * dim * heads, dtype=D)[:, :, None, None]}
    want = O.lite_mla(sd, "m", x, dim).permute(0, 2, 3, 1).reshape(B * H * W, -1)
    xs = x.permute(0, 2, 3, 1).reshape(B * H * W, c3)
    ref, _ = R.litemla_attn(torch.cat([xs, xs], 1), B, H * W, 2 * heads, dim, 1e-15)
    _close(ref, want)


@pytest.mark.parametrize("B,HW,heads,dim", [(2, 31, 2, 16), (1, 2049, 1, 16), (1, 100, 3, 32)])
def test_litemla_statement(B, HW, heads, dim):
    """Against emu_strict.litemla_attn_f32 (the textbook (v1 k^T) q form); the float32 restatement inside the bound, the pixels
    whose q is all negative exactly 0 in both."""
    ms = _ms(B, HW, heads, dim, 0)
    ref, bound = R.litemla_attn(ms.double(), B, HW, heads, dim, 1e-15)
    emu = E.litemla_attn_f32(ms.double().view(B, HW, 1, -1), heads, dim, 1e-15).reshape(B * HW, -1)
    _close(ref, emu)
    f32 = litemla_f32(ms, B, HW, heads, dim, 1e-15)
    _within(ref, bound, f32.double(), "fp32 LiteMLA")
    assert (ref[3::7, :dim] == 0).all() and (f32[3::7, :dim] == 0).all()


def test_litemla_chunk_rule():
    assert [R.litemla_chunks(n) for n in (1, 31, 2048, 2049, 4096, 6145)] == [(32, 1), (32, 1), (2048, 1), (1056, 2), (2048, 2),
                                                                               (1568, 4)]


def test_litemla_fault_leaves_the_bound():
    """A chunk that skips its last 32-pixel block, at HW = 2049 (two chunks of 1056 and 993 pixels)."""
    B, HW, heads, dim = 1, 2049, 1, 16
    ms = _ms(B, HW, heads, dim, 1)
    ref, bound = R.litemla_attn(ms.double(), B, HW, heads, dim, 1e-15)
    _outside(ref, bound, litemla_f32(ms, B, HW, heads, dim, 1e-15, skip_last_block=True).double(), "chunk 0 skips its last block")


# ----------------------------------------------------------------------------------------------------------- bilinear
def bilinear_f32(x, Ho, Wo, swap=False):
    """es3_bilinear_nhwc_f32_to_nchw in float32 at the kernel's fp32 weights (no contraction); swap: the y weights used along x and
    the x weights along y."""
    B, Hi, Wi, C = x.shape
    y0, y1, ly, hy, _ = R.source_coords(Hi, Ho)
    x0, x1, lx, hx, _ = R.source_coords(Wi, Wo)
    ly, hy, lx, hx = (t.float() for t in (ly, hy, lx, hx))
    if swap:
        n = min(Ho, Wo)
        ly, lx = torch.cat([lx[:n], ly[n:]]), torch.cat([ly[:n], lx[n:]])
        hy, hx = 1 - ly, 1 - lx
    at = lambda yi, xi: x[:, yi][:, :, xi]
    Y, X = (lambda t: t.view(1, -1, 1, 1)), (lambda t: t.view(1, 1, -1, 1))
    y = Y(hy) * (X(hx) * at(y0, x0) + X(lx) * at(y0, x1)) + Y(ly) * (X(hx) * at(y1, x0) + X(lx) * at(y1, x1))
    return y.permute(0, 3, 1, 2)


@pytest.mark.parametrize("Hi,Wi,Ho,Wo", [(4, 6, 8, 12), (8, 8, 4, 4), (3, 5, 12, 20), (16, 2, 4, 1)])
def test_bilinear_statement_exact_coordinates(Hi, Wi, Ho, Wo):
    """Scale factors that are powers of two put the fp32 source coordinates exactly where the fp64 ones are: the statement agrees
    with F.interpolate(align_corners=False) to 1e-12."""
    x = torch.randn(2, Hi, Wi, 3, generator=_g("bil", Hi, Wi, Ho, Wo), dtype=D)
    ref, _ = R.bilinear(x, Ho, Wo)
    _close(ref, F.interpolate(x.permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear", align_corners=False))


@pytest.mark.parametrize("Hi,Wi,Ho,Wo", [(10, 10, 12, 12), (7, 13, 20, 5), (23, 23, 9, 9), (1, 1, 6, 4), (9, 1, 1, 1), (32, 32, 64, 64)])
def test_bilinear_statement(Hi, Wi, Ho, Wo):
    """At any size the statement is F.interpolate up to the fp32 rounding of the weights (a few u of the values), and the float32
    restatement lies inside the bound."""
    x = torch.randn(2, Hi, Wi, 5, generator=_g("bil", Hi, Wi, Ho, Wo))
    ref, bound = R.bilinear(x.double(), Ho, Wo)
    textbook = F.interpolate(x.double().permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear", align_corners=False)
    assert ((ref - textbook).abs() <= 1e-6 * x.abs().max()).all()
    _within(ref, bound, bilinear_f32(x, Ho, Wo).double(), "fp32 bilinear")


def test_bilinear_same_size_is_the_layout_change():
    x = torch.randn(2, 5, 7, 3, generator=_g("same"), dtype=D)
    ref, bound = R.bilinear(x, 5, 7)
    assert torch.equal(ref, x.permute(0, 3, 1, 2)) and (bound <= 4 * R.U * ref.abs() + 1e-29).all()


def test_bilinear_fault_leaves_the_bound():
    x = torch.randn(1, 7, 13, 4, generator=_g("swap"))
    ref, bound = R.bilinear(x.double(), 20, 5)
    _outside(ref, bound, bilinear_f32(x, 20, 5, swap=True).double(), "x and y weights swapped")


# ----------------------------------------------------------------------------------------------------------- bias, act, residual
def bias_act_res_f32(x, bias, act, res, after, wrong_side=False):
    C = bias.numel() if bias is not None else 1
    v = x if bias is None else x + bias[torch.arange(x.numel()) % C]
    if after != wrong_side:
        v = v if res is None else v + res
        return _f32_act(v, act)
    v = _f32_act(v, act)
    return v if res is None else v + res


@pytest.mark.parametrize("act", [None, "relu", "hswish", "gelu", "sigmoid"])
@pytest.mark.parametrize("after", [False, True])
def test_bias_act_res_statement(act, after):
    """Against emu_strict.bias_act_res_f32; the float32 restatement inside the bound; total 1001 over C 7."""
    g = _g("bar", act, after)
    x, b, r = torch.randn(1001, generator=g) * 3, torch.randn(7, generator=g), torch.randn(1001, generator=g) * 2
    ref, bound = R.bias_act_res(x.double(), b.double(), act, r.double(), after)
    _close(ref, E.bias_act_res_f32(x.double().view(-1, 1), b.double()[torch.arange(1001) % 7].view(-1, 1), act, r.double().view(-1, 1),
                                   after).view(-1))
    _within(ref, bound, bias_act_res_f32(x, b, act, r, after).double(), "fp32 bias_act_res")


@pytest.mark.parametrize("after", [False, True])
def test_bias_act_res_fault_leaves_the_bound(after):
    g = _g("bar fault", after)
    x, b, r = torch.randn(1001, generator=g) * 3, torch.randn(7, generator=g), torch.randn(1001, generator=g) * 2
    ref, bound = R.bias_act_res(x.double(), b.double(), "relu", r.double(), after)
    _outside(ref, bound, bias_act_res_f32(x, b, "relu", r, after, wrong_side=True).double(), "activation on the wrong side")


def test_strict_gelu_charge_covers_erff():
    """float32 GELU as es3_act states it (erff of the rounded x / sqrt 2) against fp64 GELU, inside L_ACT (4u |x|) + eps_act."""
    x = torch.linspace(-8, 8, 20001, dtype=torch.float32)
    y = 0.5 * x * (1 + torch.erf(x * 0.70710678118654752440))
    ref = F.gelu(x.double())
    assert ((y.double() - ref).abs() <= R.eps_act(x.double(), "gelu") + 4 * R.U * ref.abs() + 1e-45).all()
