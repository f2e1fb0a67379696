"""The fp64 statements of tests/ref_fwd.py against textbook float64 torch (F.conv2d, F.hardswish, F.layer_norm, the reference's
ReLU linear attention, softmax window attention), the tie-band logic on constructed midpoints, and the host emulation of
es3_round_taps_sum_bf16.  No GPU needed."""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

import ref_fwd as R



@pytest.fixture(autouse=True)
def _float64_default():
    """Factory functions make float64 inside this module's tests only."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


def _g(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _bf(t):
    return t.to(torch.bfloat16).double()


def _within(ref, bound, other, what):
    err = (ref - other).abs()
    assert (err <= bound).all(), f"{what}: {(err > bound).sum()} elements outside the bound (max err {err.max():.3g})"
    assert (bound > 0).all()


# ----------------------------------------------------------------------------------------------------------- rounding
def test_rn_bf16_matches_fp32_rounding():
    """For fp32 values (no double rounding possible) the direct fp64 rounding is torch's fp32 -> bf16 round-to-nearest-even."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(100000, generator=g, dtype=torch.float32) * torch.exp(torch.randn(100000, generator=g, dtype=torch.float32) * 8)
    mids = (_bf(x.double()) + torch.ldexp(torch.ones(100000), torch.frexp(x.double())[1] - 9)).float()   # near-midpoints
    for v in (x, mids, torch.tensor([0.0, -0.0, 1.0, -3.0, 2.0 ** -126, 1.00390625, 1.01171875], dtype=torch.float32)):
        assert torch.equal(R.rn_bf16(v.double()), v.to(torch.bfloat16).double())


def test_band_charges_only_near_midpoints():
    """v = midpoint + t: with delta > |t| the kernel's rounding may land on either neighbour (one step charged), with delta < |t|
    it cannot (nothing charged); a value exactly on a bf16 number is never charged for delta below half a step."""
    one = torch.tensor(1.0)
    step = 2.0 ** -7
    mid = one + step / 2                                # between 1 and 1 + 2^-7
    for t in (1e-6, -1e-6, 3e-9):
        v = mid + t
        r, dev = R.band(v, torch.tensor(2 * abs(t)))
        assert dev.item() == step and r.item() in (1.0, 1.0 + step)
        r, dev = R.band(v, torch.tensor(abs(t) / 2))
        assert dev.item() == 0.0
    r, dev = R.band(one + 0.5, torch.tensor(step / 2 * 0.99))
    assert r.item() == 1.5 and dev.item() == 0.0
    # at a binade boundary the step above is twice the step below: the charge is the larger one
    v = torch.tensor(2.0 - 2.0 ** -9)                   # midpoint of 2 - 2^-8 and 2
    _, dev = R.band(v, torch.tensor(2.0 ** -8))
    assert dev.item() == 2.0 ** -7 or dev.item() == 2.0 ** -8
    assert (R.band(-v, torch.tensor(2.0 ** -8))[1] == dev).all()


# ----------------------------------------------------------------------------------------------------------- convolutions
@pytest.mark.parametrize("ks,stride,act,bias", [(3, 1, "hswish", True), (3, 2, "relu", False), (5, 1, "gelu", True), (5, 2, None, True)])
def test_dwconv_statement(ks, stride, act, bias):
    g = _g("dw", ks, stride, act)
    x = _bf(torch.randn(2, 9, 7, 24, generator=g))
    w = torch.randn(ks * ks, 24, generator=g) / ks
    b = torch.randn(24, generator=g) if bias else None
    ref, bound = R.dwconv(x, w, b, ks, stride, act)
    tb = F.conv2d(x.permute(0, 3, 1, 2), w.t().reshape(24, 1, ks, ks), b, stride=stride, padding=ks // 2, groups=24)
    tb = {None: lambda t: t, "relu": F.relu, "hswish": F.hardswish, "gelu": F.gelu}[act](tb).permute(0, 2, 3, 1)
    assert torch.allclose(ref, tb, rtol=1e-12, atol=1e-12)
    assert (bound >= 2.0 ** -8 * ref.abs()).all()


def _mbconv_textbook(x, w1, s1, b1, wdw, b2, w3, s3, b3, stride, res):
    """ops.py MBConv in float64 with nn layers: expand 1x1 + BN + hswish, depthwise 3x3 + BN + hswish, project 1x1 + BN, rounding
    e and d to bf16 (through fp32, the way a bf16 network materialises them)."""
    xn = x.permute(0, 3, 1, 2)
    mid = w1.shape[0]
    e = F.hardswish(F.conv2d(xn, w1[:, :, None, None]) * s1.view(1, -1, 1, 1) + b1.view(1, -1, 1, 1))
    e = e.float().to(torch.bfloat16).double()
    d = F.hardswish(F.conv2d(e, wdw.t().reshape(mid, 1, 3, 3), b2, stride=stride, padding=1, groups=mid))
    d = d.float().to(torch.bfloat16).double()
    y = F.conv2d(d, w3[:, :, None, None]) * s3.view(1, -1, 1, 1) + b3.view(1, -1, 1, 1)
    return (y + xn if res else y).permute(0, 2, 3, 1)


def _mb_operands(cin, mid, cout, g, B=2, H=9, W=11):
    x = _bf(torch.randn(B, H, W, cin, generator=g))
    w1 = _bf(torch.randn(mid, cin, generator=g) / math.sqrt(cin))
    s1, b1 = torch.rand(mid, generator=g) + 0.5, torch.randn(mid, generator=g) * 0.2
    wdw, b2 = _bf(torch.randn(9, mid, generator=g) / 3), torch.randn(mid, generator=g) * 0.2
    w3 = _bf(torch.randn(cout, mid, generator=g) / math.sqrt(mid))
    s3, b3 = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.2
    return x, w1, s1, b1, wdw, b2, w3, s3, b3


@pytest.mark.parametrize("cin,mid,cout,stride,res", [(32, 128, 32, 1, True), (16, 64, 32, 2, False)])
def test_mbconv_statement(cin, mid, cout, stride, res):
    """The statement equals the textbook block except where a bf16 rounding of e or d is ambiguous, and there its bound covers the
    difference; the typical output bound stays at the output's own rounding."""
    ops_ = _mb_operands(cin, mid, cout, _g("mb", cin, stride))
    ref, bound, dev_e, dev_d = R.mbconv(*ops_, stride, res)
    tb = _mbconv_textbook(*ops_, stride, res)
    _within(ref, bound, tb, "mbconv")
    assert (dev_e > 0).any() and (dev_d > 0).any()
    assert (bound / (2.0 ** -8 * ref.abs())).median() < 2.0          # the charges keep the typical bound near the output rounding


def test_mbconv_band_carries_one_step():
    """An expand output placed exactly at a bf16 midpoint (x = 1, w1 = the midpoint, s1 = 1, b1 = 0, relu-free hswish region
    avoided by act=None): the bound of the outputs its depthwise taps reach includes that step times |tap| |w3|."""
    C = 16
    x = torch.zeros(1, 3, 3, C)
    x[0, 1, 1, 0] = 1.0
    w1 = torch.zeros(4 * C, C)
    w1[0, 0] = 1.0 + 2.0 ** -8                          # midpoint of 1 and 1 + 2^-7
    ones, zeros = torch.ones(4 * C), torch.zeros(4 * C)
    wdw = torch.zeros(9, 4 * C)
    wdw[4, 0] = 1.0
    w3 = torch.zeros(C, 4 * C)
    w3[0, 0] = 1.0
    ref, bound, dev_e, dev_d = R.mbconv(x, w1, ones, zeros, wdw, zeros, w3, torch.ones(C), torch.zeros(C), 1, False, act=None)
    assert dev_e[0, 1, 1, 0] == 2.0 ** -7 and (dev_e > 0).sum() == 1
    assert bound[0, 1, 1, 0] >= 2.0 ** -7 and bound[0, 0, 0, 0] < 1e-20


def test_dwproj_stem_dsconv_narrow_statements():
    g = _g("misc")
    mid = _bf(torch.randn(2, 6, 10, 64, generator=g))
    wdw, b2 = _bf(torch.randn(9, 64, generator=g) / 3), torch.randn(64, generator=g)
    w3, s3, b3 = _bf(torch.randn(16, 64, generator=g) / 8), torch.rand(16, generator=g) + 0.5, torch.randn(16, generator=g)
    res = _bf(torch.randn(2, 6, 10, 16, generator=g))
    ref, bound = R.dwproj(mid, wdw, b2, w3, s3, b3, res)
    d = F.hardswish(F.conv2d(mid.permute(0, 3, 1, 2), wdw.t().reshape(64, 1, 3, 3), b2, padding=1, groups=64))
    d = d.float().to(torch.bfloat16).double()
    tb = (F.conv2d(d, w3[:, :, None, None]) * s3.view(1, -1, 1, 1) + b3.view(1, -1, 1, 1)).permute(0, 2, 3, 1) + res
    _within(ref, bound, tb, "dwproj")

    img = torch.randn(2, 3, 13, 9, generator=g)
    w27, bias = torch.randn(27, 24, generator=g) / 5, torch.randn(24, generator=g)
    ref, bound = R.stem_conv(img, w27, bias, "hswish")
    tb = F.hardswish(F.conv2d(img, w27.t().reshape(24, 3, 3, 3), bias, stride=2, padding=1)).permute(0, 2, 3, 1)
    assert torch.allclose(ref, tb, rtol=1e-12, atol=1e-12)

    x = _bf(torch.randn(2, 7, 5, 16, generator=g))
    wd, bd, wp, bp = torch.randn(9, 16, generator=g) / 3, torch.randn(16, generator=g), torch.randn(16, 16, generator=g) / 4, torch.randn(16, generator=g)
    ref, bound = R.dsconv_res(x, wd, bd, wp, bp, "relu")
    m = F.relu(F.conv2d(x.permute(0, 3, 1, 2), wd.t().reshape(16, 1, 3, 3), bd, padding=1, groups=16)).float().to(torch.bfloat16).double()
    tb = (F.conv2d(m, wp[:, :, None, None], bp) + x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    _within(ref, bound, tb, "dsconv_res")

    x = _bf(torch.randn(2, 9, 12, 32, generator=g))
    w = _bf(torch.randn(48, 32, 3, 3, generator=g) / 17)
    sc, bi = torch.rand(48, generator=g) + 0.5, torch.randn(48, generator=g)
    ref, _ = R.conv3x3_s2_narrow(x, w.permute(2, 3, 0, 1).reshape(9, 48, 32), sc, bi, "gelu")
    tb = F.gelu(F.conv2d(x.permute(0, 3, 1, 2), w, stride=2, padding=1) * sc.view(1, -1, 1, 1) + bi.view(1, -1, 1, 1))
    assert torch.allclose(ref, tb.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)


# ----------------------------------------------------------------------------------------------------------- LiteMLA
@pytest.mark.parametrize("dim,chunk,split,HW", [(16, 512, True, 513), (16, 128, False, 1), (32, 128, False, 300)])
def test_litemla_statement(dim, chunk, split, HW):
    """Against the reference's relu_linear_att (F.pad(v, value=1), (v k^T) q, out[:-1] / (out[-1] + eps)); the partials sum to KV."""
    g = _g("lm", dim, HW)
    heads2, B = 3, 2
    ms = _bf(torch.randn(B, HW, heads2 * 3 * dim + 8, generator=g))
    (y, yb), (part, pb) = R.litemla_attn(ms, heads2, dim, 1e-15, chunk, split)
    t = ms[..., :heads2 * 3 * dim].reshape(B, HW, heads2, 3 * dim).permute(0, 2, 3, 1)   # [B, h, 3 dim, HW]
    q, k, v = F.relu(t[:, :, :dim]), F.relu(t[:, :, dim:2 * dim]), F.pad(t[:, :, 2 * dim:], (0, 0, 0, 1), value=1.0)
    kv = v @ k.transpose(-1, -2)
    out = kv @ q
    att = (out[:, :, :-1] / (out[:, :, -1:] + 1e-15)).permute(0, 3, 1, 2).reshape(B, HW, heads2 * dim)
    assert torch.allclose(y, att, rtol=1e-10, atol=1e-12)
    assert torch.allclose(part.sum(2), kv, rtol=1e-12, atol=1e-12)
    assert part.shape == (B, heads2, (HW + chunk - 1) // chunk, dim + 1, dim)
    assert (yb >= 2.0 ** -8 * y.abs()).all()


def test_litemla_aggreg_statement():
    g = _g("agg")
    C3 = 48
    ms = _bf(torch.randn(2, 7, 9, 2 * C3, generator=g))
    wd, wp = _bf(torch.randn(25, C3, generator=g) / 5), _bf(torch.randn(C3, 16, generator=g) / 4)
    ref, bound = R.litemla_aggreg(ms, wd, wp, C3)
    a = F.conv2d(ms[..., :C3].permute(0, 3, 1, 2), wd.t().reshape(C3, 1, 5, 5), padding=2, groups=C3).float().to(torch.bfloat16).double()
    tb = F.conv2d(a, wp[:, :, None, None], groups=C3 // 16).permute(0, 2, 3, 1)
    _within(ref, bound, tb, "aggreg")


# ----------------------------------------------------------------------------------------------------------- TinyViT / RepViT
@pytest.mark.parametrize("H,W,ws", [(14, 14, 7), (9, 16, 7), (20, 15, 14)])
def test_win_attn_statement(H, W, ws):
    """Against softmax attention over the zero-padded window partition (padded tokens = qkv_pad), cropped, with the unnormalised
    probabilities rounded to bf16 before PV (through fp32) and the row sums taken before that rounding."""
    g = _g("win", H, W, ws)
    B, heads = 2, 2
    C = 32 * heads
    qkv = _bf(torch.randn(B * H * W, 3 * C, generator=g))
    pad = _bf(torch.randn(3 * C, generator=g))
    bias = torch.randn(heads, ws * ws, ws * ws, generator=g) * 3
    ref, bound = R.win_attn_bias(qkv, pad, bias, B, H, W, C, heads, ws, 32 ** -0.5)
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    full = pad.expand(B, Hp, Wp, 3 * C).clone()
    full[:, :H, :W] = qkv.reshape(B, H, W, 3 * C)
    win = full.reshape(B, Hp // ws, ws, Wp // ws, ws, heads, 3, 32).permute(0, 1, 3, 5, 6, 2, 4, 7).reshape(-1, heads, 3, ws * ws, 32)
    q, k, v = win[:, :, 0], win[:, :, 1], win[:, :, 2]
    s = q @ k.transpose(-1, -2) * 32 ** -0.5 + bias
    p = torch.exp(s - s.amax(-1, keepdim=True))
    o = (p.float().to(torch.bfloat16).double() @ v) / p.sum(-1, keepdim=True)       # [nwin, heads, N, 32]
    o = o.reshape(B, Hp // ws, Wp // ws, heads, ws, ws, 32).permute(0, 1, 4, 2, 5, 3, 6).reshape(B, Hp, Wp, C)[:, :H, :W]
    _within(ref, bound, o.reshape(B * H * W, C), "win_attn")


def test_layernorm_channel_mean_scale_statements():
    g = _g("ln")
    x = _bf(torch.randn(37, 448, generator=g) * 0.1 + 40)                            # mean-shifted rows
    gm, bt = torch.randn(448, generator=g), torch.randn(448, generator=g)
    ref, bound = R.layernorm(x, gm, bt, 1e-5)
    assert torch.allclose(ref, F.layer_norm(x, (448,), gm, bt, 1e-5), rtol=1e-10, atol=1e-10)
    assert (bound >= 2.0 ** -8 * ref.abs()).all()
    x = _bf(torch.randn(3, 300, 40, generator=g))
    ref, _ = R.channel_mean(x)
    assert torch.allclose(ref, x.mean(1))
    gate = torch.rand(3, 40, generator=g)
    ref, _ = R.scale_channels(x, gate)
    assert torch.equal(ref, x * gate[:, None])


# ----------------------------------------------------------------------------------------------------------- round_taps
@pytest.mark.parametrize("KK,C", [(9, 64), (25, 96), (9, 1000), (1, 5)])
def test_round_taps_emulation_properties(KK, C):
    """bf16-representable, at most one bf16 step from nearest rounding, and a tap sum at least as close to the fp32 sum."""
    g = _g("taps", KK, C)
    w = (torch.randn(KK, C, generator=g, dtype=torch.float32) / KK)
    w[:, :3] = 0.0
    w[0, 3] = 1e-40                                                                   # a subnormal tap: no move from it
    r = R.round_taps_sum_emu(w)
    assert torch.equal(r, r.to(torch.bfloat16).float())
    near = w.to(torch.bfloat16).float()
    assert ((r - near).abs() <= near.abs() * 2.0 ** -7 * 1.01 + 1e-38).all()
    sw = w.double().sum(0)
    assert ((r.double().sum(0) - sw).abs() <= (near.double().sum(0) - sw).abs() + 1e-7).all()
    assert torch.equal(r[:, :3], torch.zeros(KK, 3))
